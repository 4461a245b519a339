"""Encode streams for compute-sanitizer (one GPU): 1 KB pieces fed in misaligned blocks, lines longer than a piece, the
three output forms and a failing sink, each compared with encode_packed of the same lines, so a run that is clean but
wrong still fails.
    compute-sanitizer --tool memcheck --error-exitcode 9 python tools/sanitize_encode_file.py
`--emulate` runs the same script on the CPU SIMT emulator (a dry run)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_encode_file_gpu as F  # noqa: E402
from youtokentome_b200 import _lib  # noqa: E402
from youtokentome_b200.youtokentome import BPE  # noqa: E402


def main():
    if "--emulate" in sys.argv:
        from _emu import emu_lib
        os.environ.setdefault("YT_EMU_SMS", "2")
        _lib._lib = emu_lib()
    L = _lib.lib()
    bpe = BPE(F.model())
    n_ok = 0
    cases = [c[1] for c in F.edge_cases(small=True) if c[0] in ("no final newline", "utf-8 at the cuts",
                                                                 "line longer than pieces", "long word", "blank lines")]
    for data in cases:
        data = data[:40_000]
        want_ids, want_offs = F.expected(bpe, data, eos=True)
        for kind, fmt in ((7, _lib.STREAM_IDS32), ("random", _lib.STREAM_IDS16), (4093, _lib.STREAM_TEXT)):
            out, ends, _, _ = F.abi_run(L, bpe, data, kind, 1, fmt, eos=1)
            assert np.array_equal(ends, want_offs[1:])
            if fmt == _lib.STREAM_TEXT:
                assert out == F.as_text(want_ids, want_offs)
            else:
                assert np.array_equal(out.astype(np.int32), want_ids)
            n_ok += 1
    F.abi_misuse(L)
    print("sanitize_encode_file: %d checks identical to encode_packed" % n_ok)


if __name__ == "__main__":
    main()

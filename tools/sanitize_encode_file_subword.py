"""Subword encode streams for compute-sanitizer (one GPU): 1 KB pieces fed in misaligned blocks, <UNK> runs with invalid
bytes, pieces of more than 1 KB, lines longer than a piece and a misuse pass, each compared with the host path
(encode(output_type=SUBWORD)) on the same lines, so a run that is clean but wrong still fails.
    compute-sanitizer --tool memcheck --error-exitcode 9 python tools/sanitize_encode_file_subword.py
`--emulate` runs the same script on the CPU SIMT emulator (a dry run)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_encode_file_gpu as F  # noqa: E402
import test_encode_file_subword_gpu as S  # noqa: E402
from youtokentome_b200 import _lib  # noqa: E402
from youtokentome_b200.youtokentome import BPE  # noqa: E402


def main():
    if "--emulate" in sys.argv:
        from _emu import emu_lib
        os.environ.setdefault("YT_EMU_SMS", "2")
        _lib._lib = emu_lib()
    L = _lib.lib()
    n_ok = 0
    rng = np.random.default_rng(2)
    long_words = b"\n".join(b" ".join(b"ab" * int(k) for k in rng.integers(1, 2500, 6)) for _ in range(8)) + b"\n"
    cases = [("unk", S.unk_lines(120)), ("long", long_words)]
    cases += [("base", c[1][:40_000]) for c in F.edge_cases(small=True)
              if c[0] in ("no final newline", "invalid bytes at the cuts", "line longer than pieces", "blank lines")]
    for kind, data in cases:
        bpe = BPE(S.model(kind) if kind != "base" else F.model())
        for blocks, kw in ((7, {}), ("random", dict(bos=1, eos=1)), (4093, dict(rev=1, eos=1))):
            flags = {"bos": bool(kw.get("bos")), "eos": bool(kw.get("eos")), "reverse": bool(kw.get("rev"))}
            want = S.want_text(bpe, data, **flags)
            got, _, _ = S.abi_run(L, bpe, data, blocks, 1, **kw)
            assert got == want, kind
            n_ok += 1
    S.abi_misuse(L)
    print("sanitize_encode_file_subword: %d checks identical to the host path" % n_ok)


if __name__ == "__main__":
    main()

"""Decode streams for compute-sanitizer (one GPU): 1 KB pieces, id text fed in misaligned blocks, lines longer than a
piece, zero runs across rounds, both input forms and every misuse case, each compared with `yttm decode` or decode of
the same ids, so a run that is clean but wrong still fails.
    compute-sanitizer --tool memcheck --error-exitcode 9 python tools/sanitize_decode_file.py
`--emulate` runs the same script on the CPU SIMT emulator (a dry run)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_decode_file_gpu as F  # noqa: E402
import test_encode_file_gpu as EF  # noqa: E402
from youtokentome_b200 import _lib  # noqa: E402


def main():
    if "--emulate" in sys.argv:
        from _emu import emu_lib
        os.environ.setdefault("YT_EMU_SMS", "2")
        _lib._lib = emu_lib()
    L = _lib.lib()
    n_ok = 0
    for name, data in F.parser_cases(small=True):
        if name in ("table", "no final newline", "crlf", "line longer than pieces", "zero runs", "nul and invalid bytes",
                    "random long"):
            F.check_text(EF.model(), data, (1,), F.IGN)
            n_ok += 1
    F.abi(L, small=True)
    F.abi_misuse(L)
    F.out_of_range(L, 1)
    print("sanitize_decode_file: %d checks identical to yttm decode" % (n_ok + 3))


if __name__ == "__main__":
    main()

"""Fed trainings for compute-sanitizer (one GPU): small pieces, misaligned block sizes, per-piece table overflow,
arena and persistent-table growth, each compared with the restatement of tests/_front_ref.py (histogram, words and
pairs of the fed context), so a run that is clean but wrong still fails.
    compute-sanitizer --tool memcheck --error-exitcode 9 python tools/sanitize_train_feed.py
`--emulate` runs the same script on the CPU SIMT emulator (a dry run)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_train_feed_gpu as F  # noqa: E402
import test_train_front_gpu as FG  # noqa: E402
from youtokentome_b200 import _lib  # noqa: E402


def main():
    if "--emulate" in sys.argv:
        from _emu import emu_lib
        os.environ.setdefault("YT_EMU_SMS", "2")
        _lib._lib = emu_lib()
    L = _lib.lib()
    n_ok = 0
    corpora = [F.abi_text(small=True)[:16_000]] + [c[1] for c in F.edge_corpora(small=True) if c[1]][-4:]
    for text in corpora:
        want, cp2id = FG.expected(text)
        for kind, piece_kb in ((7, 1), ("random", 1), (4093, 2)):
            got = F.fed_front(L, text, cp2id, F._sizes(kind), piece_kb)
            FG.assert_same(got, want, "fed in blocks of %s bytes, %d KB pieces" % (kind, piece_kb))
            n_ok += 1
    print("sanitize_train_feed: %d checks identical to the restatement" % n_ok)


if __name__ == "__main__":
    main()

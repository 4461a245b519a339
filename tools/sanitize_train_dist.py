"""The word exchange of multi-GPU training for compute-sanitizer (one GPU): the one-rank front through
dist_export_words and dist_import_words (loaded, pipelined, fed and overflowing shards), and the export at 3 and 5 ranks
followed by every owner's import, where equal words from several sources with counts > 1 meet in one table slot.  Each
is compared with the restatement of tests/_front_ref.py, so a run that is clean but wrong still fails.
    compute-sanitizer --tool racecheck python tools/sanitize_train_dist.py
`--emulate` runs the same script on the CPU SIMT emulator (a dry run)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _cases  # noqa: E402
import test_train_dist_gpu as TD  # noqa: E402
import test_train_front_gpu as FG  # noqa: E402
from youtokentome_b200 import _lib  # noqa: E402


def main():
    dev = "--emulate" not in sys.argv
    if not dev:
        from _emu import emu_lib
        os.environ.setdefault("YT_EMU_SMS", "2")
        _lib._lib = emu_lib()
    L = _lib.lib()
    n_ok = 0
    text = _cases.dirty_zipf_text(30_000)
    TD.check_front(L, FG.corpus("chunk"), "chunk")
    TD.check_front(L, text, "fed", feed_kb=1)
    with FG.env(YTTM_TRAIN_PIPELINE=1, YTTM_TRAIN_PIPELINE_PIECE_KB=3):
        TD.check_front(L, text, "pipelined")
    TD.front_overflow(L, False)
    n_ok += 4
    half = _cases.zipf().text(8_000)
    for world in (3, 5):
        TD.check_exports(L, half + b" " + half, world, dev)
        TD.check_exports(L, text, world, dev, feed_rank=world - 1)
        n_ok += 2
    print("sanitize_train_dist: %d checks identical to the restatement" % n_ok)


if __name__ == "__main__":
    main()

"""The training byte passes on device-resident corpora at base offsets 1..15, for compute-sanitizer (one GPU):
    PYTORCH_NO_CUDA_MEMORY_CACHING=1 compute-sanitizer --tool memcheck --error-exitcode 9 \\
        python tools/sanitize_train_front.py
Every corpus sits at the END of its own allocation (with the caching allocator off, each torch tensor is one
cudaMalloc), so a read past the corpus is a read past the allocation and memcheck reports it.  Every result is also
compared with the restatement of tests/_front_ref.py, so a run that is clean but wrong still fails.  `--emulate` runs
the same script on the CPU SIMT emulator (a dry run)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_train_front_gpu as FG  # noqa: E402
from youtokentome_b200 import _lib  # noqa: E402


def main():
    dev = "--emulate" not in sys.argv
    if not dev:
        from _emu import emu_lib
        os.environ.setdefault("YT_EMU_SMS", "2")
        _lib._lib = emu_lib()
    L = _lib.lib()
    corpora = [FG.chunk_corpus()[:20_000], FG.soup(20_000, seed=21)] + FG.length_corpora()[::7]
    n_ok = 0
    for off in range(1, 16):
        for k, text in enumerate(corpora):
            FG.check(L, text, "corpus %d" % k, off=off, dev=dev)
            n_ok += 1
    print("sanitize_train_front: %d checks identical to the restatement" % n_ok)


if __name__ == "__main__":
    main()

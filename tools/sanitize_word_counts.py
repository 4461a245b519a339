"""Word-count tables for compute-sanitizer (one GPU): small tables fed as device lists whose arrays sit at the very end
of their allocations, the bytes at misaligned bases, mixed with text blocks in 1 KB pieces, each compared with the
restatement of tests/_front_ref.py (histogram, words and pairs of the fed context); then count_words and
train_from_counts against BPE.train on the expanded text, so a run that is clean but wrong still fails.
    compute-sanitizer --tool memcheck --error-exitcode 9 python tools/sanitize_word_counts.py
`--emulate` runs the same script on the CPU SIMT emulator (a dry run)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_word_counts_gpu as W  # noqa: E402
from youtokentome_b200 import _lib  # noqa: E402


def at_end(shift):
    """An array copied to the last bytes of a device allocation (the bytes array `shift` bytes off alignment)."""
    def place(a):
        a = np.ascontiguousarray(a)
        s = shift if a.dtype == np.uint8 else 0
        if "--emulate" in sys.argv:
            buf = np.zeros(a.nbytes + s, dtype=np.uint8)
            buf[s:] = a.view(np.uint8)
            return buf[s:].view(a.dtype)
        import torch
        raw = torch.empty(a.nbytes + s, dtype=torch.uint8, device="cuda")
        view = raw[raw.numel() - a.nbytes:]
        view.copy_(torch.from_numpy(a.view(np.uint8).copy()))
        return view
    return place


def main():
    if "--emulate" in sys.argv:
        from _emu import emu_lib
        os.environ.setdefault("YT_EMU_SMS", "2")
        _lib._lib = emu_lib()
    L = _lib.lib()
    n_ok = 0
    for shift in (0, 1, 3, 7):
        W.abi_mixed(L, at_end(shift), small=True)
        n_ok += 1
    for seed in (1, 3):
        words, counts = W.random_table(seed, 80)
        W.check_table(None, words, counts, 150, 1.0)
        n_ok += 1
    W.check_counting(W.counting_corpora(small=True)[1], piece_kbs=(1,))
    n_ok += 1
    print("sanitize_word_counts: %d checks identical to the restatement" % n_ok)


if __name__ == "__main__":
    main()

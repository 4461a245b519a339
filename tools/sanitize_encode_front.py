"""The word finder and the word-merge kernels of device encode on device-resident batches at base offsets 1..15, for
compute-sanitizer (one GPU):
    PYTORCH_NO_CUDA_MEMORY_CACHING=1 compute-sanitizer --tool memcheck python tools/sanitize_encode_front.py
    PYTORCH_NO_CUDA_MEMORY_CACHING=1 compute-sanitizer --tool racecheck python tools/sanitize_encode_front.py --long-only
Every batch sits at the END of its own allocation (with the caching allocator off, each torch tensor is one
cudaMalloc), so a read past the batch is a read past the allocation and memcheck reports it.  The last sentence ends
in a truncated E2 96, in a lone E2, in a 33-byte word or in a 513-byte word (block-per-word kernel); `--long-only`
keeps the batches with words of more than 512 slots, where racecheck looks at the warps of encode_long_words_kernel.
Every result is also compared with the restatement of tests/_encode_ref.py, so a run that is clean but wrong still
fails.  `--emulate` runs the same script on the CPU SIMT emulator (a dry run)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _bind  # noqa: E402
import test_encode_words_gpu as WG  # noqa: E402
from youtokentome_b200 import _lib  # noqa: E402


def main():
    dev = "--emulate" not in sys.argv
    if not dev:
        from _emu import emu_lib
        os.environ.setdefault("YT_EMU_SMS", "2")
        _lib._lib = emu_lib()
    oracle = _bind.Oracle()
    n_ok = 0
    if "--long-only" not in sys.argv:
        WG.check_misaligned_device_batches(oracle, dev)
        n_ok += 30
    case = WG.runs_case(oracle)
    words = [b"c" * 505 + b"a" * 600 + b"b" * 40, b"ab" * 300 + b"a" * 1100, b"a" * 513]
    for shift in (1, 7, 15):
        sents = [b"ab " + words[0], words[1] + b" c", b"b " + words[2]]
        buf, offs = _bind._pack(sents)
        WG._equal(WG._device(case.g, buf, offs, shift, shift, dev, {}), case.want(sents), sents, shift)
        n_ok += 1
    print("sanitize_encode_front: %d batches identical to the restatement" % n_ok)


if __name__ == "__main__":
    main()

"""Small overlapping-windows workload for compute-sanitizer (run on one GPU):
    compute-sanitizer --tool memcheck --error-exitcode 9 python tools/sanitize_windows.py
A model trained by the oracle (test infrastructure), then yttm_enc_run_windows_device through BPE.encode_windows:
batches whose bytes start at every base 1..15 mod 16 and end at the last byte of their allocation, offsets[0] > 0, a
word of more than 512 slots cut by many windows, K = 1, step 1 and wide windows, ids and spans.  Every result is
compared with the definition of tests/test_encode_windows_gpu.py over encode_packed's output, so a run that is clean but
wrong still fails.  `--emulate` runs the checks on the CPU SIMT emulator (a dry run, host inputs only)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _bind  # noqa: E402
import _cases  # noqa: E402
from _bind import _pack, tmp_model_path  # noqa: E402
from youtokentome_b200 import _lib  # noqa: E402


def main():
    emulate = "--emulate" in sys.argv
    if emulate:
        from _emu import emu_lib
        os.environ.setdefault("YT_EMU_SMS", "2")
        _lib._lib = emu_lib()
    import test_encode_padded_gpu as PG
    import test_encode_spans_gpu as SG
    import test_encode_windows_gpu as WG
    _bind.build_checkers()
    orc = _bind.Oracle()
    m = tmp_model_path("sw")
    orc.train(_cases.dirty_zipf_text(30_000), m, 700, 0.95)
    bpe = SG._bpe(m)
    long_word = b"".join(_cases.zipf().sentences(20, 60, seed=6)).replace(b" ", b"")
    sents = _cases.zipf_sentences(300) + list(_cases.EDGE_SENTENCES) + SG.ADVERSARIAL + [long_word, b"", b"x " + long_word]
    data, offs = _pack(sents)
    n_ok = 0
    for kw in (dict(), dict(bos=True, eos=True, reverse=True), dict(eos=True)):
        _, _, k = WG.check_against_packed(bpe, m, data, offs, [kw], [(1, 0), (5, 4), (9, 2), (130, 7)], not emulate,
                                          outs=["numpy"])
        n_ok += k
    if not emulate:
        import torch
        _, pad, bid, eid = PG._special(m)
        ids, oo, sp = bpe.encode_packed(data, offs, with_spans=True)
        for base in range(1, 16):
            # sentence 0 starts `base` bytes into its allocation, the last sentence ends at the allocation's last byte
            whole = torch.empty(base + len(data), dtype=torch.uint8, device="cuda")
            whole[base:] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
            d_offs = torch.from_numpy(offs.astype(np.int64) + base).cuda()
            kw = dict(bos=base % 2 == 1, eos=base % 3 == 0, reverse=base % 4 < 2)
            be = int(kw["bos"]) + int(kw["eos"])
            for K, S in ((1, 0), (2 + base, 1 + base), (3 + base, base % 3)):
                g = bpe.encode_windows(whole, d_offs, K + be, stride=S, with_spans=True, out="cuda", **kw)
                want = WG.windows_ref(ids, oo, K + be, S, bid, eid, pad, kw["bos"], kw["eos"], kw["reverse"], sp,
                                      offs.astype(np.int64) + base)
                for a, b in zip(g, want):
                    assert torch.equal(a.cpu(), b), (base, K, S)
                n_ok += 1
            del whole
    del bpe
    os.remove(m)
    print("sanitize_windows: %d calls, windows identical to the definition" % n_ok)


if __name__ == "__main__":
    main()

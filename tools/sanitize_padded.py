"""Small padded-rows workload for compute-sanitizer (run on one GPU):
    compute-sanitizer --tool memcheck --error-exitcode 9 python tools/sanitize_padded.py
A model trained by the oracle (test infrastructure), then yttm_enc_run_padded* through BPE.encode_padded: batches whose
bytes start at every base 1..15 mod 16 and end at the last byte of their allocation, offsets[0] > 0, long words cut
inside (the block kernel), L = None and fixed, ids and spans, the host-buffer form.  Every result is compared with the
definition of tests/test_encode_padded_gpu.py over encode_packed's output, so a run that is clean but wrong still fails.
`--emulate` runs the same script on the CPU SIMT emulator (a dry run, host inputs only)."""
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
    _bind.build_checkers()
    orc = _bind.Oracle()
    m = tmp_model_path("sp")
    orc.train(_cases.dirty_zipf_text(30_000), m, 700, 0.95)
    bpe = SG._bpe(m)
    long_word = b"".join(_cases.zipf().sentences(20, 60, seed=6)).replace(b" ", b"")
    sents = _cases.zipf_sentences(300) + list(_cases.EDGE_SENTENCES) + SG.ADVERSARIAL + [long_word, b"", b"x " + long_word]
    data, offs = _pack(sents)
    n_ok = 0
    for kw in (dict(), dict(bos=True, eos=True, reverse=True), dict(eos=True)):
        be = int(kw.get("bos", False)) + int(kw.get("eos", False))
        _, _, k = PG.check_against_packed(bpe, m, data, offs, [kw], [None, max(1, be), 5 + be, 130], not emulate,
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
            for L in (None, 3 + base):
                kw = dict(bos=base % 2 == 1, eos=base % 3 == 0, reverse=base % 4 < 2)
                g = bpe.encode_padded(whole, d_offs, max_length=L, with_spans=True, out="cuda", **kw)
                want = PG.padded_ref(ids, oo, L, bid, eid, pad, kw["bos"], kw["eos"], kw["reverse"], sp,
                                     offs.astype(np.int64) + base)
                assert torch.equal(g[0].cpu(), want[0]) and torch.equal(g[1].cpu(), want[1]), (base, L)
                assert torch.equal(g[2].cpu(), want[2]), (base, L)
                n_ok += 1
            del whole
    del bpe
    os.remove(m)
    print("sanitize_padded: %d calls, padded rows identical to the definition" % n_ok)


if __name__ == "__main__":
    main()

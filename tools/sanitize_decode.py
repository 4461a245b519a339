"""Small decode workload for compute-sanitizer (run on one GPU):
    compute-sanitizer --tool memcheck --error-exitcode 9 python tools/sanitize_decode.py
Models trained by the oracle (test infrastructure), ids from the GPU encoder, then yttm_dec_run through
BPE.decode_packed: multi-script pieces, pieces over 1 KB, ignore sets, empty sentences, offsets that do not start at 0,
and the two error paths (an invalid id, malformed offsets).  Every text is compared with the host BPE.decode, so a run
that is clean but wrong still fails.  `--emulate` runs the same script on the CPU SIMT emulator (a dry run)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _bind  # noqa: E402
import _cases  # noqa: E402
from _bind import tmp_model_path  # noqa: E402
from youtokentome_b200 import _lib  # noqa: E402


def _flat(sents):
    offs = np.zeros(len(sents) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(s) for s in sents])
    return np.array([t for s in sents for t in s], dtype=np.int32), offs


def _texts(text, oo):
    oo = oo.astype(np.int64)
    return [bytes(text[oo[i]:oo[i + 1]]).decode() for i in range(len(oo) - 1)]


def main():
    if "--emulate" in sys.argv:
        from _emu import emu_lib
        os.environ.setdefault("YT_EMU_SMS", "2")
        _lib._lib = emu_lib()
    import youtokentome_b200 as yttm
    from _gpu import GpuEncoder
    _bind.build_checkers()
    orc = _bind.Oracle()
    n_ok = 0
    word = b"abcd" * 400
    for text, vocab, cov in ((_cases.dirty_zipf_text(30_000), 500, 0.98), (b" ".join([word, word[:700], b"abab"] * 5), 22, 1.0)):
        m = tmp_model_path("sd")
        orc.train(text, m, vocab, cov)
        bpe, g = yttm.BPE(m), GpuEncoder(m)
        sents = _cases.zipf_sentences(100) + list(_cases.EDGE_SENTENCES) + [word, word + b" x " + word[:333]]
        ids = g.encode(sents, bos=True, eos=True) + [[], [2, 3]]
        for ign in (None, [2, 3], [2, 3, -4, 10**6]):
            flat, offs = _flat(ids)
            assert _texts(*bpe.decode_packed(flat, offs, ignore_ids=ign)) == bpe.decode(ids, ignore_ids=ign)
            shifted = np.concatenate([np.full(5, 7, np.int32), flat])
            assert _texts(*bpe.decode_packed(shifted, offs + 5, ignore_ids=ign)) == bpe.decode(ids, ignore_ids=ign)
            n_ok += 2
        flat, offs = _flat(ids + [[bpe.vocab_size()]])
        try:
            bpe.decode_packed(flat, offs)
            raise AssertionError("an invalid id was accepted")
        except ValueError as e:
            assert "id must be in the range" in str(e)
        bad = offs.copy()
        bad[3], bad[4] = bad[4], bad[3] - 1
        try:
            bpe.decode_packed(flat, bad)
            raise AssertionError("decreasing offsets were accepted")
        except ValueError as e:
            assert "offsets must be non-decreasing" in str(e)
        n_ok += 2
        del bpe, g
        os.remove(m)
    print("sanitize_decode: %d checks identical to the host decode" % n_ok)


if __name__ == "__main__":
    main()

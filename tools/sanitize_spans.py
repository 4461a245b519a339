"""Small spans / subwords workload for compute-sanitizer (run on one GPU):
    compute-sanitizer --tool memcheck --error-exitcode 9 python tools/sanitize_spans.py
Models trained by the oracle (test infrastructure), then yttm_enc_run_spans* / yttm_enc_run_subwords* through
BPE.encode_packed(with_spans=True) / BPE.encode_subwords_packed: invalid UTF-8, <UNK> runs, words over 512 bytes (the
block kernel), dropout, empty sentences and offsets that do not start at 0.  Spans are compared with the restatement of
tests/test_encode_spans_gpu.py and pieces with the host encode(output_type=SUBWORD), so a run that is clean but wrong
still fails.  `--emulate` runs the same script on the CPU SIMT emulator (a dry run)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _bind  # noqa: E402
import _cases  # noqa: E402
from _bind import _pack, tmp_model_path  # noqa: E402
from youtokentome_b200 import _lib  # noqa: E402


def main():
    if "--emulate" in sys.argv:
        from _emu import emu_lib
        os.environ.setdefault("YT_EMU_SMS", "2")
        _lib._lib = emu_lib()
    import test_encode_spans_gpu as SG
    _bind.build_checkers()
    orc = _bind.Oracle()
    n_ok = 0
    long_word = b"".join(_cases.zipf().sentences(20, 60, seed=6)).replace(b" ", b"")
    for vocab, cov in ((600, 0.9), (900, 1.0)):
        m = tmp_model_path("ss")
        orc.train(_cases.dirty_zipf_text(30_000), m, vocab, cov)
        bpe, model = SG._bpe(m), SG.Model(m)
        sents = _cases.zipf_sentences(60) + list(_cases.EDGE_SENTENCES) + SG.ADVERSARIAL + [long_word, b"", b"x " + long_word]
        data, offs = _pack(sents)
        for kw, seed in ((dict(), None), (dict(bos=True, eos=True, reverse=True), None), (dict(dropout_prob=0.3), 9)):
            SG.check_batch(bpe, model, data, offs, kw, seed=seed)
            SG.check_batch(bpe, model, b"\xe2\x96" * 5 + data, offs + 10, kw, seed=seed)
            n_ok += 2
        del bpe
        os.remove(m)
    print("sanitize_spans: %d batches with spans and subwords identical to the host paths" % n_ok)


if __name__ == "__main__":
    main()

"""Small train + encode workload for compute-sanitizer (SURVEY §8f-4, second half; run on one GPU):
    compute-sanitizer --tool memcheck  --error-exitcode 9 python tools/sanitize_small.py
    compute-sanitizer --tool racecheck --error-exitcode 9 python tools/sanitize_small.py
    compute-sanitizer --tool synccheck --error-exitcode 9 python tools/sanitize_small.py
Sizes are tiny on purpose (the tools slow kernels down 10 - 100x): stress-shaped and dirty multi-script corpora of a few
KB, RESIDENT and forced-STREAMING merge loops (roomy and tiny exchange segments / table partitions), the default encode kernels with and without dropout, then every
experimental encode variant.  Every result is also compared with the oracle (test infrastructure), so a run that is
clean but wrong still fails.  `--emulate` runs the same script on the CPU SIMT emulator (a dry run of the script)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _bind  # noqa: E402
import _cases  # noqa: E402
from _bind import read_model, tmp_model_path  # noqa: E402
from youtokentome_b200 import _lib, synth  # noqa: E402

ENC_KNOBS = ["YTTM_ENC_PLAIN", "YTTM_ENC_SLOTS", "YTTM_ENC_FIND_CACHED", "YTTM_ENC_FIND_VEC", "YTTM_ENC_BUCKETED", "YTTM_ENC_ZLIN", "YTTM_ENC_LONG", "YTTM_ENC_DEDUP"]


def main():
    if "--emulate" in sys.argv:
        from _emu import emu_lib
        os.environ.setdefault("YT_EMU_SMS", "2")
        _lib._lib = emu_lib()
    from _gpu import GpuEncoder, gpu_train
    _bind.build_checkers()
    orc = _bind.Oracle()
    n_ok = 0
    corpora = [(synth.stress_text(3), 60, 1.0), (synth.stress_text(11), 90, 0.97), (_cases.dirty_zipf_text(30_000), 400, 0.98),
               (synth.readme_corpus(n_lines=60), 120, 1.0)]
    quick = bool(os.environ.get("YTTM_SANITIZE_QUICK"))   # under a sanitizer: fewer corpora, fewer encode variants
    if quick:
        corpora = corpora[1:3]
    for stream, tiny in ((False, False), (True, False), (False, True), (True, True)):
        for k in ("YTTM_FORCE_STREAM", "YTTM_STREAM_Q", "YTTM_STAGES", "YTTM_XQ_SEG_CAP", "YTTM_PAIR_CAP_FLOOR"):
            os.environ.pop(k, None)
        if stream:
            os.environ.update(YTTM_FORCE_STREAM="1", YTTM_STREAM_Q="256", YTTM_STAGES="3")
        if tiny:   # exchange segments overflow, table partitions fill up: the rebuild / relaunch paths
            os.environ.update(YTTM_XQ_SEG_CAP="8", YTTM_PAIR_CAP_FLOOR="16")
        for text, vocab, cov in corpora:
            m_o = tmp_model_path("so")
            orc.train(text, m_o, vocab, cov)
            m_g = gpu_train(text, vocab, cov)
            assert read_model(m_g) == read_model(m_o), "train differs from the oracle (stream=%s)" % stream
            n_ok += 1
            for p in (m_o, m_g):
                os.remove(p)
    text = _cases.dirty_zipf_text(30_000)
    model = tmp_model_path("sm")
    orc.train(text, model, 500, 0.98)
    zc = _cases.zipf()
    long_word = b"".join(zc.sentences(12, 60, seed=6)).replace(b" ", b"")
    sents = _cases.zipf_sentences(150) + list(_cases.EDGE_SENTENCES) + [long_word, b"a" * 700 + b" " + b"a" * 700, long_word + b" x " + long_word]
    g, o = GpuEncoder(model), orc.encoder(model)
    variants = [[]] + [[k] for k in ENC_KNOBS] + [["YTTM_ENC_FIND_VEC", "YTTM_ENC_DEDUP"], ["YTTM_ENC_FIND_CACHED", "YTTM_ENC_BUCKETED", "YTTM_ENC_ZLIN"]]
    if quick:
        variants = [[], ["YTTM_ENC_PLAIN"], ["YTTM_ENC_SLOTS"], ["YTTM_ENC_BUCKETED", "YTTM_ENC_LONG"]]
    for env in variants:
        for k in ENC_KNOBS:
            os.environ.pop(k, None)
        for k in env:
            os.environ[k] = "1"
        assert g.encode(sents, bos=True, eos=True) == o.encode(sents, bos=True, eos=True), env
        assert g.encode(sents, reverse=True) == o.encode(sents, reverse=True), env
        assert g.encode(sents, dropout=0.3, seed=7) == o.encode(sents, dropout=0.3, seed=7), env
        n_ok += 3
    del g
    os.remove(model)
    print("sanitize_small: %d checks identical to the oracle" % n_ok)


if __name__ == "__main__":
    main()

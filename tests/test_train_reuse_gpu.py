"""Training contexts that outlive one training, on the GPU.  Every other training test runs on a fresh context; here a
context trains again after an earlier training left its buffers, flags, timers and counters behind:

  (a) sequences of trainings on the context cached by YTTM_TRAIN_KEEP_CACHE=1 (yttm_api_train_memory): corpora that
      shrink and grow, alphabets and special ids that change, RESIDENT / STREAMING, a grown pair table, pipelined and
      plain ingest.  Each model equals the oracle's (char2id, rules, special tokens) and, byte for byte, the model a
      fresh context writes for the same input without the knob;
  (b) error returns without the knob: no context stays cached, on this thread or on one that exits;
  (c) one yttm_ctx driven through the C ABI again: a second corpus, a second word set, calls that need a build of
      the new corpus before it ran, and a device-resident load after an abandoned pipelined one;
  (d) knobs changed between two cached trainings;
  (e) stage times on a context used again (training report and encoder handle);
  (f) the merge loop across the 20-bit wrap of the exchange stamps.

The bodies take the library: tests/test_train_reuse_emul_cpu.py runs (a) - (e) on the SIMT emulator with smaller
inputs (`small`) and host memory for device buffers (`dev=False`)."""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest

import _cases
import _front_ref as R
import test_train_front_gpu as FG
import test_train_loop_gpu as LG
from _bind import _pack, read_model, tmp_model_path
from youtokentome_b200 import synth

pytestmark = pytest.mark.gpu
KEEP = "YTTM_TRAIN_KEEP_CACHE"
STAMP_MOD = 0xFFFFF          # XQ_STAMP_MOD of merge_loop.cuh: an exchange entry carries round % STAMP_MOD


@pytest.fixture
def lib(product):
    return product


@pytest.fixture
def kept(lib, monkeypatch):
    """The library with YTTM_TRAIN_KEEP_CACHE=1; the context is given back afterwards, so no later test inherits it."""
    monkeypatch.setenv(KEEP, "1")
    try:
        yield lib
    finally:
        lib.yttm_api_release_training_cache()


# ---- trainings through the flat API ---------------------------------------------------------------------------------
def train(L, text, vocab, cov=1.0, pad=0, unk=1, bos=2, eos=3, model=None):
    """yttm_api_train_memory on the calling thread's cached context -> model path; ValueError(message) on failure."""
    model = model if model is not None else tmp_model_path("reuse")
    if L.yttm_api_train_memory(text, len(text), model.encode(), vocab, cov, pad, unk, bos, eos) != 0:
        raise ValueError(L.yttm_api_last_error(None).decode())
    return model


def report(L):
    out = (C.c_double * 17)()
    n = L.yttm_api_train_report(out, 17)
    names = ["n_bytes", "data_len", "n_words", "n_unique", "n_tokens", "n_pairs", "n_merges", "read_s", "h2d_ms",
             "char_hist_ms", "word_count_ms", "tokenise_ms", "pair_hist_ms", "merge_loop_ms", "total_s", "launches",
             "loop_launches"]
    return dict(zip(names[:n], list(out)[:n]))


def on_new_thread(fn, keep=False):
    """fn() on a thread of its own (so on a context of its own: the cache is per thread), with YTTM_TRAIN_KEEP_CACHE
    set or unset for its duration -> (result, exception)."""
    out = {}

    def body():
        try:
            out["r"] = fn()
        except Exception as e:      # noqa: BLE001 - handed to the caller
            out["e"] = e
    old = os.environ.pop(KEEP, None)
    if keep:
        os.environ[KEEP] = "1"
    try:
        t = threading.Thread(target=body)
        t.start()
        t.join()
    finally:
        os.environ.pop(KEEP, None)
        if old is not None:
            os.environ[KEEP] = old
    return out.get("r"), out.get("e")


def check(L, oracle, text, vocab, cov=1.0, **special):
    """One training on the current context: equal to the oracle (or the same error), and its model file equal in bytes
    to the one a fresh context writes for the same input without the knob."""
    m_o = tmp_model_path("orc")
    try:
        oracle.train(text, m_o, vocab, cov, **special)
    except ValueError as e:
        with pytest.raises(ValueError) as ei:
            train(L, text, vocab, cov, **special)
        assert str(ei.value) == str(e)
        return None
    m = train(L, text, vocab, cov, **special)
    a, b = read_model(m_o), read_model(m)
    assert a[0] == b[0], "char2id differs from the oracle (%d bytes, vocab %d)" % (len(text), vocab)
    assert a[2] == b[2], "special tokens differ from the oracle"
    if a[1] != b[1]:
        k = next((i for i, (p, q) in enumerate(zip(a[1], b[1])) if p != q), min(len(a[1]), len(b[1])))
        raise AssertionError("rules differ from the oracle: %d vs %d rules, first difference at %d" % (len(a[1]), len(b[1]), k))
    m_f, err = on_new_thread(lambda: train(L, text, vocab, cov, **special))
    assert err is None, err
    with open(m, "rb") as f, open(m_f, "rb") as g:
        assert f.read() == g.read(), "model file differs from a fresh context's"
    return m


def held(L):
    return L.yttm_api_training_cache_held()


# ---- (a) bodies: cached sequences -------------------------------------------------------------------------------------
def big_text(small):
    return synth.FastZipf(n_words=5_000 if small else 50_000, seed=7).text(60_000 if small else 3 << 20)


def seq_sizes(L, oracle, small=False):
    """big -> tiny -> empty -> medium -> big: the buffers of the context shrink and grow."""
    big, big_vocab = big_text(small), 600 if small else 3000
    tiny, tiny_vocab, tiny_cov, _ = _cases.stress_case(3)
    medium = _cases.dirty_zipf_text(40_000 if small else 200_000)
    for text, vocab, cov in [(big, big_vocab, 1.0), (tiny, tiny_vocab, tiny_cov), (b"", 10, 1.0), (medium, 800, 0.98),
                             (big, big_vocab, 1.0)]:
        check(L, oracle, text, vocab, cov)
    assert held(L) == 1


def _latin(n):
    return synth.readme_corpus(n_lines=n, alphabet="abcdefgh ", seed=4)


def seq_alphabets(L, oracle, small=False):
    """Latin -> Cyrillic + CJK -> Latin at coverage 1.0 / 0.98 / 0.9: no code point of an earlier alphabet may keep
    its id."""
    rus = synth.GOLDEN_TEXTS["russian"][0]
    jap = synth.GOLDEN_TEXTS["japanese"][0]
    cyr_cjk = ((rus + jap) * (5 if small else 40)).encode()
    for text, cov in [(_latin(200 if small else 1000), 1.0), (cyr_cjk, 0.98), (_latin(150 if small else 800), 0.9),
                      (cyr_cjk, 1.0)]:
        vocab = len(set(text.decode())) + 4 + 150
        check(L, oracle, text, vocab, cov)


def seq_special_ids(L, oracle, small=False):
    text = synth.readme_corpus(n_lines=150 if small else 300)
    for cov, sp in [(1.0, dict(pad=-1, unk=5, bos=29, eos=-1)), (1.0, {}), (0.999, dict(pad=7, unk=0, bos=3, eos=299)),
                    (1.0, dict(pad=-1, unk=0, bos=-1, eos=-1))]:
        check(L, oracle, text, 300, cov, **sp)


def seq_resident_streaming(L, oracle, monkeypatch, small=False):
    """RESIDENT -> STREAMING (forced, 64-slot tiles) -> RESIDENT; the knobs are read on every call."""
    texts = [_cases.stress_case(s)[:3] for s in (5, 6, 7)]
    if not small:
        texts.append((_cases.dirty_zipf_text(), 1500, 0.98))
    for stream in (False, True, False):
        if stream:
            monkeypatch.setenv("YTTM_FORCE_STREAM", "1")
            monkeypatch.setenv("YTTM_STREAM_Q", "64")
        else:
            monkeypatch.delenv("YTTM_FORCE_STREAM", raising=False)
            monkeypatch.delenv("YTTM_STREAM_Q", raising=False)
        for text, vocab, cov in texts:
            check(L, oracle, text, vocab, cov)


def seq_pair_table_growth(L, oracle, monkeypatch, small=False):
    """A training whose pair table starts at 16 slots and grows, then trainings with a roomy table."""
    text = _cases.zipf().text(30_000 if small else 100_000)
    monkeypatch.setenv("YTTM_PAIR_CAP_FLOOR", "16")
    check(L, oracle, text, 500 if small else 1000)
    monkeypatch.delenv("YTTM_PAIR_CAP_FLOOR")
    check(L, oracle, text, 500 if small else 1000)
    check(L, oracle, _cases.stress_case(8)[0], *_cases.stress_case(8)[1:3])


def compacting_text(n_words, seed=12):
    """Distinct words "abababab" + 5 letters of twenty: the first merge (a, b) kills 4 of the 14 token slots of every
    word, so every block of the merge loop passes its dead-slot limit and the loop leaves to compact the words."""
    rng = np.random.default_rng(seed)
    tails = rng.choice(20 ** 5, size=n_words, replace=False)
    letters = np.stack([(tails // 20 ** k) % 20 for k in range(5)], axis=1).astype(np.uint8) + ord("c")
    rows = np.concatenate([np.frombuffer(b"abababab", dtype=np.uint8)[None, :].repeat(n_words, 0), letters,
                           np.full((n_words, 1), ord(" "), dtype=np.uint8)], axis=1)
    return rows.tobytes()


def seq_compaction(L, oracle, small=False):
    """A training whose merge loop compacts the words (it relaunches), then one that does not; then the first again."""
    comp = compacting_text(3_000 if small else 200_000)
    plain = synth.readme_corpus(n_lines=100 if small else 300)
    check(L, oracle, comp, 300)
    launches_comp = report(L)["loop_launches"]
    check(L, oracle, plain, 200)
    check(L, oracle, comp, 300)
    assert launches_comp >= 2, "the compacting corpus did not relaunch the merge loop"


def seq_pipelined(L, oracle, monkeypatch, small=False):
    """Plain -> pipelined in 1 KB pieces -> plain; then a pipelined word table that overflows, then a small plain
    training."""
    text = _cases.dirty_zipf_text(30_000 if small else 200_000)
    other = _cases.stress_case(9)[:3]
    for pipe in ("0", "1", "0", "1"):
        monkeypatch.setenv("YTTM_TRAIN_PIPELINE", pipe)
        monkeypatch.setenv("YTTM_TRAIN_PIPELINE_PIECE_KB", "1")
        check(L, oracle, text, 700)
        check(L, oracle, *other)
    monkeypatch.setenv("YTTM_TRAIN_PIPELINE", "1")
    monkeypatch.setenv("YTTM_TRAIN_PIPELINE_PIECE_KB", "64")
    check(L, oracle, FG.overflow_corpus(), 200)
    monkeypatch.setenv("YTTM_TRAIN_PIPELINE", "0")
    check(L, oracle, *_cases.stress_case(10)[:3])


# ---- (b) bodies: error returns without the knob ---------------------------------------------------------------------
def error_after_pipelined_load(L, oracle, monkeypatch):
    """Vocab too small after a pipelined load (the error return comes after char_hist, before build): no context may
    stay cached, and the next training equals the oracle."""
    monkeypatch.delenv(KEEP, raising=False)
    monkeypatch.setenv("YTTM_TRAIN_PIPELINE", "1")
    monkeypatch.setenv("YTTM_TRAIN_PIPELINE_PIECE_KB", "1")
    text = _cases.dirty_zipf_text(30_000)
    with pytest.raises(ValueError, match="Vocabulary size too small"):
        train(L, text, 12)
    assert held(L) == 0, "a training that failed left its context cached"
    with pytest.raises(ValueError, match="Can't open file"):
        train(L, text, 500, model=os.path.join(tmp_model_path("dir"), "missing", "model"))
    assert held(L) == 0, "a training that could not write its model left its context cached"
    monkeypatch.setenv("YTTM_TRAIN_PIPELINE", "0")
    check(L, oracle, *_cases.stress_case(11)[:3])
    check(L, oracle, text, 500)
    assert held(L) == 0


def error_on_exiting_thread(L):
    """The same on a thread that exits afterwards: nothing is left behind (the cache has no destructor at thread
    exit, so a context cached there would hold its device memory for the life of the process)."""
    _, err = on_new_thread(lambda: train(L, _cases.dirty_zipf_text(30_000), 12))
    assert isinstance(err, ValueError) and "Vocabulary size too small" in str(err)
    assert held(L) == 0
    _, err = on_new_thread(lambda: train(L, b"ab ab abc", 20))
    assert err is None and held(L) == 0


# ---- (c) bodies: one yttm_ctx through the C ABI -------------------------------------------------------------------------
def abi_train(ctx, text, merges):
    """load_corpus -> char_hist -> the reference's alphabet (coverage 1.0; 4 special ids first, so the internal ids
    are the model's) -> build -> run -> (the rules (x, y, z), the vocabulary size that asks for `merges` merges)."""
    L = ctx.L
    dl, nd = C.c_uint64(0), C.c_uint64(0)
    assert L.yttm_train_load_corpus(ctx.h, C.cast(C.c_char_p(text), C.c_void_p), len(text), 0) == 0, ctx.err()
    assert L.yttm_train_char_hist(ctx.h, C.byref(dl), C.byref(nd)) == 0, ctx.err()
    set_alphabet(ctx, nd.value)
    assert L.yttm_train_build(ctx.h, None) == 0, ctx.err()
    rc, rules = ctx.run(4 + 1 + nd.value, merges)
    assert rc == 0, ctx.err()
    return [r[:3] for r in rules], 5 + nd.value + merges


def set_alphabet(ctx, n_distinct):
    L = ctx.L
    cps = np.zeros(n_distinct, dtype=np.uint32)
    cnt = np.zeros(n_distinct, dtype=np.uint64)
    L.yttm_train_get_char_hist(ctx.h, cps.ctypes.data, cnt.ctypes.data)
    order = np.lexsort((cps, cnt))[::-1]
    kc = np.concatenate([[R.SPACE_CP], cps[order]]).astype(np.uint32)
    ki = np.arange(4, 4 + len(kc), dtype=np.uint32)
    assert L.yttm_train_set_alphabet(ctx.h, kc.ctypes.data, ki.ctypes.data, len(kc), 4) == 0, ctx.err()


def oracle_rules(oracle, text, vocab):
    m = tmp_model_path("orc")
    oracle.train(text, m, vocab, 1.0)
    return read_model(m)[1]


def abi_two_corpora(L, oracle, small=False):
    a = _cases.zipf().text(20_000 if small else 300_000)
    b = b"\n".join(synth.stress_text(k, 300, train=True) for k in range(20 if small else 60))
    ctx = LG.Ctx(L)
    try:
        for text in (a, b, a):
            rules, vocab = abi_train(ctx, text, 300)
            assert rules == oracle_rules(oracle, text, vocab)
    finally:
        ctx.close()


def abi_import_twice(L, oracle, small=False):
    rng = np.random.default_rng(31)
    n = 1500 if small else 20_000
    w1 = LG.Words.of(*LG.hand_words(rng, n, [3, 5, 8], np.arange(20, 50), np.arange(1000, 1032)))
    w2 = LG.Words.of(*LG.hand_words(rng, n // 2, [2, 4, 12], np.arange(60, 70), np.arange(2000, 2100)))
    ctx = LG.Ctx(L)
    try:
        for w, first in ((w1, 3000), (w2, 4000), (w1, 3000)):
            ctx.import_words(w)
            LG.check_run(ctx, oracle, w, first, 120 if small else 600)
    finally:
        ctx.close()


def abi_calls_before_build(L, oracle):
    """After a full training on corpus A, load_corpus(B) + char_hist + set_alphabet without build: run, export_words,
    dump_pairs and scan_once fail and say why; A's words and pairs are not handed out as B's."""
    a = _cases.zipf().text(20_000)
    b = b"\n".join(synth.stress_text(k, 200, train=True) for k in range(10))
    ctx = LG.Ctx(L)
    try:
        rules, vocab = abi_train(ctx, a, 200)
        assert rules == oracle_rules(oracle, a, vocab)
        dl, nd = C.c_uint64(0), C.c_uint64(0)
        assert L.yttm_train_load_corpus(ctx.h, C.cast(C.c_char_p(b), C.c_void_p), len(b), 0) == 0, ctx.err()
        assert L.yttm_train_char_hist(ctx.h, C.byref(dl), C.byref(nd)) == 0, ctx.err()
        set_alphabet(ctx, nd.value)
        rc, rules = ctx.run(5 + nd.value, 50)
        assert rc != 0 and not rules and "has not run" in ctx.err(), (rc, len(rules), ctx.err())
        nw, nt = C.c_uint64(7), C.c_uint64(7)
        assert L.yttm_train_export_words(ctx.h, None, 0, None, None, 0, C.byref(nw), C.byref(nt)) != 0
        assert "has not run" in ctx.err()
        n = C.c_uint64(7)
        keys = np.zeros(16, dtype=np.uint64)
        assert L.yttm_train_dump_pairs(ctx.h, keys.ctypes.data, keys.ctypes.data, 16, C.byref(n)) != 0
        assert "has not run" in ctx.err() and n.value == 0
        ms, ab = C.c_double(0), C.c_uint64(0)
        assert L.yttm_train_scan_once(ctx.h, C.byref(ms), C.byref(ab)) != 0 and "has not run" in ctx.err()
        assert L.yttm_train_build(ctx.h, None) == 0, ctx.err()      # and then B trains as on a fresh context
        rc, rules = ctx.run(5 + nd.value, 200)
        assert rc == 0 and [r[:3] for r in rules] == oracle_rules(oracle, b, 5 + nd.value + 200)
    finally:
        ctx.close()


def abi_abandoned_pipelined_load(L, dev=False):
    """A pipelined host load of A that no char_hist / build consumes, then a device-resident load of B: the histogram,
    the words and the pair table are B's."""
    a = FG.corpus("soup", small=True)
    b = FG.corpus("chunk")
    want, cp2id = FG.expected(b)
    ctx = LG.Ctx(L)
    try:
        with FG.env(YTTM_TRAIN_PIPELINE=1, YTTM_TRAIN_PIPELINE_PIECE_KB=1):
            assert L.yttm_train_load_corpus(ctx.h, C.cast(C.c_char_p(a), C.c_void_p), len(a), 0) == 0, ctx.err()
        got = FG.device_front(L, b, cp2id, off=3, dev=dev, ctx=ctx.h)
        FG.assert_same(got, want, "device-resident corpus after an abandoned pipelined load")
    finally:
        ctx.close()


# ---- (d) bodies: knobs on a kept context ----------------------------------------------------------------------------
def knob_seg_cap(L, oracle, monkeypatch, small=False):
    """YTTM_XQ_SEG_CAP from the default to 8 between two cached trainings: the second reaches the segment overflow ->
    table rebuild -> relaunch path (a geometry knob: the cache builds a context for the new value)."""
    text = synth.readme_corpus(n_lines=100 if small else 600)
    monkeypatch.delenv("YTTM_XQ_SEG_CAP", raising=False)
    check(L, oracle, text, 300)
    roomy = report(L)["loop_launches"]
    monkeypatch.setenv("YTTM_XQ_SEG_CAP", "8")
    check(L, oracle, text, 300)
    assert report(L)["loop_launches"] > roomy >= 1, (roomy, report(L))
    assert held(L) == 1
    monkeypatch.setenv("YTTM_LOOP_THREADS", "64")             # a geometry knob changed on a kept context
    check(L, oracle, text, 300)
    assert held(L) == 1
    monkeypatch.delenv("YTTM_LOOP_THREADS")
    monkeypatch.delenv("YTTM_XQ_SEG_CAP")
    check(L, oracle, text, 300)


# ---- (e) bodies: stage times -----------------------------------------------------------------------------------------
def stage_times_training(L, monkeypatch, small=False):
    """A pipelined training after a plain one on a kept context: char_hist did not run (the histogram is counted per
    piece behind the copy), so the report gives -1 for it, as a fresh context does."""
    text = _cases.dirty_zipf_text(30_000 if small else 300_000)
    monkeypatch.setenv("YTTM_TRAIN_PIPELINE", "0")
    train(L, text, 600)
    plain = report(L)
    assert plain["char_hist_ms"] >= 0 and plain["word_count_ms"] >= 0, plain
    monkeypatch.setenv("YTTM_TRAIN_PIPELINE", "1")
    monkeypatch.setenv("YTTM_TRAIN_PIPELINE_PIECE_KB", "1")
    train(L, text, 600)
    piped = report(L)
    fresh, err = on_new_thread(lambda: (train(L, text, 600), report(L))[1])
    assert err is None, err
    assert fresh["char_hist_ms"] == -1, fresh
    assert piped["char_hist_ms"] == fresh["char_hist_ms"], (piped, fresh)
    assert piped["h2d_ms"] >= 0 and piped["word_count_ms"] >= 0


def _enc_stage(L, h, name):
    return L.yttm_stage_ms(L.yttm_api_device_context(h), name.encode())


def stage_times_encoder(L, oracle):
    """One encoder handle: an ids call after a spans call reports no enc_spans time, a dropout call after a
    deduplicating one no enc_dedup / enc_rep time — the values of a fresh handle."""
    text, vocab, _, sents = _cases.stress_case(4)
    m = tmp_model_path("enc")
    oracle.train(text, m, vocab, 1.0)
    raw, offs = _pack(sents)
    buf = C.cast(C.c_char_p(raw), C.c_void_p)
    cap = len(raw) + 3 * len(sents) + 8
    ids = np.zeros(cap, dtype=np.int32)
    oo = np.zeros(len(sents) + 1, dtype=np.uint64)
    spans = np.zeros(2 * cap, dtype=np.uint64)
    tot = C.c_uint64(0)

    def ids_call(h, dropout):
        assert L.yttm_api_encode_ids_into(h, buf, offs.ctypes.data, len(sents), 0, 0, 0, dropout, ids.ctypes.data, cap,
                                          oo.ctypes.data, C.byref(tot)) == 0, L.yttm_api_last_error(h)

    def spans_call(h):
        assert L.yttm_api_encode_spans_into(h, buf, offs.ctypes.data, len(sents), 0, 0, 0, 0.0, ids.ctypes.data, cap,
                                            oo.ctypes.data, spans.ctypes.data, C.byref(tot)) == 0, L.yttm_api_last_error(h)

    h, f1, f2 = (L.yttm_api_open(m.encode(), 1) for _ in range(3))
    try:
        spans_call(h)
        assert _enc_stage(L, h, "enc_spans") >= 0 and _enc_stage(L, h, "enc_dedup") >= 0
        ids_call(h, 0.0)
        ids_call(f1, 0.0)
        assert _enc_stage(L, f1, "enc_spans") < 0
        assert _enc_stage(L, h, "enc_spans") == _enc_stage(L, f1, "enc_spans"), "stale enc_spans after an ids call"
        assert _enc_stage(L, h, "enc_dedup") >= 0
        ids_call(h, 0.5)
        ids_call(f2, 0.5)
        for st in ("enc_dedup", "enc_rep"):
            assert _enc_stage(L, f2, st) < 0
            assert _enc_stage(L, h, st) == _enc_stage(L, f2, st), "stale %s after a dropout call" % st
        assert _enc_stage(L, h, "enc_words") >= 0
    finally:
        for x in (h, f1, f2):
            L.yttm_api_close(x)


# ---- GPU tests ------------------------------------------------------------------------------------------------------
def test_kept_context_corpus_sizes(kept, oracle):
    seq_sizes(kept, oracle)


def test_kept_context_alphabets(kept, oracle):
    seq_alphabets(kept, oracle)


def test_kept_context_special_ids(kept, oracle):
    seq_special_ids(kept, oracle)


def test_kept_context_resident_streaming(kept, oracle, monkeypatch):
    seq_resident_streaming(kept, oracle, monkeypatch)


def test_kept_context_pair_table_growth(kept, oracle, monkeypatch):
    seq_pair_table_growth(kept, oracle, monkeypatch)


def test_kept_context_compaction(kept, oracle):
    seq_compaction(kept, oracle)


def test_kept_context_pipelined_and_plain(kept, oracle, monkeypatch):
    seq_pipelined(kept, oracle, monkeypatch)


def test_error_after_pipelined_load_releases(lib, oracle, monkeypatch):
    error_after_pipelined_load(lib, oracle, monkeypatch)


def test_error_on_exiting_thread_releases(lib, monkeypatch):
    monkeypatch.delenv(KEEP, raising=False)
    error_on_exiting_thread(lib)


def test_abi_two_corpora_on_one_context(lib, oracle):
    abi_two_corpora(lib, oracle)


def test_abi_import_twice_on_one_context(lib, oracle):
    abi_import_twice(lib, oracle)


def test_abi_calls_before_build_fail(lib, oracle):
    abi_calls_before_build(lib, oracle)


def test_abi_device_load_after_abandoned_pipelined_load(lib):
    abi_abandoned_pipelined_load(lib, dev=True)


def test_kept_context_seg_cap_and_geometry(kept, oracle, monkeypatch):
    knob_seg_cap(kept, oracle, monkeypatch)


def test_kept_context_stage_times(kept, monkeypatch):
    stage_times_training(kept, monkeypatch)


def test_encoder_handle_stage_times(lib, oracle):
    stage_times_encoder(lib, oracle)


# ---- (f) across the 20-bit stamp wrap ---------------------------------------------------------------------------------
def test_merge_loop_across_the_stamp_wrap(lib, oracle, monkeypatch):
    """One context: import_words(W) + run(first, M) again and again, until the exchange round counter has passed
    0xfffff (where the stamps of the exchange entries start over) by more than one full run; one of the runs that
    cross it is a forced STREAMING run.  W: 60 000 words x 8 tokens (RESIDENT), M = 20 000 merges.  Every run gives
    the rules of the first, and the first those of the oracle.
    Measured on an H100 80GB HBM3 (700 W power limit): 54 runs, 1 080 000 rounds, 9.5 - 10.2 s inside yttm_train_run
    (about 9 us per merge), 10 - 10.5 s for the whole loop; the test prints the figures of each run."""
    ctx = LG.Ctx(lib)
    try:
        w = ctx.synth(60_000, 8, 300, 6, seed=3)
        first, M = 4 + 64 + 300, 20_000
        want = oracle.train_words(w.tok, w.off, w.frq, first, M)
        assert len(want) == M
        t0 = time.perf_counter()
        rc, r0 = ctx.run(first, M)
        assert rc == 0 and r0 == want, ctx.err()
        per_run = int(ctx.stage("xq_round"))
        assert per_run > 0
        runs, streamed, loop_s = 1, False, 0.0
        while True:
            before = int(ctx.stage("xq_round"))
            if before >= STAMP_MOD + per_run:
                break
            stream = not streamed and before + per_run >= STAMP_MOD   # this run crosses the wrap
            if stream:
                monkeypatch.setenv("YTTM_FORCE_STREAM", "1")
            ctx.import_words(w)
            t = time.perf_counter()
            rc, r = ctx.run(first, M)
            loop_s += time.perf_counter() - t
            if stream:
                monkeypatch.delenv("YTTM_FORCE_STREAM")
                assert ctx.stage("loop_resident") == 0
                streamed = True
            after = int(ctx.stage("xq_round"))
            assert rc == 0, ctx.err()
            assert r == r0, "run %d (rounds %d..%d%s) differs from the first" % (runs, before, after,
                                                                                  ", STREAMING" if stream else "")
            runs += 1
        total = int(ctx.stage("xq_round"))
        assert streamed and total >= STAMP_MOD + per_run
        print("stamp wrap: %d runs, %d rounds, %.1f s in yttm_train_run, %.1f s in all" %
              (runs, total, loop_s, time.perf_counter() - t0))
    finally:
        ctx.close()

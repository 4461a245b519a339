"""The product's CUDA kernels — the very sources of youtokentome_b200/csrc, compiled by g++ against the stand-in
cuda_runtime.h of tests/emul/simt — run on the CPU under a fiber SIMT emulator and go through the SAME parity
checks as the GPU tests (the bodies of tests/test_train_gpu.py / tests/test_encode_gpu.py are reused as they are).

TEST HARNESS ONLY.  The emulated library is reachable from tests/ alone (tests/_emu.py); the package loads
libyttm_b200.so and nothing else, and the GPU tests stay the parity tests proper.  What this buys in a container
without a GPU: every kernel's control flow (tile rings and mbarrier phases of the STREAMING merge loop, claim
bitmaps, vectorised hit scans, update queues, cooperative grid barriers, the slot scheme of the encoder) is executed
and compared bit for bit with the oracle by `pytest -m "not gpu"`; it cannot see memory-ordering races or speed."""
import numpy as np
import pytest

import _cases
import test_encode_gpu as EG
import test_encode_words_gpu as WG
import test_train_gpu as TG
from _bind import tmp_model_path
from youtokentome_b200 import _lib, synth


@pytest.fixture
def emu(monkeypatch):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)  # what _lib.lib() hands to tests/_gpu.py and to the Python BPE class
    monkeypatch.setenv("YT_EMU_SMS", "2")
    monkeypatch.setattr(WG, "_cache", {})   # the shared bodies keep encoders: they belong to the library that made them
    return L


# ---- hot path (a): training ---------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(16))
def test_train_stress(emu, oracle, seed):
    TG.test_stress(emu, oracle, seed)


@pytest.mark.parametrize("sms", ["1", "3", "5"])
def test_train_other_grid_sizes(emu, oracle, monkeypatch, sms):
    """1, 3 and 5 blocks: tile ownership, table partitions, exchange rows and the front's gather all change shape, in
    RESIDENT and in STREAMING mode."""
    monkeypatch.setenv("YT_EMU_SMS", sms)
    for seed in (1, 3, 4, 9):
        text, vocab, cov, _ = _cases.stress_case(seed)
        TG._same(oracle, text, vocab, cov)
    TG._same(oracle, _cases.dirty_zipf_text(60_000), 700, 0.98)
    monkeypatch.setenv("YTTM_FORCE_STREAM", "1")
    monkeypatch.setenv("YTTM_STREAM_Q", "128")
    text, vocab, cov, _ = _cases.stress_case(5)
    TG._same(oracle, text, vocab, cov)


@pytest.mark.parametrize("top,sms", [("1", "4"), ("2", "3"), ("6", "2")])
def test_train_front_refresh(emu, oracle, monkeypatch, top, sms):
    """The replicated front: with one or two pairs per partition the front is exhausted every few merges (refresh,
    bound, new pairs below / above the bound), with 6 it fills up from the new pairs instead."""
    monkeypatch.setenv("YTTM_FRONT_TOP", top)
    monkeypatch.setenv("YT_EMU_SMS", sms)
    for seed in (2, 7):
        text, vocab, cov, _ = _cases.stress_case(seed)
        TG._same(oracle, text, vocab, cov)
    TG._same(oracle, _cases.dirty_zipf_text(50_000), 600, 0.98)
    TG._same(oracle, synth.readme_corpus(n_lines=200), 250)


@pytest.mark.parametrize("limit", ["1", "3"])
def test_train_new_pairs_beyond_the_table(emu, oracle, monkeypatch, limit):
    """More new pairs in a round than the per-round table takes: the rest is only bounded (hash-bucket sums raise the
    bound of the front) — the front must refresh early enough to stay exact."""
    monkeypatch.setenv("YTTM_NEWP_LIMIT", limit)
    monkeypatch.setenv("YT_EMU_SMS", "3")
    for seed in (3, 8):
        text, vocab, cov, _ = _cases.stress_case(seed)
        TG._same(oracle, text, vocab, cov)
    TG._same(oracle, _cases.dirty_zipf_text(50_000), 600, 0.98)


@pytest.mark.parametrize("piece_kb", ["1", "7"])
def test_train_pipelined_ingest(emu, oracle, monkeypatch, piece_kb):
    """The corpus copied in pieces that end behind an ASCII space / newline, histogram + word table per piece: multi-byte
    characters, U+2581, invalid bytes and words at the piece ends; a text without any space (one piece); the
    phase-by-phase device ABI."""
    monkeypatch.setenv("YTTM_TRAIN_PIPELINE", "1")
    monkeypatch.setenv("YTTM_TRAIN_PIPELINE_PIECE_KB", piece_kb)
    TG._same(oracle, _cases.dirty_zipf_text(60_000), 700, 0.98)
    TG._same(oracle, _cases.dirty_zipf_text(70_001), 600, 0.98)
    for seed in (0, 4, 5, 11):
        text, vocab, cov, _ = _cases.stress_case(seed)
        TG._same(oracle, text, vocab, cov)
    TG._same(oracle, synth.readme_corpus(n_lines=200), 250)
    TG._same(oracle, b"ab" * 3000 + "\u2581x\u2581".encode() + b"cd" * 2000, 30)
    text = _cases.zipf().text(33_333)
    rules, _, _ = _abi_train(emu, text, 500)
    assert rules == _oracle_rules(oracle, text, 500)


@pytest.mark.parametrize("places", ["1", "2"])
def test_train_drain_places(emu, oracle, monkeypatch, places):
    """Multi-GPU geometry of the drain: only the first place(s) of a segment are handled by per-thread items, the rest
    (place matrix, then the sender's segment) by the shared walk."""
    monkeypatch.setenv("YTTM_DRAIN_PLACES", places)
    monkeypatch.setenv("YT_EMU_SMS", "3")
    for seed in (1, 6):
        text, vocab, cov, _ = _cases.stress_case(seed)
        TG._same(oracle, text, vocab, cov)
    TG._same(oracle, _cases.dirty_zipf_text(50_000), 600, 0.98)


def test_train_unicode_and_runs(emu, oracle):
    TG._same(oracle, _cases.dirty_zipf_text(120_000), 900, 0.98)
    TG._same(oracle, b"a" * 500 + b" " + b"ab" * 300 + b" aaa aaaa aaaaa " + b"b" * 1001, 40)
    TG._same(oracle, synth.readme_corpus(n_lines=300), 300)


@pytest.mark.parametrize("q", ["64", "1000"])
def test_train_streaming_tiles(emu, oracle, monkeypatch, q):
    """STREAMING mode forced: TMA ring model (mbarrier phases persisting across merges), eight-tokens-per-lane
    scan over 16-byte aligned windows, deferred rewrites, tiles cut inside words' neighbourhoods."""
    monkeypatch.setenv("YTTM_FORCE_STREAM", "1")
    monkeypatch.setenv("YTTM_STREAM_Q", q)
    for seed in range(6):
        text, vocab, cov, _ = _cases.stress_case(seed)
        TG._same(oracle, text, vocab, cov)
    TG._same(oracle, _cases.dirty_zipf_text(60_000), 600, 0.98)
    TG._same(oracle, b"a" * 500 + b" " + b"ab" * 300 + b" aaa aaaa aaaaa " + b"b" * 1001, 40)


@pytest.mark.parametrize("stages", ["3", "4"])
def test_train_streaming_deeper_rings(emu, oracle, monkeypatch, stages):
    monkeypatch.setenv("YTTM_FORCE_STREAM", "1")
    monkeypatch.setenv("YTTM_STREAM_Q", "128")
    monkeypatch.setenv("YTTM_STAGES", stages)
    for seed in (2, 5):
        text, vocab, cov, _ = _cases.stress_case(seed)
        TG._same(oracle, text, vocab, cov)


def test_train_words_of_33_plus_tokens(emu, oracle):
    rng = np.random.default_rng(9)
    words = [bytes(rng.choice(list(b"abcd"), size=int(n)).tolist()) for n in rng.integers(1, 90, size=400)]
    TG._same(oracle, b" ".join(words), 200)


def test_train_errors_and_special_ids(emu, oracle):
    TG._same(oracle, b"abc abd", 5)                      # vocab too small: same Status text
    TG._same(oracle, _cases.dirty_zipf_text(40_000), 500, 1.0, pad=-1, bos=-1, eos=5, unk=0)


# ---- hot path (b): encoding ---------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(10))
def test_encode_stress(emu, oracle, seed):
    EG.test_stress(emu, oracle, seed)


@pytest.mark.parametrize("name", sorted(synth.GOLDEN_TEXTS))
def test_encode_manual_corpora(emu, oracle, name):
    EG.test_manual_corpora(emu, oracle, name)


def test_encode_unicode_long_words_dropout(emu, oracle):
    """Multi-script words, invalid bytes, words longer than the thread-local arrays (LOCAL_W) and than 512 slots, and
    more than 3 x 512 words in one batch; with and without dropout."""
    m = EG._model(oracle, _cases.dirty_zipf_text(), 1500, 0.95)
    zc = _cases.zipf()
    long_word = b"".join(zc.sentences(20, 60, seed=6)).replace(b" ", b"")  # > LOCAL_W: works in its global slots
    sents = (_cases.zipf_sentences(400) + _cases.EDGE_SENTENCES +
             [long_word, b"a" * 700, long_word + b" x " + long_word, b"\x80\x80\x80 \xbf\xbf"])
    assert sum(len(s.split()) for s in sents) > 3 * 512
    g, o = EG.GpuEncoder(m), oracle.encoder(m)
    for kw in EG.KW:
        assert g.encode(sents, **kw) == o.encode(sents, **kw)
    for p, seed in ((0.1, 3), (0.3, 9), (0.6, 4), (1.0, 5)):
        assert g.encode(sents, dropout=p, seed=seed) == o.encode(sents, dropout=p, seed=seed)


@pytest.mark.parametrize("special", [dict(), dict(pad=-1, bos=-1, eos=7, unk=0), dict(pad=3, unk=40, bos=41, eos=1000)])
def test_encode_special_id_layouts(emu, oracle, special):
    """Special ids below, between and above the ids of the characters and rules (the product of rule k is the k-th
    free id): with and without dropout."""
    WG.check_special_id_layouts(oracle, special)


def test_encode_rule_products_are_read_from_the_model(emu, oracle, tmp_path):
    """A model whose rule products are NOT the k-th free id (two product ids swapped by hand): the encoder takes the
    id a rule produces from the model, never from the rule's rank."""
    WG.check_rule_products_are_read_from_the_model(oracle, tmp_path)


def test_encode_chunked_pipeline(emu, oracle, monkeypatch):
    m = EG._model(oracle, _cases.dirty_zipf_text(), 1500)
    zc = _cases.zipf()
    sents = zc.sentences(3000, 400, seed=21) + _cases.EDGE_SENTENCES + zc.sentences(3000, 400, seed=22) + zc.sentences(3000, 400, seed=23)
    want = oracle.encoder(m).encode(sents, bos=True, eos=True)
    monkeypatch.setenv("YTTM_ENC_CHUNK_MB", "1")   # 3.6 MB of sentences: at least three chunks, both buffer sets reused
    g = EG.GpuEncoder(m)
    assert g.encode(sents, bos=True, eos=True) == want
    # (the previous version used 1.2 MB: the "no tiny tail chunk" rule folded it into ONE chunk)
    assert emu.yttm_stage_ms(emu.yttm_api_device_context(g.h), b"enc_chunks") >= 3
    assert g.encode(sents, dropout=0.2, seed=77) == oracle.encoder(m).encode(sents, dropout=0.2, seed=77)


def test_python_api_on_the_emulated_library(emu, tmp_path):
    EG.test_python_api_roundtrip(emu, tmp_path)


# ---- rare paths of the merge loop, reached through host-only test knobs ---------------------------
def _abi_train(L, text, vocab):
    """Drive the device ABI of include/yttm_b200.h phase by phase (as tools/probe_train.py does); returns
    (rules as a list of tuples, number of merge-loop launches)."""
    import ctypes as C
    ctx = C.c_void_p()
    assert L.yttm_ctx_create(0, C.byref(ctx)) == 0
    try:
        dl, nd = C.c_uint64(0), C.c_uint64(0)
        assert L.yttm_train_load_corpus(ctx, C.cast(C.c_char_p(text), C.c_void_p), len(text), 0) == 0
        assert L.yttm_train_char_hist(ctx, C.byref(dl), C.byref(nd)) == 0
        cps = np.zeros(nd.value, dtype=np.uint32)
        cnt = np.zeros(nd.value, dtype=np.uint64)
        L.yttm_train_get_char_hist(ctx, cps.ctypes.data, cnt.ctypes.data)
        order = np.lexsort((cps, cnt))[::-1]
        kc = np.concatenate([[9601], cps[order]]).astype(np.uint32)
        ki = np.arange(4, 4 + len(kc), dtype=np.uint32)
        assert L.yttm_train_set_alphabet(ctx, kc.ctypes.data, ki.ctypes.data, len(kc), 4) == 0
        st = _lib.TrainStats()
        assert L.yttm_train_build(ctx, C.byref(st)) == 0, L.yttm_last_error(ctx)
        nm = vocab - 4 - len(kc)
        rules = np.zeros(3 * nm, dtype=np.uint32)
        fr = np.zeros(nm, dtype=np.uint64)
        done = C.c_uint32(0)
        assert L.yttm_train_run(ctx, 4 + len(kc), nm, rules.ctypes.data, fr.ctypes.data, C.byref(done)) == 0, \
            L.yttm_last_error(ctx)
        launches = int(L.yttm_stage_ms(ctx, b"loop_launches"))
        return [tuple(r) for r in rules[:3 * done.value].reshape(-1, 3).tolist()], launches, st
    finally:
        L.yttm_ctx_destroy(ctx)


def _oracle_rules(oracle, text, vocab):
    from _bind import read_model
    m = tmp_model_path("orc")
    oracle.train(text, m, vocab, 1.0)
    return read_model(m)[1]


def test_train_table_rebuilds_on_a_tiny_pair_table(emu, oracle, monkeypatch):
    """YTTM_PAIR_CAP_FLOOR=16: the table starts at load 3/8 of a few dozen slots, so the loop stops again and
    again for a rebuild (stop = 2 / probe overflow) — the relaunch path, with the tokens as the only truth."""
    monkeypatch.setenv("YTTM_PAIR_CAP_FLOOR", "16")
    monkeypatch.setenv("YTTM_PAIR_MAX_LOAD_PCT", "70")   # accept at 35 %, leave at 70 %: the 4096-slot table is rebuilt on the way
    text = _cases.zipf().text(20_000)
    rules, launches, _ = _abi_train(emu, text, 700)
    assert launches >= 2
    assert rules == _oracle_rules(oracle, text, 700)


def test_train_compaction_of_dead_slots(emu, oracle):
    """> 65 536 token slots and enough merges to tombstone a quarter of them: the loop stops with stop = 3, the host
    compacts the packed words (compact_len / scan / compact_copy) and relaunches on the other buffer."""
    text = synth.readme_corpus(n_lines=1300, n_chars=100, seed=5)
    rules, launches, st = _abi_train(emu, text, 260)
    assert st.n_tokens > 65536 and launches >= 2
    assert rules == _oracle_rules(oracle, text, 260)


def test_train_deferred_list_overflow_falls_back_to_the_direct_pass(emu, oracle, monkeypatch):
    monkeypatch.setenv("YTTM_FORCE_STREAM", "1")
    monkeypatch.setenv("YTTM_STREAM_Q", "128")
    monkeypatch.setenv("YTTM_DEFER_CAP", "1")
    for seed in (0, 3):
        text, vocab, cov, _ = _cases.stress_case(seed)
        TG._same(oracle, text, vocab, cov)
    TG._same(oracle, synth.readme_corpus(n_lines=120), 150)


def test_encode_long_words_merged_by_a_block(emu, oracle):
    """Words of more than 512 slots get a whole block and are merged pass by pass (all occurrences of the minimum rule
    per pass) instead of one merge at a time by one thread (dropout = 0: the dedup path hands its long representatives
    to encode_long_words_kernel)."""
    rng = np.random.default_rng(3)
    train = synth.readme_corpus(n_lines=400) + b" " + _cases.dirty_zipf_text(60_000)
    m = EG._model(oracle, train, 700)
    rnd = lambda n, alpha=b"abcd": bytes(rng.choice(list(alpha), size=n).tolist())
    zc = _cases.zipf()
    glued = b"".join(zc.sentences(60, 80, seed=6)).replace(b" ", b"")       # ~4 KB multi-script word
    sents = [rnd(600), rnd(5000), b"a" * 513, b"a" * 4001, b"ab" * 700, b"aab" * 400, rnd(3000, b"ab"),
             glued, glued[:700] + b"\xff\xfe" + glued[700:1500] + "☃☃☃".encode() * 30 + rnd(900),
             b"x " + rnd(2000) + b" y " + rnd(513) + b" " + rnd(512) + b" " + rnd(511) + b" z",
             b"\xff" * 600, b"\xf0\x9f\x98\x80" * 200 + b"abab" * 200] + _cases.zipf_sentences(50) + _cases.EDGE_SENTENCES
    g, o = EG.GpuEncoder(m), oracle.encoder(m)
    for kw in EG.KW:
        assert g.encode(sents, **kw) == o.encode(sents, **kw)
    # with dropout the words stay on the sequential path (the per-event draws are order dependent)
    assert g.encode(sents[:4], dropout=0.3, seed=5) == o.encode(sents[:4], dropout=0.3, seed=5)
    # a model made of x x rules ((a,a), (aa,aa), ...): runs take every second occurrence from the run's start
    runs = b" ".join(b"a" * int(k) + b" " + b"b" * int(j) + b"ab" * int(k % 5) for k, j in rng.integers(1, 40, (300, 2)))
    m2 = EG._model(oracle, runs, 40)
    sents2 = [b"a" * k for k in (513, 514, 515, 1023, 1024, 1025, 2047, 4096, 7001)] + [b"b" * 999 + b"a" * 1000, b"ab" * 600 + b"a" * 777,
              b"a" * 300 + b"b" + b"a" * 300, b"a" * 512 + b" " + b"a" * 600]
    g2, o2 = EG.GpuEncoder(m2), oracle.encoder(m2)
    assert g2.encode(sents2) == o2.encode(sents2)
    assert g2.encode(sents2, bos=True, eos=True, reverse=True) == o2.encode(sents2, bos=True, eos=True, reverse=True)


@pytest.mark.parametrize("knobs", [dict(), dict(YTTM_ENC_DEDUP_SLOTS="4"), dict(YTTM_ENC_DEDUP_WEAKTAG="1"),
                                   dict(YTTM_ENC_DEDUP_SLOTS="64", YTTM_ENC_DEDUP_WEAKTAG="1")])
def test_encode_word_dedup(emu, oracle, monkeypatch, knobs):
    """The word-dedup path (dropout = 0): every distinct word of the batch is encoded once, the other occurrences
    copy the ids of their representative.  Same ids as the oracle, including words that differ only in
    what follows them (end of sentence / space / U+2581), prefixes of each other, truncated UTF-8, repeated long words
    (> LOCAL_W, merged in global slots); a 4-slot table (nearly every word represents itself), equal tags (every
    probe ends in the byte compare) and both."""
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    m = EG._model(oracle, _cases.dirty_zipf_text(), 1500, 0.95)
    zc = _cases.zipf()
    long_word = b"".join(zc.sentences(20, 60, seed=6)).replace(b" ", b"")
    edge = [b"ab\xe2\x96", b"ab\xe2\x96 x", b"ab\xe2\x96\x81x ab", b"ab\xe2", b"ab\xe2 ab\xe2\x96 ab", b"x ab\xf0\x9f\x98",
            b"ab\xf0\x9f\x98 ab\xf0\x9f\x98\x80 ab\xf0\x9f\x98", b"abc abcd ab a abcd abc ab a", b"\xe2\x96\x81ab\xe2\x96\x81ab\xe2\x96",
            b"\xe2\x96 \xe2\x96", b"\x96 \x96\x81 \x96", b"", b" ", b"\xff\xff \xff \xff\xff", b"\x80 \x80 \xbf",
            long_word + b" " + long_word + b"x " + long_word, long_word[:41] + b" " + long_word[:40] + b" " + long_word[:41],
            "☃ ☃☃ ☃ zz☃ zz☃".encode(), b"a" * 700 + b" " + b"a" * 700 + b" " + b"a" * 699,
            long_word * 3 + b" q " + long_word * 3 + b" " + long_word * 3 + b"q"]   # > 512 slots: block-per-word representatives
    # (a 4- or 64-slot table makes every probe a long walk: those variants get a fifth of the filler sentences, the
    # emulator would spend minutes in them otherwise; the edge cases are the same)
    n1, n2 = (400, 100) if "YTTM_ENC_DEDUP_SLOTS" not in knobs else (80, 20)
    sents = _cases.zipf_sentences(n1) + _cases.EDGE_SENTENCES + edge + _cases.zipf_sentences(n2) + edge[::-1]
    g, o = EG.GpuEncoder(m), oracle.encoder(m)
    for kw in EG.KW:
        assert g.encode(sents, **kw) == o.encode(sents, **kw)
    # with dropout every occurrence draws for itself: the per-word kernel runs
    assert g.encode(sents[:200], dropout=0.3, seed=5) == o.encode(sents[:200], dropout=0.3, seed=5)
    monkeypatch.setenv("YTTM_ENC_CHUNK_MB", "1")  # representatives never cross a chunk of the host-buffer pipeline
    if n1 == 400:   # (2 MB through a 4-slot table would take the emulator minutes; the chunking does not depend on the table)
        big = sents * 40
        assert sum(map(len, big)) > 2 << 20
        assert g.encode(big, eos=True) == o.encode(big, eos=True)


def test_encode_word_finder_edges_and_misaligned_base(emu, oracle):
    """The word-start kernel gives a lane four bytes (one aligned 32-bit load) and decides on a register window.
    Sentence starts at every alignment, sentences shorter / equal / longer than the flag cache and than 255 / 256 / 257
    bytes, U+2581 and stray bytes at the sentence bounds, and a batch whose base address is not 4-byte aligned
    (yttm_enc_run_device on an offset pointer)."""
    import ctypes as C
    m = EG._model(oracle, _cases.dirty_zipf_text(), 1500)
    zc = _cases.zipf()
    sp = b"\xe2\x96\x81"
    edge = [sp, sp + sp, sp + b"a", b"a" + sp, b"a" + sp + b"b", sp[:2], sp[:1], sp[1:], sp[2:] + b"a", b"a" + sp[:2], b"ab " + sp[:2] + b" " + sp[1:],
            b"\x81a \x81", b"\x96\x81 a", b"a\xe2", b"\xe2 \x96 \x81", b"a" * 127 + b" b", b"a" * 128 + b" b", b"a " * 64, b" a" * 64 + b" ",
            b"x" * 125 + sp + b"y", b"x" * 126 + sp + b"y", b"x" * 127 + sp + b"y", b"x" * 128 + sp + b"y", b"", b" ", b"\t\n", b"a",
            # U+2581 split over a sentence boundary must not be seen as one: neither side's neighbour bytes count
            b"a\xe2\x96", b"\x81b c", b"a\xe2", b"\x96\x81b c", b"ab\xe2\x96", b"\x81", b"q", b"\x96\x81", b"zz " + sp[:2], sp[2:] + sp + b"k"]
    sents = (_cases.zipf_sentences(200) + _cases.EDGE_SENTENCES + edge + zc.sentences(12, 1023, seed=2) + zc.sentences(12, 1025, seed=3) +
             [b" ".join(zc.sentences(40, 100, seed=5)), b"x" * 1024, b"x " * 700, b" " * 1100 + b"y", b"z" * 31 + b" " + b"w" * 1300] + edge[::-1] +
             zc.sentences(40, 255, seed=2) + zc.sentences(40, 257, seed=3) +
             [b" ".join(zc.sentences(30, 100, seed=5)), b"x" * 256, b"x " * 128, b" " * 300 + b"y", b"z" * 31 + b" " + b"w" * 300])
    g, o = EG.GpuEncoder(m), oracle.encoder(m)
    for kw in EG.KW:
        assert g.encode(sents, **kw) == o.encode(sents, **kw)
    assert g.encode(sents, dropout=0.4, seed=11) == o.encode(sents, dropout=0.4, seed=11)
    # misaligned batch base: the same bytes at offsets 1, 2, 3 of an aligned buffer
    import _bind
    buf, offs = _bind._pack(sents)
    want = o.encode(sents)
    ctx, enc = emu.yttm_api_device_context(g.h), emu.yttm_api_device_encoder(g.h)
    for shift in (1, 2, 3):
        raw = np.zeros(len(buf) + 16, dtype=np.uint8)
        base = raw.ctypes.data + (-raw.ctypes.data) % 4 + shift
        C.memmove(base, bytes(buf), len(buf))
        p_ids, p_off, n = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
        rc = emu.yttm_enc_run_device(enc, base, offs.ctypes.data, len(buf), len(sents), 0, 0, 0, 0.0, 0, 0,
                                     C.byref(p_ids), C.byref(p_off), C.byref(n))
        assert rc == 0, emu.yttm_last_error(ctx)
        ids = np.ctypeslib.as_array(C.cast(p_ids, C.POINTER(C.c_int32)), shape=(n.value,)).copy()
        oo = np.ctypeslib.as_array(C.cast(p_off, C.POINTER(C.c_uint64)), shape=(len(sents) + 1,)).copy()
        assert _bind._unpack(ids, oo) == want, shift


@pytest.mark.parametrize("floor,seg", [(None, None), ("16", "4"), (None, "16"), ("64", None)])
def test_train_exchange_segments(emu, oracle, monkeypatch, floor, seg):
    """The owner-computes merge loop (round 2): count changes travel through per-block exchange segments and are applied
    by the block that owns the key's table partition.  YTTM_XQ_SEG_CAP = 4 / 16 entries makes segments overflow on almost
    every early merge (the merge is still applied to the words and the table is rebuilt from them); pair-table floors of
    16 / 64 slots keep the partitions tiny (16 slots each), so that they fill up, the loop leaves for a larger table and
    probe chains wrap around the end of a partition.  Same rules as the oracle on stress seeds, dirty Unicode, runs,
    RESIDENT and STREAMING tiles."""
    if seg:
        monkeypatch.setenv("YTTM_XQ_SEG_CAP", seg)
    if floor:
        monkeypatch.setenv("YTTM_PAIR_CAP_FLOOR", floor)
    for seed in range(8):
        text, vocab, cov, _ = _cases.stress_case(seed)
        TG._same(oracle, text, vocab, cov)
    TG._same(oracle, _cases.dirty_zipf_text(60_000), 700, 0.98)
    TG._same(oracle, b"a" * 500 + b" " + b"ab" * 300 + b" aaa aaaa aaaaa " + b"b" * 1001, 40)
    text = _cases.zipf().text(20_000)
    rules, launches, _ = _abi_train(emu, text, 700)
    assert launches >= 2 or not seg
    assert rules == _oracle_rules(oracle, text, 700)
    monkeypatch.setenv("YTTM_FORCE_STREAM", "1")
    monkeypatch.setenv("YTTM_STREAM_Q", "128")
    for seed in (1, 5):
        text, vocab, cov, _ = _cases.stress_case(seed)
        TG._same(oracle, text, vocab, cov)
    monkeypatch.setenv("YT_EMU_SMS", "5")
    TG._same(oracle, _cases.dirty_zipf_text(40_000), 500, 0.98)


@pytest.mark.parametrize("pct", ["30", "50", "90"])
def test_train_pair_table_load_knob(emu, oracle, monkeypatch, pct):
    """YTTM_PAIR_MAX_LOAD_PCT (A/B knob, default 50): the load factor at which the loop leaves for a rebuild (a rebuilt
    table is accepted at half of it) changes table sizes and rebuild points, never the rules."""
    monkeypatch.setenv("YTTM_PAIR_MAX_LOAD_PCT", pct)
    monkeypatch.setenv("YTTM_PAIR_CAP_FLOOR", "32")
    for seed in (0, 2, 6):
        text, vocab, cov, _ = _cases.stress_case(seed)
        TG._same(oracle, text, vocab, cov)
    text = _cases.zipf().text(20_000)
    rules, launches, _ = _abi_train(emu, text, 700)
    assert rules == _oracle_rules(oracle, text, 700)   # (at 30 % the first table is large enough for the whole run)


def test_release_training_cache(emu, oracle):
    """release_training_cache(): a no-op before any training, and a training after it builds a fresh context."""
    emu.yttm_api_release_training_cache()
    text, vocab, cov, _ = _cases.stress_case(2)
    TG._same(oracle, text, vocab, cov)
    emu.yttm_api_release_training_cache()
    emu.yttm_api_release_training_cache()
    TG._same(oracle, text, vocab, cov)


def test_graft_entry_smoke_on_the_emulator(emu, capsys):
    """__graft_entry__.smoke() as the driver calls it on the GPU box, here with the emulated library in place."""
    import __graft_entry__ as ge
    ge.smoke()
    assert "smoke ok" in capsys.readouterr().out


@pytest.mark.parametrize("special", [dict(pad=-1, unk=1, bos=2, eos=3), dict(pad=-1, unk=5, bos=-1, eos=-1)])
def test_encode_space_token_with_id_zero(emu, oracle, special):
    """U+2581 with final id 0 (no special token at 0): the reference drops a never-merged word-initial "▁"
    (bpe.cpp:1591-1596; oracle pinned to it in test_oracle_vs_reference.py).  Default kernels (dedup + long words),
    plain kernels and dropout."""
    EG.check_space_id_zero(oracle, special)


def test_api_pieces_with_u0001(emu, tmp_path):
    EG.check_pieces_with_u0001(tmp_path)


def test_api_shared_handle_between_threads(emu, oracle):
    EG.check_shared_handle_between_threads(oracle)


def test_api_encode_packed_torch_output(emu, oracle):
    import torch
    import youtokentome_b200 as yttm
    m = EG._model(oracle, _cases.dirty_zipf_text(), 1200)
    bpe = yttm.BPE(m)
    sents = _cases.zipf_sentences(200) + list(_cases.EDGE_SENTENCES)
    buf, offs = EG._pack(sents)
    want, woo = oracle.encoder(m).encode_packed(buf, offs, eos=True)
    t_ids, t_oo = bpe.encode_packed(torch.frombuffer(bytearray(buf), dtype=torch.uint8), offs, eos=True, out="torch")
    assert np.array_equal(t_ids.numpy(), want) and np.array_equal(t_oo.numpy(), woo.astype(np.int64))
    ids, oo = bpe.encode_packed(np.frombuffer(buf, dtype=np.uint8), offs, eos=True)
    assert np.array_equal(ids, want) and np.array_equal(oo, woo)


def test_train_edge_inputs(emu, oracle):
    """Empty / all-space / one-letter / invalid-only corpora, vocab too small, merges running out."""
    TG.test_edge_inputs(emu, oracle)

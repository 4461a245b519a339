"""The merge-loop checks of tests/test_train_loop_gpu.py on the CPU under the SIMT emulator, at small sizes and with 1, 2
and 5 SMs; and the words-in oracle itself: against the numpy recount of tests/test_train_scale_gpu.py, and against
the oracle's own text trainer on the words the emulated trainer exports."""
import ctypes as C

import numpy as np
import pytest

import _cases
import test_train_loop_gpu as LG
import test_train_scale_gpu as SG
from _bind import read_model, tmp_model_path
from youtokentome_b200 import _lib


@pytest.fixture(params=["1", "2", "5"])
def emu(monkeypatch, request):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


@pytest.fixture
def emu2(monkeypatch):
    """2 SMs only (the knob cases, which set their own geometry)"""
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", "2")
    return L


@pytest.fixture
def ctx(emu):
    c = LG.Ctx(emu)
    yield c
    c.close()


# ---- the loop on the emulator ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", [30, 200])
def test_streaming(ctx, oracle, monkeypatch, alpha):
    monkeypatch.setenv("YTTM_FORCE_STREAM", "1")
    monkeypatch.setenv("YTTM_STREAM_Q", "128")
    w = ctx.synth(1500, 8, alpha, 0)
    LG.check_run(ctx, oracle, w, 4 + 1 + alpha, 120)
    assert LG.observed(ctx)["loop_resident"] == 0


@pytest.mark.parametrize("cap", ["1", "4"])
def test_streaming_deferred_list_overflow(ctx, oracle, monkeypatch, cap):
    monkeypatch.setenv("YTTM_FORCE_STREAM", "1")
    monkeypatch.setenv("YTTM_STREAM_Q", "128")
    monkeypatch.setenv("YTTM_DEFER_CAP", cap)
    w = ctx.synth(1500, 8, 40, 2, seed=11)
    LG.check_run(ctx, oracle, w, 4 + 4 + 40, 100, want_done=100)


@pytest.mark.parametrize("name", list(LG.KNOBS))
def test_knobs(emu2, oracle, monkeypatch, name):
    c = LG.Ctx(emu2)
    try:
        LG.run_knob(c, oracle, monkeypatch, name, 1500, 150, paths=False)
    finally:
        c.close()


@pytest.mark.parametrize("knob", ["", "YTTM_NEWP_LIMIT=1", "YTTM_FRONT_TOP=1", "YTTM_XQ_SEG_CAP=4"])
def test_counts_above_32_bits(ctx, oracle, monkeypatch, knob):
    LG.test_counts_above_32_bits(ctx, oracle, monkeypatch, knob)


def test_import_rejects_counts_beyond_the_exchange_entry(ctx):
    LG.test_import_rejects_counts_beyond_the_exchange_entry(ctx)


def test_ids_at_the_22_bit_limit(ctx, oracle):
    LG.test_ids_at_the_22_bit_limit(ctx, oracle)


@pytest.mark.parametrize("stream", [False, True])
def test_exact_ties_and_runs(ctx, oracle, monkeypatch, stream):
    LG.test_exact_ties_and_runs(ctx, oracle, monkeypatch, stream)


@pytest.mark.parametrize("stream", [False, True])
def test_long_words(ctx, oracle, monkeypatch, stream):
    if stream:
        monkeypatch.setenv("YTTM_FORCE_STREAM", "1")
        monkeypatch.setenv("YTTM_STREAM_Q", "256")
    w = LG.long_words(np.random.default_rng(9), [200, 1000])
    ctx.import_words(w)
    LG.check_run(ctx, oracle, w, 3000, 100, want_done=100)


@pytest.mark.parametrize("seg", ["", "8"])
def test_run_split_in_two(emu, oracle, monkeypatch, seg):
    if seg:
        monkeypatch.setenv("YTTM_XQ_SEG_CAP", seg)
    rng = np.random.default_rng(21)
    w = LG.Words.of(*LG.hand_words(rng, 1500, [3, 5, 8], np.arange(20, 50), np.arange(1000, 1032)))
    n, first = 120, 2000
    want = oracle.train_words(w.tok, w.off, w.frq, first, n)
    for k in (1, 37, 119):
        c = LG.Ctx(emu)
        try:
            c.import_words(w)
            rc, r1 = c.run(first, k)
            assert rc == 0 and r1 == want[:k], (k, c.err())
            oracle.train_words(w.tok, w.off, w.frq, first, k)
            LG.check_state(c, oracle, "after run(%d)" % k)
            rc, r2 = c.run(first + k, n - k)
            assert rc == 0 and r2 == want[k:], (k, c.err())
            oracle.train_words(w.tok, w.off, w.frq, first, n)
            LG.check_state(c, oracle, "after run(%d) + run(%d)" % (k, n - k))
        finally:
            c.close()


# ---- the words-in oracle --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wl,alpha,n_first,seed", [(8, 30, 1, 1), (6, 12, 8, 2), (12, 5, 2, 3), (3, 50, 1, 4)])
def test_oracle_against_the_numpy_recount(oracle, wl, alpha, n_first, seed):
    """20 merges of the words-in oracle against a full numpy recount per merge: rules and counts, then the words and
    the pair table after those merges."""
    rng = np.random.default_rng(seed)
    n = 3000
    rows = np.empty((n, wl), dtype=np.uint32)
    rows[:, 0] = 4 + np.arange(n) % n_first
    rows[:, 1:] = 4 + n_first + rng.integers(0, alpha, size=(n, wl - 1))
    frq = rng.integers(1, 9, n).astype(np.uint64)
    first = 4 + n_first + alpha
    got = oracle.train_words(rows.ravel(), np.arange(n + 1, dtype=np.uint32) * wl, frq, first, 20)
    want = []
    for m in range(20):
        uk, cnt = SG.np_pair_counts(rows, frq)
        x, y, c = SG.np_best(uk, cnt)
        want.append((x, y, first + m, c))
        rows = SG.np_apply(rows, x, y, first + m)
    assert got == want
    tok, off, ofrq, keys, cnts = oracle.words_state()
    o_rows = [tok[off[i]:off[i + 1]].tolist() for i in range(n)]
    assert o_rows == [[t for t in r if t != LG.DEAD] for r in rows.tolist()]
    assert np.array_equal(ofrq, frq)
    uk, cnt = SG.np_pair_counts(rows, frq)
    live = cnt > 0
    assert np.array_equal(*(LG.sorted_table(keys, cnts)[0], uk[live])) and \
        np.array_equal(LG.sorted_table(keys, cnts)[1], cnt[live])


@pytest.mark.parametrize("corpus", ["zipf", "stress"])
def test_oracle_words_in_equals_the_text_trainer(emu2, oracle, corpus):
    """The words the emulated trainer builds from a text, fed to orc_train_words, give the rules of orc_train_memory on
    that text (with 4 special ids the internal ids are the model's)."""
    from youtokentome_b200 import synth
    text = _cases.zipf().text(30_000) if corpus == "zipf" else b"\n".join(
        synth.stress_text(k, 300, train=True) for k in range(40))
    vocab = 500
    L = emu2
    c = LG.Ctx(L)
    try:
        dl, nd = C.c_uint64(0), C.c_uint64(0)
        assert L.yttm_train_load_corpus(c.h, C.cast(C.c_char_p(text), C.c_void_p), len(text), 0) == 0
        assert L.yttm_train_char_hist(c.h, C.byref(dl), C.byref(nd)) == 0
        cps = np.zeros(nd.value, dtype=np.uint32)
        cnt = np.zeros(nd.value, dtype=np.uint64)
        L.yttm_train_get_char_hist(c.h, cps.ctypes.data, cnt.ctypes.data)
        order = np.lexsort((cps, cnt))[::-1]
        kc = np.concatenate([[9601], cps[order]]).astype(np.uint32)
        ki = np.arange(4, 4 + len(kc), dtype=np.uint32)
        assert L.yttm_train_set_alphabet(c.h, kc.ctypes.data, ki.ctypes.data, len(kc), 4) == 0
        assert L.yttm_train_build(c.h, None) == 0, c.err()
        w = c.export()
    finally:
        c.close()
    m = tmp_model_path("orc")
    oracle.train(text, m, vocab, 1.0)
    want = read_model(m)[1]
    got = oracle.train_words(w.tok, w.off, w.frq, 4 + len(kc), vocab - 4 - len(kc))
    assert [r[:3] for r in got] == want

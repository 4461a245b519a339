"""The merge loop (merge_loop.cuh + yttm_train_run) on the GPU against the words-in oracle (orc_train_words): long
STREAMING runs at 12 M tokens, the rare paths behind the test knobs, counts above 32 bits, token ids at the 22-bit
limit, exact ties, runs, long words and a run split in two.  Every case loads a word set into a fresh context, runs the
loop and checks three things against the oracle on the same words:
  (a) the rules (x, y, z, count at merge time) and the number of merges;
  (b) the words the context holds afterwards (yttm_train_export_words) as a multiset of live tokens -> summed
      frequency, dead slots stripped and words of fewer than 2 tokens dropped;
  (c) the live pair table (yttm_train_dump_pairs) — exactly.
Each case also asserts, through yttm_stage_ms, that it reached the path it is named for."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
DEAD = 0xFFFFFFFF
ID_LIMIT = 1 << 22          # BB_ID_LIMIT: token ids of the merge loop fit 22 bits


# ---- word sets ------------------------------------------------------------------------------------------------------
class Words:
    """A word set: word i = tok[off[i]:off[i+1]], frequency frq[i]."""

    def __init__(self, tok, off, frq):
        self.tok = np.ascontiguousarray(tok, dtype=np.uint32)
        self.off = np.ascontiguousarray(off, dtype=np.uint32)
        self.frq = np.ascontiguousarray(frq, dtype=np.uint64)

    @staticmethod
    def of(words, freqs):
        off = np.zeros(len(words) + 1, dtype=np.uint32)
        off[1:] = np.cumsum([len(w) for w in words])
        tok = np.array([t for w in words for t in w], dtype=np.uint32)
        return Words(tok, off, freqs)

    def check_initial_ids(self):
        """The precondition of yttm_train_import_words: a word's first token appears at no other position."""
        firsts = self.tok[self.off[:-1][np.diff(self.off) > 0]]
        rest = np.ones(len(self.tok), dtype=bool)
        rest[self.off[:-1][np.diff(self.off) > 0]] = False
        assert not np.isin(self.tok[rest], firsts).any(), "a word-initial id appears inside a word"


def hand_words(rng, n_words, lens, alphabet, initials, freq_hi=8):
    """Random words: first token from `initials` (ids used nowhere else), the rest from `alphabet`."""
    words = []
    for _ in range(n_words):
        n = int(rng.choice(lens))
        words.append([int(rng.choice(initials))] + [int(t) for t in rng.choice(alphabet, n - 1)])
    return words, [int(f) for f in rng.integers(1, freq_hi + 1, n_words)]


# ---- the context ----------------------------------------------------------------------------------------------------
class Ctx:
    def __init__(self, L):
        self.L = L
        self.h = C.c_void_p()
        assert L.yttm_ctx_create(0, C.byref(self.h)) == 0, L.yttm_last_error(None)

    def close(self):
        self.L.yttm_ctx_destroy(self.h)

    def err(self):
        e = self.L.yttm_last_error(self.h)
        return e.decode() if isinstance(e, bytes) else str(e)

    def stage(self, name):
        return self.L.yttm_stage_ms(self.h, name.encode())

    def import_words(self, w):
        assert self.L.yttm_train_import_words(self.h, w.tok.ctypes.data, len(w.tok), w.off.ctypes.data,
                                              w.frq.ctypes.data, len(w.frq), None) == 0, self.err()

    def synth(self, n_words, wl, alpha, log2_first, seed=7):
        assert self.L.yttm_train_synth_words(self.h, n_words, wl, alpha | (log2_first << 24), seed) == 0, self.err()
        return self.export()

    def export(self):
        nw, nt = C.c_uint64(0), C.c_uint64(0)
        assert self.L.yttm_train_export_words(self.h, None, 0, None, None, 0, C.byref(nw), C.byref(nt)) == 0
        tok = np.zeros(nt.value + 1, dtype=np.uint32)
        off = np.zeros(nw.value + 1, dtype=np.uint32)
        frq = np.zeros(nw.value + 1, dtype=np.uint64)
        assert self.L.yttm_train_export_words(self.h, tok.ctypes.data, len(tok), off.ctypes.data, frq.ctypes.data,
                                              len(frq), C.byref(nw), C.byref(nt)) == 0, self.err()
        return Words(tok[:nt.value], off, frq[:nw.value])

    def run(self, first_new_id, max_merges):
        """-> (rc, rules [(x, y, z, count)])"""
        rules = np.zeros(3 * max(max_merges, 1), dtype=np.uint32)
        fr = np.zeros(max(max_merges, 1), dtype=np.uint64)
        nd = C.c_uint32(0)
        rc = self.L.yttm_train_run(self.h, first_new_id, max_merges, rules.ctypes.data, fr.ctypes.data, C.byref(nd))
        return rc, [tuple(int(v) for v in rules[3 * i:3 * i + 3]) + (int(fr[i]),) for i in range(nd.value)]

    def pairs(self):
        n = C.c_uint64(0)
        assert self.L.yttm_train_dump_pairs(self.h, None, None, 0, C.byref(n)) == 0, self.err()
        keys = np.zeros(n.value + 1, dtype=np.uint64)
        cnts = np.zeros(n.value + 1, dtype=np.uint64)
        assert self.L.yttm_train_dump_pairs(self.h, keys.ctypes.data, cnts.ctypes.data, len(keys), C.byref(n)) == 0
        return keys[:n.value], cnts[:n.value]


def word_multiset(tok, off, frq):
    """The multiset `live tokens -> summed frequency` (dead slots stripped, words of fewer than 2 live tokens dropped),
    as {length: (the distinct words of that length in sorted order, their summed frequencies)}, all as bytes."""
    tok = np.asarray(tok, dtype=np.uint32)
    off = np.asarray(off, dtype=np.int64)
    frq = np.asarray(frq, dtype=np.uint64)
    live = tok != DEAD
    csum = np.concatenate([[0], np.cumsum(live)])
    lens = csum[off[1:]] - csum[off[:-1]]
    starts = csum[off[:-1]]
    lt = tok[live]
    out = {}
    for n in np.unique(lens):
        if n < 2:
            continue
        sel = np.flatnonzero(lens == n)
        rows = np.ascontiguousarray(lt[starts[sel][:, None] + np.arange(n)])
        u, inv = np.unique(rows.view(np.dtype((np.void, 4 * int(n)))).ravel(), return_inverse=True)
        order = np.argsort(inv, kind="stable")
        cuts = np.concatenate([[0], np.flatnonzero(np.diff(inv[order])) + 1])
        out[int(n)] = (u.tobytes(), np.add.reduceat(frq[sel][order], cuts).astype(np.uint64).tobytes())
    return out


def sorted_table(keys, cnts):
    o = np.argsort(keys, kind="stable")
    return keys[o], cnts[o]


def check_state(ctx, oracle, label=""):
    """(b) the words and (c) the pair table of the context equal the oracle's state after its last train_words."""
    o_tok, o_off, o_frq, o_keys, o_cnts = oracle.words_state()
    got = ctx.export()
    assert word_multiset(got.tok, got.off, got.frq) == word_multiset(o_tok, o_off, o_frq), "words differ " + label
    gk, gc = sorted_table(*ctx.pairs())
    ok, oc = sorted_table(o_keys, o_cnts)
    if not (np.array_equal(gk, ok) and np.array_equal(gc, oc)):
        g, o = dict(zip(gk.tolist(), gc.tolist())), dict(zip(ok.tolist(), oc.tolist()))
        bad = sorted(k for k in set(g) | set(o) if g.get(k) != o.get(k))
        pytest.fail("pair table differs %s at %d keys, e.g. %s" %
                    (label, len(bad), [((k >> 32, k & 0xFFFFFFFF), g.get(k), o.get(k)) for k in bad[:5]]))
    return got


def check_run(ctx, oracle, words, first_new_id, max_merges, want_done=None):
    """Run the loop on the words the context holds (= `words`), compare (a), (b), (c); -> (rules, words after)."""
    rc, got = ctx.run(first_new_id, max_merges)
    assert rc == 0, ctx.err()
    want = oracle.train_words(words.tok, words.off, words.frq, first_new_id, max_merges)
    if want_done is not None:
        assert len(want) == want_done
    assert len(got) == len(want)
    if got != want:
        i = next(i for i in range(len(got)) if got[i] != want[i])
        pytest.fail("rule %d differs: gpu %s, oracle %s" % (i, got[i], want[i]))
    after = check_state(ctx, oracle)
    return got, after


@pytest.fixture
def ctx(product):
    c = Ctx(product)
    yield c
    c.close()


def observed(ctx):
    return {k: ctx.stage(k) for k in ("loop_resident", "loop_launches", "loop_refreshes", "table_capacity")}


# ---- 1. STREAMING by itself at scale --------------------------------------------------------------------------------
@pytest.mark.parametrize("log2_first,alpha,merges", [(0, 300, 2000), (6, 300, 2000), (0, 2000, 600)])
def test_streaming_at_scale(ctx, oracle, log2_first, alpha, merges):
    """1.5 M words x 8 tokens = 12 M tokens: beyond the shared memory of all SMs, STREAMING without forcing.  alpha
    2000: every merge creates more new pairs than the per-round table takes, the sketch decides."""
    w = ctx.synth(1_500_000, 8, alpha, log2_first)
    check_run(ctx, oracle, w, 4 + (1 << log2_first) + alpha, merges, want_done=merges)
    ob = observed(ctx)
    print(log2_first, alpha, ob)
    assert ob["loop_resident"] == 0 and ob["loop_refreshes"] >= 1, ob


# ---- 2. STREAMING compaction ----------------------------------------------------------------------------------------
def test_streaming_compaction(ctx, oracle):
    """4 M words [first, a, b] over 6 symbols (12 M tokens): each of the leading (first, a) merges kills one slot in a
    sixth of all words, so every block passes 25 % dead slots and the loop relaunches for a compaction, still in
    STREAMING mode (first call, 20 merges).  The second call merges the words down to one token; they leave the buffer
    at the next compaction, and the set shrinks until it fits shared memory."""
    w = ctx.synth(4_000_000, 3, 6, 0)
    first = 4 + 1 + 6
    want = oracle.train_words(w.tok, w.off, w.frq, first, 60)
    rc, r1 = ctx.run(first, 20)
    assert rc == 0 and r1 == want[:20], ctx.err()
    ob = observed(ctx)
    print("compaction, first call", ob)
    assert ob["loop_resident"] == 0 and ob["loop_launches"] >= 2, ob
    oracle.train_words(w.tok, w.off, w.frq, first, 20)
    check_state(ctx, oracle, "after 20 merges")
    rc, r2 = ctx.run(first + 20, 40)
    assert rc == 0 and r1 + r2 == want, ctx.err()
    oracle.train_words(w.tok, w.off, w.frq, first, 60)
    after = check_state(ctx, oracle, "after the second call")
    print("compaction, second call", observed(ctx), len(w.frq), len(after.frq))
    assert len(after.frq) < len(w.frq) // 2 and observed(ctx)["loop_launches"] >= 2


# ---- 3. STREAMING with an overflowing deferred list -----------------------------------------------------------------
@pytest.mark.parametrize("cap", ["1", "64"])
def test_streaming_deferred_list_overflow(ctx, oracle, monkeypatch, cap):
    monkeypatch.setenv("YTTM_DEFER_CAP", cap)
    w = ctx.synth(1_500_000, 8, 300, 6, seed=11)
    check_run(ctx, oracle, w, 4 + 64 + 300, 300, want_done=300)
    assert observed(ctx)["loop_resident"] == 0


# ---- 4. RESIDENT knobs ----------------------------------------------------------------------------------------------
KNOBS = {
    "front_top_1": {"YTTM_FRONT_TOP": "1"},
    "newp_limit_1": {"YTTM_NEWP_LIMIT": "1"},
    "seg_cap_8": {"YTTM_XQ_SEG_CAP": "8"},
    "seg_cap_64": {"YTTM_XQ_SEG_CAP": "64"},
    "table_growth": {"YTTM_PAIR_CAP_FLOOR": "16", "YTTM_PAIR_MAX_LOAD_PCT": "70"},
    "threads_64": {"YTTM_LOOP_THREADS": "64"},
    "drain_places_1": {"YTTM_DRAIN_PLACES": "1"},
    "stream_q64_stages3": {"YTTM_FORCE_STREAM": "1", "YTTM_STREAM_Q": "64", "YTTM_STAGES": "3"},
    "stream_q64_stages4": {"YTTM_FORCE_STREAM": "1", "YTTM_STREAM_Q": "64", "YTTM_STAGES": "4"},
}


def run_knob(ctx, oracle, monkeypatch, name, n_words, merges, paths=True):
    """paths: also assert that the knob's path was taken (the word sets of the emulator are too small for some)."""
    for k, v in KNOBS[name].items():
        monkeypatch.setenv(k, v)
    w = ctx.synth(n_words, 8, 4, 1, seed=5)      # 4 symbols: a merge rewrites 1/3 of all words, segments overflow
    cap0 = ctx.stage("table_capacity")
    check_run(ctx, oracle, w, 4 + 2 + 4, merges, want_done=merges)
    ob = observed(ctx)
    print(name, ob)
    stream = "YTTM_FORCE_STREAM" in KNOBS[name]
    assert ob["loop_resident"] == (0 if stream else 1), ob
    if name == "front_top_1" and paths:
        assert ob["loop_refreshes"] * 2 >= merges, ob           # a refresh at least every other merge
    if name.startswith("seg_cap") and paths:
        assert ob["loop_launches"] >= 2, ob                      # overflow -> rebuild -> relaunch
    if name == "table_growth" and paths:
        assert ob["table_capacity"] > cap0 and ob["loop_launches"] >= 2, (cap0, ob)
    return ob


@pytest.mark.parametrize("name", list(KNOBS))
def test_resident_knobs(ctx, oracle, monkeypatch, name):
    """60 000 words x 8 tokens (480 k tokens, RESIDENT), 1 200 merges, one knob at a time."""
    run_knob(ctx, oracle, monkeypatch, name, 60_000, 1200)


# ---- 5. counts above 32 bits ----------------------------------------------------------------------------------------
def big_count_words():
    """Frequencies around 2^31, 2^32 and 2^33.  Initial ids 1000.., symbols 10..; every freq x tokens << 2^43."""
    words, freqs = [], []
    nxt = [1000]

    def add(body, f):
        words.append([nxt[0]] + body)
        freqs.append(f)
        nxt[0] += 1
    add([10, 11], (1 << 31) - 1)                 # (10, 11) just below 2^31 ...
    add([12, 13], (1 << 31) + 1)                 # ... (12, 13) just above
    add([14, 15], (1 << 32) + 9)                 # low 32 bits 9 ...
    add([16, 17], (1 << 33) + 7)                 # ... low 32 bits 7: a 32-bit compare elects (14, 15) first
    add([18, 19], (1 << 32) - 3)                 # just below 2^32
    add([20, 20, 20, 20, 20], (1 << 33) + 5)     # (20, 20) twice in one word: one entry of 2^34 + 10
    add([21, 22, 23], (1 << 33) + 3)             # a single entry above 2^32 for each pair
    for k in range(24):                          # (30, 31) -> z; (z, 32) sums 24 x 2^28 = 6 x 2^30 only over words
        add([30, 31, 32], 1 << 28)
    for k in range(6):
        add([33, 34, 35, 33, 34], (1 << 31) + k)
    return Words.of(words, freqs)


@pytest.mark.parametrize("knob", ["", "YTTM_NEWP_LIMIT=1", "YTTM_FRONT_TOP=1", "YTTM_XQ_SEG_CAP=4"])
def test_counts_above_32_bits(ctx, oracle, monkeypatch, knob):
    if knob:
        monkeypatch.setenv(*knob.split("="))
    w = big_count_words()
    w.check_initial_ids()
    ctx.import_words(w)
    rules, _ = check_run(ctx, oracle, w, 2000, 200)
    counts = [r[3] for r in rules]
    assert max(counts) > 1 << 34 and any((1 << 31) < c < (1 << 32) for c in counts) and any(c > 1 << 32 for c in counts)
    # (16, 17) outranks (14, 15) only above 32 bits
    order = [(r[0], r[1]) for r in rules]
    assert order.index((16, 17)) < order.index((14, 15))


def test_import_rejects_counts_beyond_the_exchange_entry(ctx):
    """An entry carries a signed 44-bit count change: freq x tokens of a word must stay below 2^43."""
    w = Words.of([[1000, 10, 11, 12]], [1 << 42])
    ctx.L.yttm_train_import_words(ctx.h, w.tok.ctypes.data, len(w.tok), w.off.ctypes.data, w.frq.ctypes.data, 1, None)
    assert "2^43" in ctx.err()
    ok = Words.of([[1000, 10, 11, 12]], [(1 << 41) - 1])
    ctx.import_words(ok)


# ---- 6. the 22-bit id edge ------------------------------------------------------------------------------------------
def test_ids_at_the_22_bit_limit(ctx, oracle):
    M = 300
    first = ID_LIMIT - M
    rng = np.random.default_rng(3)
    words, freqs = hand_words(rng, 3000, [3, 5, 8, 12], np.arange(first - 8, first), np.arange(first - 28, first - 8))
    w = Words.of(words, freqs)
    w.check_initial_ids()
    ctx.import_words(w)
    rc, _ = ctx.run(first, M)                                    # first + M == 2^22: refused
    assert rc != 0 and "2^22" in ctx.err()
    rules, _ = check_run(ctx, oracle, w, first, M - 1, want_done=M - 1)   # the context is still usable
    assert rules[-1][2] == ID_LIMIT - 2
    assert max(max(r[0], r[1]) for r in rules) >= first        # merged ids near 2^22 take part again


# ---- 7. order and the run rule --------------------------------------------------------------------------------------
def tie_words():
    words, freqs = [], []
    ini = 5
    sym = list(range(10, 22))
    for a in sym:                                 # every ordered pair of 12 symbols once: all counts 1
        for b in sym:
            if a != b:
                words.append([ini, a, b]); freqs.append(1)
    for k in range(2, 10):                        # a^k: (a, a) = floor(k/2), tied with (a, b)
        a, b = 100 + 2 * k, 101 + 2 * k
        words.append([ini] + [a] * k); freqs.append(1)
        words.append([ini, a, b]); freqs.append(k // 2)
        words.append([ini, b, a]); freqs.append(k // 2)
    return Words.of(words, freqs)


@pytest.mark.parametrize("stream", [False, True])
def test_exact_ties_and_runs(ctx, oracle, monkeypatch, stream):
    if stream:
        monkeypatch.setenv("YTTM_FORCE_STREAM", "1")
        monkeypatch.setenv("YTTM_STREAM_Q", "64")
    w = tie_words()
    w.check_initial_ids()
    ctx.import_words(w)
    check_run(ctx, oracle, w, 500, 400)


def long_words(rng, tile_lens):
    """Words of 31, 32, 33 and 64 tokens, words around a tile's length, and many short words."""
    words, freqs = hand_words(rng, 4000, [2, 3, 5, 8], np.arange(20, 36), np.arange(1000, 1100), freq_hi=5)
    for n in [31, 32, 33, 64] * 8 + tile_lens:
        words.append([int(rng.integers(1100, 1200))] + [int(t) for t in rng.integers(20, 26, n - 1)])
        freqs.append(int(rng.integers(1, 4)))
    return Words.of(words, freqs)


@pytest.mark.parametrize("stream", [False, True])
def test_long_words(ctx, oracle, monkeypatch, stream):
    """A word of more than 32 tokens is rewritten by one lane; in STREAMING a word longer than a pipeline stage (about
    18.6 k tokens at two stages) goes through the thread-per-word pass in HBM (process_tile_direct)."""
    if stream:
        monkeypatch.setenv("YTTM_FORCE_STREAM", "1")
    w = long_words(np.random.default_rng(9), [17_000, 21_000])
    w.check_initial_ids()
    ctx.import_words(w)
    check_run(ctx, oracle, w, 3000, 400, want_done=400)
    assert observed(ctx)["loop_resident"] == (0 if stream else 1)


# ---- 8. a run split in two ------------------------------------------------------------------------------------------
def split_words():
    rng = np.random.default_rng(21)
    return Words.of(*hand_words(rng, 20_000, [3, 5, 8, 12], np.arange(20, 60), np.arange(1000, 1064)))


@pytest.mark.parametrize("seg", ["", "8"])
def test_run_split_in_two(product, oracle, monkeypatch, seg):
    """run(k) + run(n - k, first + k) == run(n): the rules, the words and the table.  With 8-entry exchange segments
    the last merge of the first call overflows a segment, and its lost count changes must not survive the call."""
    if seg:
        monkeypatch.setenv("YTTM_XQ_SEG_CAP", seg)
    w = split_words()
    n, first = 600, 2000
    want = oracle.train_words(w.tok, w.off, w.frq, first, n)
    assert len(want) == n
    for k in (1, 7, 150, 599):
        c = Ctx(product)
        try:
            c.import_words(w)
            rc, r1 = c.run(first, k)
            assert rc == 0 and r1 == want[:k], (k, c.err())
            oracle.train_words(w.tok, w.off, w.frq, first, k)
            check_state(c, oracle, "after run(%d)" % k)
            rc, r2 = c.run(first + k, n - k)
            assert rc == 0 and r2 == want[k:], (k, c.err())
            oracle.train_words(w.tok, w.off, w.frq, first, n)
            check_state(c, oracle, "after run(%d) + run(%d)" % (k, n - k))
        finally:
            c.close()

"""Hot path (a) at sizes where the packed words no longer fit the chip's shared memory: the merge loop runs in
STREAMING mode by itself (TMA ring, deferred rewrites) — the regime bench.py's `roofline.train_scan` measures.  The
oracle cannot follow at this size, so the first merges are recomputed on the host with numpy from the very words the
device generated (yttm_train_synth_words -> yttm_train_export_words): pair counts under the run rule, arg-max under
MergeCandidate::operator< (bpe.cpp:110-126), greedy left-to-right rewrite (stress_test.cpp:181-188)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
DEAD = np.uint32(0xFFFFFFFF)


def np_pair_counts(tok, freq):
    """tok [n, L] uint32 (DEAD padded at the tail), freq [n] -> dict key (x << 32 | y) -> count (run rule: inside a run
    a^k only every second position starts a pair, pairsInSeg bpe.cpp:140-143)."""
    n, L = tok.shape
    par = np.zeros(n, dtype=np.uint8)     # parity of the position inside its run of equal tokens
    keys, wts = [], []
    for j in range(L - 1):
        a, b = tok[:, j], tok[:, j + 1]
        if j > 0:
            par = np.where(tok[:, j] == tok[:, j - 1], par ^ 1, 0).astype(np.uint8)
        live = (a != DEAD) & (b != DEAD)
        counted = live & ((a != b) | (par == 0))
        keys.append((a[counted].astype(np.uint64) << np.uint64(32)) | b[counted].astype(np.uint64))
        wts.append(freq[counted])
    keys, wts = np.concatenate(keys), np.concatenate(wts)
    uk, inv = np.unique(keys, return_inverse=True)
    return uk, np.bincount(inv, weights=wts.astype(np.float64)).astype(np.uint64)


def np_best(uk, cnt):
    x, y = (uk >> np.uint64(32)).astype(np.int64), (uk & np.uint64(0xFFFFFFFF)).astype(np.int64)
    mx, mn = np.maximum(x, y), np.minimum(x, y)
    order = np.lexsort((-x, mn, mx, -cnt.astype(np.int64)))   # count desc, max asc, min asc, x desc
    i = order[0]
    return int(x[i]), int(y[i]), int(cnt[i])


def np_apply(tok, x, y, z):
    n, L = tok.shape
    out = np.full_like(tok, DEAD)
    w = np.zeros(n, dtype=np.int64)
    skip = np.zeros(n, dtype=bool)
    rows = np.arange(n)
    for j in range(L):
        a = tok[:, j]
        active = ~skip & (a != DEAD)
        nxt = tok[:, j + 1] if j + 1 < L else np.full(n, DEAD)
        pair = active & (a == np.uint32(x)) & (nxt == np.uint32(y))
        val = np.where(pair, np.uint32(z), a)
        out[rows[active], w[active]] = val[active]
        w += active
        skip = pair
    return out


@pytest.mark.parametrize("log2_first,alpha", [(0, 300), (6, 300), (0, 2000)])
def test_streaming_merges_equal_a_numpy_recount(product, log2_first, alpha):
    """alpha 2000: every merge creates more new pairs than the per-round table of the front takes (768) — the rounds
    whose new pairs are only bounded by the hash-bucket sketch (merge_loop.cuh: front_take)."""
    L = product
    ctx = C.c_void_p()
    assert L.yttm_ctx_create(0, C.byref(ctx)) == 0
    try:
        wl, iters = 8, 6
        n_w = 1_500_000                     # 12 M tokens = 48 MB: beyond the 132 x 227 KB of shared memory of an H100
        assert L.yttm_train_synth_words(ctx, n_w, wl, alpha | (log2_first << 24), 7) == 0, L.yttm_last_error(ctx)
        nw, nt = C.c_uint64(0), C.c_uint64(0)
        assert L.yttm_train_export_words(ctx, None, 0, None, None, 0, C.byref(nw), C.byref(nt)) == 0
        tok = np.zeros(nt.value, dtype=np.uint32)
        off = np.zeros(nw.value + 1, dtype=np.uint32)
        frq = np.zeros(nw.value, dtype=np.uint64)
        assert L.yttm_train_export_words(ctx, tok.ctypes.data, len(tok), off.ctypes.data, frq.ctypes.data, len(frq),
                                         C.byref(nw), C.byref(nt)) == 0
        assert nw.value == n_w and np.all(np.diff(off.astype(np.int64)) == wl)
        rows = tok.reshape(n_w, wl).copy()
        first_id = 4 + (1 << log2_first) + alpha
        rules = np.zeros(3 * iters, dtype=np.uint32)
        fr = np.zeros(iters, dtype=np.uint64)
        nd = C.c_uint32(0)
        assert L.yttm_train_run(ctx, first_id, iters, rules.ctypes.data, fr.ctypes.data, C.byref(nd)) == 0, L.yttm_last_error(ctx)
        assert nd.value == iters and L.yttm_stage_ms(ctx, b"loop_resident") == 0.0     # STREAMING by itself
        got = [tuple(int(v) for v in rules[3 * i:3 * i + 3]) + (int(fr[i]),) for i in range(iters)]
        want = []
        for m in range(iters):
            uk, cnt = np_pair_counts(rows, frq)
            x, y, c = np_best(uk, cnt)
            want.append((x, y, first_id + m, c))
            rows = np_apply(rows, x, y, first_id + m)
        assert got == want
    finally:
        L.yttm_ctx_destroy(ctx)

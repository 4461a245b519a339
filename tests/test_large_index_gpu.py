"""Positions, cells and byte counts past 2^31 and 2^32, reached with shapes whose inputs are small and whose device peak
is worked out before each test runs.

A. Absolute positions.  The device entry points read sentence i at d_bytes[offsets[i] - offsets[0], ...), the host ones
   at bytes[offsets[i], ...), and spans are in the coordinates of offsets; so a batch of a few KB can carry offsets
   from 2^31 - 3 up to 2^63 - 2^20, and offsets that cross 2^31 and 2^32 in the middle of a word.  Every encode entry
   point (packed ids, spans, padded rows with spans, windows with spans, subword pieces; device and host forms) must give
   at every base the ids, lengths and pieces it gives at base 0, and spans shifted by the base; spans must equal the
   restatement of tests/test_encode_spans_gpu.py, padded rows and windows their definitions.  BPE-dropout keys a word by
   its byte offset inside its sentence, not by its absolute position: the ids at every base equal the reference's replay
   (tests/_dropout_ref.py) under that key, from the device entry and from the chunked host pipeline alike.
B. Outputs past 2^31 cells and 2^32 bytes from small inputs: decoded text of more than 2^32 bytes (one sentence, and
   sentence boundaries at 2^31 + r and 2^32 + r), padded rows whose cell index passes 2^30, 2^31 and 2^32 (ids) and 2^28
   (spans), windows whose cells pass 2^31 and 2^32 (ids) and 2^28 (spans).  Results stay on the device and are compared there,
   exactly, chunk by chunk.

Every GPU test reads torch.cuda.mem_get_info() first and skips, with the numbers, when less than its estimated peak plus
2 GB is free; it closes its handles and empties torch's cache before it returns.  The check bodies of part A take `dev`:
tests/test_large_index_emul_cpu.py runs them under the SIMT emulator, whose device memory is host memory."""
import ctypes as C
import gc

import numpy as np
import pytest

import _cases
import test_encode_dropout_gpu as DG
import test_encode_padded_gpu as PG
import test_encode_spans_gpu as SG
import test_encode_windows_gpu as WG
from _bind import _pack, read_model, tmp_model_path
from youtokentome_b200 import _lib

pytestmark = pytest.mark.gpu

GB = 1 << 30
# the CUDA context, the encoder's tables and the scratch of one call, on top of a test's results
LIB_SLACK = 3 * GB
# the key test of tests/test_encode_dropout_gpu.py (check_keys): its replayed answers are stored
KEY_SEED, KEY_FIRST = 0xDEADBEEF_00000007, 2**32 - 3


# ---- device memory: CUDA memory on a GPU, host memory under the emulator -------------------------------------------
def _put(arr, gpu):
    """(keep-alive, pointer) of a copy of `arr` in device memory."""
    arr = np.ascontiguousarray(arr)
    if gpu:
        import torch
        t = torch.from_numpy(arr.copy()).cuda() if arr.size else torch.zeros(16, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        return t, t.data_ptr()
    return arr, arr.ctypes.data


_TS = {np.int32: ("<i4", C.c_int32), np.uint64: ("<i8", C.c_int64), np.uint8: ("|u1", C.c_uint8)}


def _get(ptr, count, dtype, gpu):
    """A host copy of `count` values of library-owned device memory."""
    count = int(count)
    if count == 0:
        return np.zeros(0, dtype)
    ts, ct = _TS[dtype]
    if gpu:
        import torch
        from youtokentome_b200.distributed import _DevView
        a = torch.as_tensor(_DevView(ptr.value, count, ts), device="cuda").cpu().numpy()
    else:
        a = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ct)), shape=(count,)).copy()
    return a.view(dtype)


# ---- part A: every encode entry point at one base ------------------------------------------------------------------
WIN_K, WIN_S, PAD_W = 8, 3, 7


def encode_all(bpe, data, offs, base, kw, gpu, host=True):
    """{call: [(array, is_span)]} of every encode entry point on the batch (data, offs) with offsets moved to `base`.
    kw: bos / eos / reverse / p / seed / first.  Device forms read the batch at its first byte; host forms get the
    pointer of byte 0 of the offsets' coordinates (the batch's address minus `base`, as a caller passes for a batch in
    the middle of a large mapped buffer)."""
    L = _lib.lib()
    ctx = L.yttm_api_device_context(bpe._h)
    enc = L.yttm_api_device_encoder(bpe._h)
    pad = read_model(bpe.model)[2][1]

    def ok(rc):
        assert rc == 0, L.yttm_last_error(ctx)
    n = len(offs) - 1
    nb = len(data)
    offs = (np.asarray(offs, dtype=np.uint64) + np.uint64(base)).astype(np.uint64)
    b, e, r = (int(kw.get(k, False)) for k in ("bos", "eos", "reverse"))
    fl = (b, e, r, float(kw.get("p", 0.0)), int(kw.get("seed", 0)), int(kw.get("first", 0)))
    keep_b, d_bytes = _put(np.frombuffer(data, dtype=np.uint8), gpu)
    keep_o, d_offs = _put(offs, gpu)
    u8, i4, u1 = np.uint64, np.int32, np.uint8
    g = lambda ptr, count, dt: _get(ptr, count, dt, gpu)
    out = {}
    pi, po, ps, tot = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_uint64(0)
    ok(L.yttm_enc_run_device(enc, d_bytes, d_offs, nb, n, *fl, C.byref(pi), C.byref(po), C.byref(tot)))
    out["device ids"] = [(g(pi, tot.value, i4), False), (g(po, n + 1, u8), False)]
    ok(L.yttm_enc_run_spans_device(enc, d_bytes, d_offs, nb, n, *fl, C.byref(pi), C.byref(po), C.byref(ps),
                                   C.byref(tot)))
    out["device spans"] = [(g(pi, tot.value, i4), False), (g(po, n + 1, u8), False), (g(ps, 2 * tot.value, u8), True)]
    for width in (0, PAD_W + b + e):
        w = C.c_uint32(0)
        ok(L.yttm_enc_run_padded_device(enc, d_bytes, d_offs, nb, n, *fl, width, pad, 1, C.byref(pi), C.byref(po),
                                        C.byref(ps), C.byref(w)))
        out["device padded %d" % width] = [(g(pi, n * w.value, i4), False), (g(po, n, u8), False),
                                           (g(ps, 2 * n * w.value, u8), True)]
    q = [C.c_void_p() for _ in range(5)]
    width = WIN_K + b + e
    ok(L.yttm_enc_run_windows_device(enc, d_bytes, d_offs, nb, n, *fl, width, WIN_S, pad, 1, *[C.byref(x) for x in q],
                                     C.byref(tot)))
    W = tot.value
    out["device windows"] = [(g(q[0], W * width, i4), False)] + [(g(q[k], W, u8), False) for k in (1, 2, 3)] + \
                            [(g(q[4], 2 * W * width, u8), True)]
    n_p, n_b = C.c_uint64(0), C.c_uint64(0)
    ok(L.yttm_enc_run_subwords_device(enc, d_bytes, d_offs, nb, n, *fl, C.byref(pi), C.byref(po), C.byref(ps),
                                      C.byref(n_p), C.byref(n_b)))
    out["device subwords"] = [(g(pi, n_b.value, u1), False), (g(po, n_p.value + 1, u8), False), (g(ps, n + 1, u8), False)]
    del keep_b, keep_o
    if not host:
        return out
    raw = np.frombuffer(data + b"\0", dtype=np.uint8).copy()
    hb = (raw.ctypes.data - base) % 2**64      # byte 0 of the offsets' coordinates
    cap = nb + 3 * n + 16
    ids, oo, sp = np.zeros(cap, i4), np.zeros(n + 1, u8), np.zeros((cap, 2), u8)
    ok(L.yttm_enc_run(enc, hb, offs.ctypes.data, n, *fl, ids.ctypes.data, cap, oo.ctypes.data, C.byref(tot)))
    out["host ids"] = [(ids[:tot.value].copy(), False), (oo.copy(), False)]
    ok(L.yttm_enc_run_spans(enc, hb, offs.ctypes.data, n, *fl, ids.ctypes.data, cap, oo.ctypes.data, sp.ctypes.data,
                            C.byref(tot)))
    out["host spans"] = [(ids[:tot.value].copy(), False), (oo.copy(), False), (sp[:tot.value].reshape(-1).copy(), True)]
    width = PAD_W + b + e
    rows, lens, rsp = np.zeros(n * width, i4), np.zeros(n, u8), np.zeros(2 * n * width, u8)
    ok(L.yttm_enc_run_padded(enc, hb, offs.ctypes.data, n, *fl, width, pad, rows.ctypes.data, lens.ctypes.data,
                             rsp.ctypes.data))
    out["host padded %d" % width] = [(rows, False), (lens, False), (rsp, True)]
    bcap = 4 * nb + 10 * n + 16
    text, tpo, tso = np.zeros(bcap, u1), np.zeros(cap + 1, u8), np.zeros(n + 1, u8)
    ok(L.yttm_enc_run_subwords(enc, hb, offs.ctypes.data, n, *fl, text.ctypes.data, bcap, tpo.ctypes.data, cap,
                               tso.ctypes.data, C.byref(n_p), C.byref(n_b)))
    out["host subwords"] = [(text[:n_b.value].copy(), False), (tpo[:n_p.value + 1].copy(), False), (tso, False)]
    return out


def check_definitions(m, model, sents, offs, res, kw):
    """At one base: spans == the restatement (base included), padded rows and windows == their definitions over the
    packed ids and spans of the same call, host forms == device forms."""
    import torch
    b, e, r = (bool(kw.get(k, False)) for k in ("bos", "eos", "reverse"))
    _, pad, bos_id, eos_id = read_model(m)[2]
    ids, oo, spans = (x for x, _ in res["device spans"])
    oo_i = oo.astype(np.int64)
    for s in range(len(sents)):
        got = [tuple(x) for x in spans.reshape(-1, 2)[oo_i[s]:oo_i[s + 1]].tolist()]
        assert got == SG.oracle_spans(model, sents[s], ids[oo_i[s]:oo_i[s + 1]], int(offs[s]), b, e, r), s
    assert np.array_equal(res["device ids"][0][0], ids) and np.array_equal(res["device ids"][1][0], oo)
    for name in [k for k in res if k.startswith("host")]:
        twin = res["device" + name[4:]]
        assert all(np.array_equal(x, y) for (x, _), (y, _) in zip(res[name], twin)), name
    # the definitions are stated over the ids and spans of the same call without bos / eos / reverse: take them from
    # the rows, whose contents are those ids
    n = len(sents)
    plain = [ids[oo_i[s]:oo_i[s + 1]] for s in range(n)]
    plain_sp = [spans.reshape(-1, 2)[oo_i[s]:oo_i[s + 1]] for s in range(n)]
    if r:
        plain, plain_sp = [x[::-1] for x in plain], [x[::-1] for x in plain_sp]
    plain = [x[int(b):len(x) - int(e)] for x in plain]
    plain_sp = [x[int(b):len(x) - int(e)] for x in plain_sp]
    cat = np.concatenate(plain) if n else np.zeros(0, np.int32)
    cat_sp = np.concatenate(plain_sp) if n else np.zeros((0, 2), np.uint64)
    coo = np.zeros(n + 1, np.int64)
    coo[1:] = np.cumsum([len(x) for x in plain])
    t_offs = torch.from_numpy(offs.astype(np.int64))
    t_sp = torch.from_numpy(cat_sp.astype(np.int64))
    for name in [k for k in res if k.startswith("device padded")]:
        width = int(name.split()[-1]) or None
        want = PG.padded_ref(cat, coo, width, bos_id, eos_id, pad, b, e, r, spans=t_sp, offs=t_offs)
        rows, lens, sp = (x for x, _ in res[name])
        assert np.array_equal(rows, want[0].numpy().reshape(-1)), name
        assert np.array_equal(lens.astype(np.int64), want[1].numpy()), name
        assert np.array_equal(sp.astype(np.int64), want[2].numpy().reshape(-1)), name
    width = WIN_K + int(b) + int(e)
    want = WG.windows_ref(cat, coo, width, WIN_S, bos_id, eos_id, pad, b, e, r, spans=t_sp, offs=t_offs)
    got = [x for x, _ in res["device windows"]]
    assert np.array_equal(got[0], want[0].numpy().reshape(-1))
    for k in (1, 2, 3):
        assert np.array_equal(got[k].astype(np.int64), want[k].numpy()), k
    assert np.array_equal(got[4].astype(np.int64), want[4].numpy().reshape(-1))


def same_shifted(res, res0, base, tag):
    assert res.keys() == res0.keys()
    for name in res0:
        for k, ((x, span), (x0, _)) in enumerate(zip(res[name], res0[name])):
            want = x0 + np.uint64(base) if span else x0
            assert x.dtype == want.dtype and np.array_equal(x, want), (tag, name, k, base)


def _bases(data, offs):
    """Offset bases: next to 2^31, 2^32, above 2^32, 2^40 and 2^63 - 2^20; and 2^31 / 2^32 two bytes into the middle
    sentence, so that those positions fall inside the batch, inside a word."""
    mid = int(offs[(len(offs) - 1) // 2]) + 2
    return [2**31 - 3, 2**31 - mid, 2**32 - 1, 2**32 - mid, 2**32 + 5, 2**40 + 7, 2**63 - 2**20]


def check_bases(oracle, dev=False):
    """Part A without dropout and with it: every entry point at every base == base 0 shifted; definitions hold at
    every base."""
    m = DG._zipf_model(oracle)
    bpe, model = SG._bpe(m), SG.Model(m)
    zc = _cases.zipf()
    long_word = b"".join(zc.sentences(4, 60, seed=6)).replace(b" ", b"")
    sents = (_cases.zipf_sentences(60) + _cases.EDGE_SENTENCES + SG.ADVERSARIAL +
             [long_word, b"q " + long_word[:41] + b" " + long_word[:300],
              b" ".join(zc.sentences(250, 80, seed=5))])                  # longer than the finder's 16 KB piece
    data, offs = _pack(sents)
    for kw in (dict(), dict(bos=True, eos=True, reverse=True), dict(p=0.1, seed=KEY_SEED, first=KEY_FIRST)):
        res0 = encode_all(bpe, data, offs, 0, kw, dev)
        check_definitions(m, model, sents, offs, res0, kw)
        for base in _bases(data, offs):
            res = encode_all(bpe, data, offs, base, kw, dev)
            same_shifted(res, res0, base, kw)
            check_definitions(m, model, sents, offs + np.uint64(base), res, kw)
    del bpe


def check_dropout_key(oracle, dev=False):
    """BPE-dropout at every base == the reference's replay keyed by (seed, sentence index, byte offset of the word in
    its sentence, draw): sentence indices across 2^32, a seed with a high half; the device entry and the host form."""
    m = DG._zipf_model(oracle)
    bpe = SG._bpe(m)
    sents = _cases.zipf().sentences(8, 80, seed=41)
    data, offs = _pack(sents)
    for p in (0.1, 0.5):
        want = DG.expected(m, sents, p, KEY_SEED, KEY_FIRST)
        kw = dict(p=p, seed=KEY_SEED, first=KEY_FIRST)
        for base in [0] + _bases(data, offs):
            res = encode_all(bpe, data, offs, base, kw, dev)
            for name in ("device ids", "host ids"):
                ids, oo = (x for x, _ in res[name])
                oo = oo.astype(np.int64)
                DG.same([ids[oo[i]:oo[i + 1]].tolist() for i in range(len(sents))], want, sents, (name, p, base))
    del bpe


def check_chunked_bases(oracle, monkeypatch):
    """The host pipeline cut into 1 MB chunks (each chunk's offsets start far from 0) at bases across 2^32 and at
    2^40 + 7, with dropout: the ids and spans of the one-chunk device entry at base 0."""
    monkeypatch.setenv("YTTM_ENC_CHUNK_MB", "1")
    m = DG._zipf_model(oracle)
    bpe = SG._bpe(m)
    sents = _cases.zipf().sentences(30_000, 100, seed=47)
    data, offs = _pack(sents)
    assert len(data) > 2.5 * (1 << 20)
    kw = dict(p=0.2, seed=9, first=2**31 - 7)
    res0 = encode_all(bpe, data, offs, 0, kw, True, host=False)
    L = _lib.lib()
    for base in (2**32 - len(data) // 2, 2**40 + 7):
        res = encode_all(bpe, data, offs, base, kw, True)
        assert L.yttm_stage_ms(L.yttm_api_device_context(bpe._h), b"enc_chunks") >= 2
        for name, twin in (("host ids", "device ids"), ("host spans", "device spans")):
            for k, ((x, span), (x0, _)) in enumerate(zip(res[name], res0[twin])):
                assert np.array_equal(x, x0 + np.uint64(base) if span else x0), (name, k, base)
    del bpe


# ---- device memory bookkeeping -------------------------------------------------------------------------------------
class DeviceBudget:
    """Skips unless `need` bytes + 2 GB are free; samples free memory after the library calls and at the end to report
    the test's peak (workspace a call allocates and frees before it returns is not seen)."""

    def __init__(self, need, what):
        import torch
        torch.cuda.empty_cache()
        free, total = torch.cuda.mem_get_info()
        self.need, self.what, self.free0, self.low = need, what, free, free
        if free < need + 2 * GB:
            pytest.skip("%s needs about %.1f GB of device memory + 2 GB headroom; %.1f GB of %.1f GB are free"
                        % (what, need / GB, free / GB, total / GB))

    def sample(self):
        import torch
        torch.cuda.synchronize()
        self.low = min(self.low, torch.cuda.mem_get_info()[0])

    def close(self):
        import torch
        self.sample()
        gc.collect()
        torch.cuda.empty_cache()
        print("\n[device peak] %s: estimated %.2f GB, measured %.2f GB" % (self.what, self.need / GB,
                                                                          (self.free0 - self.low) / GB))


# ---- part B: decode to more than 2^32 bytes ------------------------------------------------------------------------
def _long_piece_model(oracle):
    """A model of long space-free words: its longest piece is a whole 4 400-byte word with its leading U+2581."""
    word = b"abcd" * 1100
    text = b" ".join([word, word[:1500], word, b"abcdab" * 300] * 6)
    m = tmp_model_path("orc")
    oracle.train(text, m, 40)
    return m


def _device_piece_table(bpe, m):
    import torch
    import test_decode_gpu as DE
    flat, starts, lens, lead = DE.piece_table(bpe, m)
    t = lambda a: torch.from_numpy(np.asarray(a)).cuda()
    return t(flat.copy()), t(starts), t(lens), t(lead), (flat, starts, lens, lead)


def check_decode_against_oracle(tab, ids, offs, text, toff, chunk_bytes=1 << 27):
    """text / toff == oracle_decode of tests/test_decode_gpu.py, evaluated on the device chunk of ids by chunk."""
    import torch
    flat, starts, lens, lead = tab[:4]
    offs = torch.as_tensor(np.asarray(offs, dtype=np.int64)).cuda()
    n_ids = int(offs[-1])
    sent = torch.repeat_interleave(torch.arange(len(offs) - 1, device="cuda"), offs[1:] - offs[:-1], output_size=n_ids)
    first = torch.ones(n_ids, dtype=torch.bool, device="cuda")
    first[1:] = sent[1:] != sent[:-1]
    ids = ids.to(torch.int64)
    strip = (first & lead[ids]).to(torch.int64)
    ln, st = lens[ids] - strip, starts[ids] + strip
    out_start = torch.cumsum(ln, 0) - ln
    total = int(ln.sum())
    assert text.numel() == total
    per = torch.zeros(len(offs) - 1, dtype=torch.int64, device="cuda").index_add_(0, sent, ln)
    want_off = torch.zeros(len(offs), dtype=torch.int64, device="cuda")
    want_off[1:] = torch.cumsum(per, 0)
    assert torch.equal(toff.to(torch.int64), want_off)
    a = 0
    ends = torch.cumsum(ln, 0).cpu().numpy()
    while a < n_ids:
        lo_byte = int(out_start[a])
        b = max(int(np.searchsorted(ends, lo_byte + chunk_bytes, side="right")), a + 1)
        nb = int(ends[b - 1]) - lo_byte
        idx = torch.repeat_interleave(st[a:b] - (out_start[a:b] - lo_byte), ln[a:b], output_size=nb) + \
            torch.arange(nb, device="cuda")
        if not torch.equal(flat[idx], text[lo_byte:lo_byte + nb]):
            bad = int(torch.nonzero(flat[idx] != text[lo_byte:lo_byte + nb])[0]) + lo_byte
            raise AssertionError("decoded text differs at byte %d (ids %d..%d)" % (bad, a, b))
        del idx
        a = b


def _decode_case(oracle, shape):
    """(model, bpe, ids, offsets) of a decode whose text passes 2^32 bytes."""
    m = _long_piece_model(oracle)
    bpe = SG._bpe(m)
    vocab = bpe.vocab()
    special = set(read_model(m)[2])
    text_len = lambda i: len(vocab[i].replace("▁", " ").encode())     # decoded, not first in its sentence
    big = max(range(len(vocab)), key=text_len)
    one = min(i for i in range(len(vocab)) if i not in special and text_len(i) == 1 and vocab[i] != "▁")
    P = text_len(big)
    assert P >= 4096, P
    rng = np.random.default_rng(11)
    # every sentence starts with the 1-byte piece, so no leading space is stripped and a big piece always gives P bytes
    if shape == "one sentence":
        # 1.1 M ids, about one in 64 a 1-byte piece: every alignment of a 4 KB piece, 2^32 passed mid-piece
        n = 1_100_000
        ids = np.where(rng.random(n) < 1 / 64, one, big).astype(np.int32)
        ids[0] = one
        offs = np.array([0, n], dtype=np.uint64)
        assert int(np.where(ids == big, P, 1).astype(np.int64).sum()) > 2**32
        return m, bpe, ids, offs
    # sentence ends at 2^31 + r and 2^32 + r, r = 0 .. 3: 1-byte sentences between, the long ones shifted by 1 .. 3
    runs, pos = [], 0

    def fill(to):   # one sentence of big pieces and 1-byte pieces from pos up to `to`
        nonlocal pos
        k, rem = divmod(to - pos - 1, P)
        s = np.full(1 + k + rem, big, dtype=np.int32)
        s[0] = one
        s[1 + rng.choice(k + rem, rem, replace=False)] = one
        runs.append(s)
        pos = to
    for hi in (2**31, 2**32):
        fill(hi)
        for _ in range(3):
            fill(pos + 1)
    fill(pos + 5 * P + 3)
    ids = np.concatenate(runs)
    offs = np.zeros(len(runs) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(s) for s in runs])
    return m, bpe, ids, offs


@pytest.mark.parametrize("shape", ["one sentence", "boundaries at 2^31 + r and 2^32 + r"])
def test_decode_past_2_32_bytes(product, oracle, shape):
    import torch
    n_text = 2**32 + 2**29
    budget = DeviceBudget(2 * n_text + LIB_SLACK, "decode_packed(out='cuda') to 4.3 GB of text (%s)" % shape)
    m, bpe, ids, offs = _decode_case(oracle, shape)
    tab = _device_piece_table(bpe, m)
    d_ids = torch.from_numpy(ids).cuda()
    text, toff = bpe.decode_packed(d_ids, torch.from_numpy(offs.astype(np.int64)).cuda(), out="cuda")
    budget.sample()
    assert text.is_cuda and text.numel() > 2**32
    if shape != "one sentence":
        got = toff.cpu().numpy()
        for hi in (2**31, 2**32):
            assert [v for v in got.tolist() if hi <= v < hi + 4] == [hi, hi + 1, hi + 2, hi + 3]
    check_decode_against_oracle(tab, d_ids, offs, text, toff)
    budget.sample()
    del text, toff, d_ids, tab, bpe
    budget.close()


# ---- part B: padded rows past 2^30, 2^31, 2^32 cells (ids) and 2^28 cells (spans) ----------------------------------
def _rows_case(oracle, n_rows):
    m = DG._zipf_model(oracle)
    bpe = SG._bpe(m)
    sents = _cases.zipf().sentences(n_rows, 120, seed=71)
    data, offs = _pack(sents)
    ids, oo, spans = bpe.encode_packed(data, offs, with_spans=True)
    assert all(oo[i + 1] - oo[i] >= 8 for i in range(n_rows))
    return m, bpe, data, offs, ids, oo.astype(np.int64), spans.astype(np.int64)


def _check_rows(rows, lens, spans, ids, oo, p_spans, offs, pad, boundaries):
    """Row i == its ids then pads; the cells around every boundary cell index exactly; spans likewise."""
    import torch
    n, L = rows.shape
    want_len = oo[1:] - oo[:-1]
    assert lens.cpu().numpy().tolist() == want_len.tolist()
    flat = rows.view(-1)
    step = 1 << 28
    for i in range(n):
        k = int(want_len[i])
        assert rows[i, :k].cpu().numpy().tolist() == ids[oo[i]:oo[i + 1]].tolist(), i
        for a in range(k, L, step):
            assert not bool((rows[i, a:min(a + step, L)] != pad).any()), (i, a)
        if spans is not None:
            assert np.array_equal(spans[i, :k].cpu().numpy(), p_spans[oo[i]:oo[i + 1]]), i
            for a in range(k, L, step // 2):
                assert not bool((spans[i, a:min(a + step // 2, L)] != int(offs[i + 1])).any()), (i, a)
    for c in boundaries:   # the cells next to the boundary, against the definition written out
        want = []
        for j in range(c - 4, c + 4):
            i, col = divmod(j, L)
            want.append(int(ids[oo[i] + col]) if col < want_len[i] else pad)
        assert flat[c - 4:c + 4].cpu().numpy().tolist() == want, c
        if spans is not None:
            sflat = spans.view(-1, 2)
            for j in range(c - 4, c + 4):
                i, col = divmod(j, L)
                w = p_spans[oo[i] + col].tolist() if col < want_len[i] else [int(offs[i + 1])] * 2
                assert sflat[j].cpu().numpy().tolist() == w, (c, j)


@pytest.mark.parametrize("case", ["ids past 2^30 and 2^31 cells", "ids past 2^32 cells", "spans past 2^28 cells"])
def test_padded_rows_past_2_31_cells(product, oracle, case):
    """encode_padded(out='cuda') with a few short sentences and a large max_length: row i starts at i * L.  With
    L = 2^30 - 1 rows 1 and 2 start just below 2^30 and 2^31 and their ids cross them; with L = 2^30 + 1 rows 2 and 4
    start just past 2^31 and 2^32 (a row base a 32-bit product would wrap); with spans, L = 2^27 - 1 puts the span
    bytes of row 2 across 2^32."""
    spans = case.startswith("spans")
    n_rows, L = {"ids past 2^30 and 2^31 cells": (3, 2**30 - 1), "ids past 2^32 cells": (5, 2**30 + 1),
                 "spans past 2^28 cells": (3, 2**27 - 1)}[case]
    cells = n_rows * L
    per_cell = 4 + (16 if spans else 0)
    budget = DeviceBudget(2 * per_cell * cells + LIB_SLACK, "encode_padded of %d x %d cells%s" % (n_rows, L,
                                                                                           " with spans" * spans))
    m, bpe, data, offs, ids, oo, p_spans = _rows_case(oracle, n_rows)
    pad = read_model(m)[2][1]
    res = bpe.encode_padded(data, offs, max_length=L, out="cuda", with_spans=spans)
    budget.sample()
    rows, lens = res[0], res[1]
    assert rows.shape == (n_rows, L) and rows.is_cuda
    boundaries = [c for c in (2**28, 2**30, 2**31, 2**32) if c < cells and (spans or c >= 2**30)] + \
        [i * L for i in range(1, n_rows)]
    _check_rows(rows, lens, res[2] if spans else None, ids, oo, p_spans, offs, pad, boundaries)
    budget.sample()
    del res, rows, lens, bpe
    budget.close()


# ---- part B: windows past 2^31 cells (ids) and 2^28 cells (spans) --------------------------------------------------
def _one_sentence_of(bpe, n_min, n_max):
    """A sentence whose packed encode has between n_min and n_max ids (cut behind a word), with its ids and spans."""
    zc = _cases.zipf()
    text = b" ".join(zc.sentences(n_max // 12, 100, seed=81))
    ids, oo, spans = bpe.encode_packed(text, np.array([0, len(text)], dtype=np.uint64), with_spans=True)
    assert len(ids) > n_min
    ends = spans[:, 1].astype(np.int64)
    j = next(j for j in range(n_min, len(ids)) if ends[j - 1] < len(text) and text[ends[j - 1]] == 0x20)
    assert j <= n_max
    sent = text[:ends[j - 1]]
    ids, oo, spans = bpe.encode_packed(sent, np.array([0, len(sent)], dtype=np.uint64), with_spans=True)
    assert len(ids) == j
    return sent, ids, spans.astype(np.int64)


@pytest.mark.parametrize("case", ["ids past 2^31 cells", "ids past 2^32 cells", "spans past 2^28 cells"])
def test_windows_past_2_31_cells(product, oracle, case):
    """encode_windows of one sentence of 100 k or 130 k ids with a step of one id (stride = K - 1): W = n - K + 1 rows
    of L = 2^16 cells, just past 2^31 or 2^32 cells; with spans L = 2^12, past 2^28 cells (2^32 bytes of spans)."""
    import torch
    spans = case.startswith("spans")
    L = 2**12 if spans else 2**16
    bound = {"ids past 2^31 cells": 2**31, "ids past 2^32 cells": 2**32, "spans past 2^28 cells": 2**28}[case]
    n_lo = bound // L + L + 1      # n - L + 1 rows of L cells past the boundary
    per_cell = 4 + (16 if spans else 0)
    est_rows = n_lo + 2000 - L + 1
    budget = DeviceBudget(2 * per_cell * est_rows * L + LIB_SLACK, "encode_windows of %d-cell rows%s" % (L, " with spans" * spans))
    m = DG._zipf_model(oracle)
    bpe = SG._bpe(m)
    sent, ids, p_spans = _one_sentence_of(bpe, n_lo, n_lo + 2000)
    n = len(ids)
    res = bpe.encode_windows(sent, np.array([0, len(sent)], dtype=np.uint64), max_length=L, stride=L - 1, out="cuda",
                             with_spans=spans)
    budget.sample()
    W = n - L + 1
    rows, lens, sent_of, start = res[:4]
    assert rows.shape == (W, L) and W * L > bound
    ar = torch.arange(W, device="cuda")
    assert bool((lens == L).all()) and bool((sent_of == 0).all()) and torch.equal(start, ar)
    c = torch.from_numpy(ids).cuda().unfold(0, L, 1)                         # row r = ids[r : r + L]
    cs = torch.from_numpy(p_spans).cuda().unfold(0, L, 1).permute(0, 2, 1) if spans else None
    step = max(1, (1 << 26) // L)
    for a in range(0, W, step):
        b = min(a + step, W)
        assert torch.equal(rows[a:b], c[a:b]), (a, b)
        if spans:
            assert torch.equal(res[4][a:b], cs[a:b]), (a, b)
    flat = rows.view(-1)
    for bnd in (2**28, 2**31, 2**32):
        if bnd < W * L:
            want = [int(ids[j // L + j % L]) for j in range(bnd - 4, bnd + 4)]
            assert flat[bnd - 4:bnd + 4].cpu().numpy().tolist() == want, bnd
    budget.sample()
    del res, rows, lens, sent_of, start, c, cs, flat, bpe
    budget.close()


# ---- part A on the GPU ---------------------------------------------------------------------------------------------
def test_absolute_offsets(product, oracle):
    budget = DeviceBudget(GB, "encode of a few KB at large offsets")
    check_bases(oracle, dev=True)
    budget.close()


def test_dropout_key_at_absolute_offsets(product, oracle):
    budget = DeviceBudget(GB, "dropout encode of a few KB at large offsets")
    check_dropout_key(oracle, dev=True)
    budget.close()


def test_chunked_host_pipeline_at_absolute_offsets(product, oracle, monkeypatch):
    budget = DeviceBudget(GB, "chunked host encode of 3 MB at large offsets")
    check_chunked_bases(oracle, monkeypatch)
    budget.close()


# ---- part C: streams of more than 4 GiB through pipes, nothing on disk ---------------------------------------------
# encode_file and decode_file write "-" to file descriptor 1 (a named output is written under a temporary name and
# renamed); the tests point descriptor 1 at a pipe for the call.  decode_file's .npy pair is read with fstat and pread,
# so it cannot come from a pipe: the id base past 2^32 of that stream is not reached here.
import os
import subprocess
import sys
import threading


def _writer(fd, block, k):
    """A thread that writes block * k to fd (or to the named pipe at that path, opened in the thread) and closes it."""
    def run():
        try:
            with (open(fd, "wb", buffering=0) if isinstance(fd, str) else os.fdopen(fd, "wb", buffering=0)) as f:
                big = block * max(1, (16 << 20) // len(block))
                per = len(big) // len(block)
                left = k
                while left:
                    n = min(per, left)
                    f.write(big if n == per else block * n)
                    left -= n
        except BrokenPipeError:
            pass
    t = threading.Thread(target=run, daemon=True)
    t.start()
    return t


class _Stdout:
    """Descriptor 1 pointed at `fd` (the write end of a pipe) inside the with-block."""

    def __init__(self, fd):
        self.fd = fd

    def __enter__(self):
        sys.stdout.flush()
        self.saved = os.dup(1)
        os.dup2(self.fd, 1)
        os.close(self.fd)

    def __exit__(self, *exc):
        os.dup2(self.saved, 1)
        os.close(self.saved)


def _cli(*args, stdin):
    env = dict(os.environ, PYTHONPATH=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    return subprocess.Popen([sys.executable, "-m", "youtokentome_b200.yttm_cli"] + list(args), stdin=stdin,
                            stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env)


def _round_trip_block(oracle):
    """(model, lines of words of the model joined by single spaces): every character is in the model, so decoding the
    encoding gives the lines back."""
    zc = _cases.zipf()
    lines = [b" ".join(s.split()) for s in zc.sentences(600, 100, seed=91)]
    block = b"\n".join(l for l in lines if l) + b"\n"
    m = tmp_model_path("orc")
    oracle.train(block, m, 900, 1.0)
    return m, block


def test_stream_round_trip_past_4_gib(product, oracle):
    """4.6 GB of lines through a pipe into encode_file(text=True), its id text through a pipe into `yttm decode_file
    --text`, the decoded text through a pipe back: it must equal the input byte for byte; the id total is the block's
    (from the oracle, once) times the repeats; the encoder's device peak is that of a 512 MB stream."""
    budget = DeviceBudget(8 * GB, "encode and decode streams")
    import youtokentome_b200 as yttm
    m, block = _round_trip_block(oracle)
    reps = (int(4.6e9) + len(block) - 1) // len(block)
    n_lines_block = block.count(b"\n")
    block_ids = sum(len(x) for x in oracle.encoder(m).encode(block.split(b"\n")[:-1]))
    bpe = yttm.BPE(m)
    L = _lib.lib()
    ctx = L.yttm_api_device_context(bpe._h)
    r0, w0 = os.pipe()
    s_r, s_w = os.pipe()
    drain = threading.Thread(target=lambda: [None for _ in iter(lambda: os.read(s_r, 1 << 20), b"")], daemon=True)
    drain.start()
    small_reps = (512 << 20) // len(block)                  # 16 pieces of 32 MB
    writer = _writer(w0, block, small_reps)
    with _Stdout(s_w):
        small = bpe.encode_file(r0, "-", text=True)
    os.close(r0)
    writer.join()
    drain.join()
    os.close(s_r)
    small_peak = L.yttm_stage_ms(ctx, b"stream_dev_peak_bytes")
    assert small["lines"] == small_reps * n_lines_block and small["ids"] == small_reps * block_ids

    a_r, a_w = os.pipe()      # generator -> encode_file
    b_r, b_w = os.pipe()      # encode_file -> decode_file
    dec = _cli("decode_file", "--model", m, "--input", "-", "--output", "-", "--text", stdin=b_r)
    os.close(b_r)
    seen = {"n": 0, "bad": None}

    def read():
        pat = block * max(1, (8 << 20) // len(block))
        while True:
            chunk = dec.stdout.read(4 << 20)
            if not chunk:
                break
            at = seen["n"] % len(block)
            k = len(chunk)
            if seen["bad"] is None and memoryview(pat)[at:at + k] != chunk:
                seen["bad"] = seen["n"]
            seen["n"] += k
    reader = threading.Thread(target=read, daemon=True)
    reader.start()
    writer = _writer(a_w, block, reps)
    try:
        with _Stdout(b_w):
            stats = bpe.encode_file(a_r, "-", text=True)
    finally:
        os.close(a_r)
        writer.join()
        reader.join()
        dec.wait()
        err = dec.stderr.read()
    budget.sample()
    assert dec.returncode == 0, err.decode(errors="replace")[-2000:]
    assert stats["bytes"] == reps * len(block) > 2**32
    assert stats["lines"] == reps * n_lines_block
    assert stats["ids"] == reps * block_ids
    assert seen["bad"] is None, "decoded text differs from the input in the 4 MB read at byte %d" % seen["bad"]
    assert seen["n"] == reps * len(block)
    assert L.yttm_stage_ms(ctx, b"stream_dev_peak_bytes") == small_peak
    del bpe
    budget.close()


def test_stream_line_counter_past_2_31(product, oracle):
    """2^31 + 2^20 lines of one and two bytes through a pipe into encode_file(text=True, dropout_prob=0.5): the line
    counter and the dropout sentence index pass 2^31.  The lines next to line 2^31 equal yttm_enc_run of each line alone
    with its own sentence index; the line and id totals are the analytic ones."""
    budget = DeviceBudget(8 * GB, "encode stream of 2^31 lines")
    import youtokentome_b200 as yttm
    m = tmp_model_path("orc")
    oracle.train(b"ab a b ba abb " * 2000, m, 12, 1.0)
    bpe = yttm.BPE(m)
    block = b"a\nab\na\nba\n"
    per = block.count(b"\n")
    n_lines = 2**31 + 2**20
    reps = n_lines // per
    want_lines = [(block.split(b"\n")[i % per]) for i in range(2**31 - 3, 2**31 + 3)]
    seed, p = 12345, 0.5
    bpe.dropout_seed(seed)
    out_r, out_w = os.pipe()
    grab = {"lines": 0, "carry": b"", "got": [], "ids": 0}
    lo, hi = 2**31 - 3, 2**31 + 3

    def read():
        with os.fdopen(out_r, "rb", buffering=0) as f:
            while True:
                chunk = f.read(4 << 20)
                if not chunk:
                    break
                grab["ids"] += chunk.count(b" ")
                nl = chunk.count(b"\n")
                first = grab["lines"]
                if first + nl >= lo and first < hi:
                    parts = (grab["carry"] + chunk).split(b"\n")
                    for j, line in enumerate(parts[:-1]):
                        if lo <= first + j < hi:
                            grab["got"].append(line)
                    grab["carry"] = parts[-1]
                else:
                    grab["carry"] = chunk[chunk.rfind(b"\n") + 1:] if nl else grab["carry"] + chunk
                grab["lines"] += nl
    reader = threading.Thread(target=read, daemon=True)
    reader.start()
    in_r, in_w = os.pipe()
    writer = _writer(in_w, block, reps)
    try:
        with _Stdout(out_w):
            stats = bpe.encode_file(in_r, "-", text=True, dropout_prob=p)
    finally:
        os.close(in_r)
        writer.join()
        reader.join()
    budget.sample()
    assert stats["lines"] == grab["lines"] == reps * per > 2**31
    assert stats["ids"] == grab["ids"]
    # the spot check: each line alone, as sentence index i of the same seed
    enc = _lib.lib().yttm_api_device_encoder(bpe._h)
    Lb = _lib.lib()
    want = []
    for i, line in zip(range(lo, hi), want_lines):
        offs = np.array([0, len(line)], dtype=np.uint64)
        ids, oo, tot = np.zeros(16, np.int32), np.zeros(2, np.uint64), C.c_uint64(0)
        assert Lb.yttm_enc_run(enc, line, offs.ctypes.data, 1, 0, 0, 0, p, seed, i, ids.ctypes.data, 16,
                               oo.ctypes.data, C.byref(tot)) == 0
        want.append(b"".join(b"%d " % x for x in ids[:tot.value]))
    assert grab["got"] == want
    del bpe
    budget.close()


def test_fed_training_past_2_32(product, oracle):
    """A 6.9 GB corpus through a named pipe into BPE.train (a pipe is always fed) and through a pipe into count_words:
    one word occurs more than 2^31 times, one code point more than 2^32 times.  The corpus is one block repeated, so
    its table is the block's times the repeats: count_words must return exactly that, data_len is above 2^32, and the
    model equals, byte for byte, train_from_counts on that table and the oracle trained on the block (every count
    scaled by the same factor: the same merges)."""
    budget = DeviceBudget(2 * GB, "fed training")
    import tempfile
    import youtokentome_b200 as yttm
    block = b"a " * 60 + b"a" * 60 + b" ab abc bca cab\n"
    reps = 2**31 // 60 + 1
    assert 60 * reps > 2**31 and 121 * reps > 2**32
    small = yttm.BPE.count_words(block)
    r, w = os.pipe()
    writer = _writer(w, block, reps)
    try:
        big = yttm.BPE.count_words(r)
    finally:
        os.close(r)
        writer.join()
    budget.sample()
    words = lambda t: {bytes(t.word_bytes[int(t.word_offsets[i]):int(t.word_offsets[i + 1])]): int(t.counts[i])
                       for i in range(len(t.counts))}
    assert words(big) == {k: v * reps for k, v in words(small).items()}
    assert words(big)[b"a"] > 2**31
    assert big.separators == small.separators * reps and big.data_len == small.data_len * reps > 2**32
    d = tempfile.mkdtemp(prefix="yttm_b200_")
    fifo = os.path.join(d, "corpus")
    os.mkfifo(fifo)
    m_fed, m_tab, m_orc = (os.path.join(d, x) for x in ("fed.yttm", "table.yttm", "orc.yttm"))
    t = _writer(fifo, block, reps)
    try:
        yttm.BPE.train(fifo, m_fed, 40)
    finally:
        t.join()
        os.unlink(fifo)
    report = yttm.train_report()
    budget.sample()
    assert int(report["data_len"]) == small.data_len * reps
    yttm.BPE.train_from_counts(big, m_tab, 40)
    oracle.train(block, m_orc, 40)
    blob = lambda path: open(path, "rb").read()
    assert blob(m_fed) == blob(m_tab)
    assert read_model(m_fed) == read_model(m_orc)
    for x in (m_fed, m_tab, m_orc):
        os.unlink(x)
    os.rmdir(d)
    budget.close()

"""Overlapping windows of device encode (`BPE.encode_windows`, yttm_enc_run_windows_device, win_count_kernel /
win_gather_kernel in youtokentome_b200/csrc/encode.cu).  Two expectations: `windows_ref`, the definition of
yttm_enc_run_windows_device applied with torch to encode_packed's ids, offsets and spans of the same call (encode_packed
is pinned to the oracle elsewhere), and `windows_from_lists`, the definition in plain Python over the oracle's id lists.
The check bodies take `dev`: True runs them through the Python surface with every input and output kind and at the
sizes only a GPU finishes quickly; tests/test_encode_windows_emul_cpu.py runs them with False under the SIMT emulator,
through the device C entry on host memory (the emulator's device memory)."""
import ctypes as C

import numpy as np
import pytest

import _cases
import test_encode_emit_gpu as EM
import test_encode_padded_gpu as PG
import test_encode_spans_gpu as SG
from _bind import _pack, tmp_model_path
from youtokentome_b200 import _lib, synth

pytestmark = pytest.mark.gpu

KWS = SG.KWS
PAD_FROM_MODEL = -2**63


# ---- the definition ------------------------------------------------------------------------------------------------
def windows_ref(ids, oo, L, S, bos_id, eos_id, pad, bos=False, eos=False, reverse=False, spans=None, offs=None):
    """Windows of encode_packed's output (ids / oo / spans of a call with bos = eos = reverse = False) as torch tensors
    on the ids' device: (ids [W, L] int32, lengths [W], sentence [W], start [W] int64, spans [W, L, 2] int64 or None)."""
    import torch
    t = lambda x: x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x).astype(np.int64))
    ids = t(ids).to(torch.int64)
    dev = ids.device
    oo = t(oo).to(torch.int64).to(dev)
    n, be = oo.numel() - 1, int(bos) + int(eos)
    K = L - be
    D = K - S
    cnt = oo[1:] - oo[:-1]
    w = torch.where(cnt <= K, torch.ones_like(cnt), 1 + (cnt - K + D - 1).clamp(min=0) // D)
    W = int(w.sum())
    sent = torch.repeat_interleave(torch.arange(n, device=dev), w, output_size=W)
    first = torch.cumsum(w, 0) - w
    start = (torch.arange(W, device=dev) - first[sent]) * D
    lens = torch.clamp(cnt[sent] - start, max=K) + be
    col = torch.arange(L, device=dev)[None, :]
    last = lens[:, None] - 1
    p = last - col if reverse else col.expand(W, L)          # place in the unreversed row
    valid = col < lens[:, None]
    is_bos = valid & (p == 0) if bos else torch.zeros_like(valid)
    is_eos = valid & (p == last) if eos else torch.zeros_like(valid)
    content = valid & ~is_bos & ~is_eos
    src = (oo[:-1][sent][:, None] + start[:, None] + p - int(bos)).clamp(0, max(ids.numel() - 1, 0))
    out = torch.full((W, L), pad, dtype=torch.int64, device=dev)
    if ids.numel():
        out = torch.where(content, ids[src], out)
    out = torch.where(is_bos, torch.full_like(out, bos_id), out)
    out = torch.where(is_eos, torch.full_like(out, eos_id), out)
    sp = None
    if spans is not None:
        spans, o = t(spans).to(torch.int64).reshape(-1, 2).to(dev), t(offs).to(torch.int64).to(dev)
        lo, hi = o[:-1][sent][:, None, None].expand(W, L, 2), o[1:][sent][:, None, None].expand(W, L, 2)
        sp = hi.clone()
        if spans.shape[0]:
            sp = torch.where(content[..., None], spans[src], sp)
        sp = torch.where(is_bos[..., None], lo, sp)
    return out.to(torch.int32), lens, sent, start, sp


def windows_from_lists(content, L, S, bos_id, eos_id, pad, bos, eos, reverse):
    """The definition in plain Python over per-sentence id lists (the oracle's): (ids, lengths, sentence, start)."""
    be = int(bos) + int(eos)
    K = L - be
    D = K - S
    rows, lens, sent, start = [], [], [], []
    for i, c in enumerate(content):
        c = list(c)
        w = 1 if len(c) <= K else 1 + -(-(len(c) - K) // D)
        for k in range(w):
            row = ([bos_id] if bos else []) + c[k * D:k * D + K] + ([eos_id] if eos else [])
            row = row[::-1] if reverse else row
            rows.append(row + [pad] * (L - len(row)))
            lens.append(len(row))
            sent.append(i)
            start.append(k * D)
    return (np.array(rows, np.int32).reshape(-1, L), np.array(lens, np.int64), np.array(sent, np.int64),
            np.array(start, np.int64))


# ---- library calls -------------------------------------------------------------------------------------------------
def windows_abi(bpe, data, offs, L, S, pad, kw, spans):
    """yttm_api_encode_windows_device on HOST memory: the emulator's device memory is host memory."""
    Lb = _lib.lib()
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    raw = bytes(data)
    n = len(offs) - 1
    first = int(offs[0])
    buf = C.create_string_buffer(raw[first:] + b"\0")
    p = [C.c_void_p() for _ in range(5)]
    rows = C.c_uint64(0)
    rc = Lb.yttm_api_encode_windows_device(bpe._h, C.cast(buf, C.c_void_p), offs.ctypes.data, int(offs[-1]) - first, n,
                                           int(kw.get("bos", False)), int(kw.get("eos", False)),
                                           int(kw.get("reverse", False)), float(kw.get("dropout_prob", 0.0)), L, S, pad,
                                           int(spans), *[C.byref(x) for x in p], C.byref(rows))
    if rc != 0:
        raise ValueError(Lb.yttm_api_last_error(bpe._h).decode())
    W = rows.value

    def arr(ptr, count, ct, shape):
        if count == 0:
            return np.zeros(shape, dtype=np.dtype(ct))
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ct)), shape=(count,)).copy().reshape(shape)
    res = [arr(p[0], W * L, C.c_int32, (W, L))] + [arr(p[i], W, C.c_int64, (W,)) for i in (1, 2, 3)]
    if spans:
        res.append(arr(p[4], 2 * W * L, C.c_uint64, (W, L, 2)))
    else:
        assert not p[4].value
    return tuple(res)


def call_windows(bpe, data, offs, L, S, kw, spans, dev, out="numpy", pad_id=None):
    """encode_windows; without a GPU through the device C entry on host memory."""
    if not dev:
        return windows_abi(bpe, data, offs, L, S, PAD_FROM_MODEL if pad_id is None else pad_id, kw, spans)
    return bpe.encode_windows(data, offs, max_length=L, stride=S, pad_id=pad_id, with_spans=spans, out=out, **kw)


def check_against_packed(bpe, m, data, offs, kws, KS, dev, spans=True, pad_id=None, seed=None, outs=None):
    """encode_windows == the definition over encode_packed's ids (and spans) for every kw and (K, S), L = K + bos + eos.
    Returns the packed (ids, offsets) and the number of calls checked."""
    _, mpad, bid, eid = PG._special(m)
    pad = mpad if pad_id is None else pad_id
    offs = np.asarray(offs, dtype=np.uint64)
    drop = {k: v for k, v in kws[0].items() if k == "dropout_prob"} if kws else {}

    def fresh():
        if seed is not None:
            bpe.dropout_seed(seed)
    fresh()
    if spans:
        ids, oo, sp = bpe.encode_packed(data, offs, with_spans=True, **drop)
    else:
        (ids, oo), sp = bpe.encode_packed(data, offs, **drop), None
    n_checked = 0
    for kw in kws:
        be = int(kw.get("bos", False)) + int(kw.get("eos", False))
        for K, S in KS:
            L = K + be
            want = [x.cpu().numpy() if x is not None else None for x in
                    windows_ref(ids, oo, L, S, bid, eid, pad, kw.get("bos", False), kw.get("eos", False),
                                kw.get("reverse", False), sp, offs)]
            for out in (outs or (["numpy"] + (["torch", "cuda"] if dev else []))):
                fresh()
                got = call_windows(bpe, data, offs, L, S, kw, spans, dev, out, pad_id)
                assert len(got) == (5 if spans else 4)
                if dev and out != "numpy":
                    import torch
                    assert all(isinstance(x, torch.Tensor) and x.is_cuda == (out == "cuda") for x in got)
                g = [PG._np(x) for x in got]
                assert g[0].dtype == np.int32 and all(x.dtype == np.int64 for x in g[1:4]), [x.dtype for x in g]
                assert g[0].shape == want[0].shape, (kw, K, S, g[0].shape, want[0].shape)
                for a, b, what in zip(g[:4], want[:4], ("ids", "lengths", "sentence", "start")):
                    assert np.array_equal(a, b), (what, kw, K, S)
                if spans:
                    assert g[4].shape == g[0].shape + (2,)
                    if dev and out == "numpy":
                        assert g[4].dtype == np.uint64
                    assert np.array_equal(g[4].astype(np.int64), want[4]), (kw, K, S)
                n_checked += 1
    return ids, oo, n_checked


def _w1(bpe):
    """A word of exactly one id, so that a sentence of m of them has m ids."""
    for w in b" ".join(_cases.zipf_sentences(40, seed=4)).split():
        if PG._word_ids(bpe, w) == 1:
            return w
    raise AssertionError("no one-id word")


def _of(word, m):
    return b" ".join([word] * m)


# ---- bodies shared with the emulator test --------------------------------------------------------------------------
def check_flags(oracle, n, dev=False, kws=KWS):
    """Every bos / eos / reverse combination, ids and spans, at K = 1 (S = 0), K = 2 with step 1, K = 5 with S = 0, 2
    and K - 1, K = 16 with S = 7 and K above every sentence, over a batch of n sentences; a subset against the oracle's
    id lists."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    sents = PG._mix(n, seed=n)
    data, offs = _pack(sents)
    ids, oo = bpe.encode_packed(data, offs)
    longest = int(np.diff(oo.astype(np.int64)).max()) if n else 0
    KS = [(1, 0), (2, 1), (5, 0), (5, 2), (5, 4), (16, 7), (longest + 3, 2)]
    for kw in kws:
        check_against_packed(bpe, m, data, offs, [kw], KS, dev, spans=True, outs=["numpy"])
    check_against_packed(bpe, m, data, offs, kws[::3], KS[::2], dev, spans=False, outs=["numpy"])
    _, pad, bid, eid = PG._special(m)
    content = oracle.encoder(m).encode(sents)
    for kw in (KWS[0], KWS[-1]):
        be = int(kw["bos"]) + int(kw["eos"])
        for K, S in ((3, 1), (7, 0)):
            g = call_windows(bpe, data, offs, K + be, S, kw, False, dev)
            want = windows_from_lists(content, K + be, S, bid, eid, pad, **kw)
            for a, b in zip(g, want):
                assert np.array_equal(PG._np(a), b), (kw, K, S)


def check_count_edges(oracle, dev=False):
    """Sentences of 0, K, K + 1, K + D and K + D + 1 ids (1, 1, 2, 2 and 3 windows) for several (K, S), the step-1 and
    K = 1 extremes included, among sentences with many windows."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    w1 = _w1(bpe)
    for K, S in ((1, 0), (2, 1), (4, 0), (6, 3), (9, 8), (13, 5)):
        D = K - S
        counts = [0, K, K + 1, K + D, K + D + 1, 1, 3 * K + 2]
        sents = [_of(w1, c) for c in counts] + [b"ab " + _of(w1, K + D) + b" \xff", b""]
        data, offs = _pack(sents)
        _, oo = bpe.encode_packed(data, offs)
        assert np.diff(oo.astype(np.int64))[:7].tolist() == counts
        for kw in (KWS[0], KWS[3], KWS[5], KWS[6]):
            be = int(kw["bos"]) + int(kw["eos"])
            got = call_windows(bpe, data, offs, K + be, S, kw, False, dev)
            rows = np.bincount(PG._np(got[2]), minlength=len(sents))
            assert rows[:5].tolist() == [1, 1, 2, 2, 3], (K, S, rows.tolist())
        check_against_packed(bpe, m, data, offs, KWS, [(K, S)], dev, outs=["numpy"])


def check_many_rows(oracle, n, dev=False):
    """Tiles whose rows far outnumber their sentences: n sentences of many ids at K = 6 with step 1 and 2 (about 100
    rows per sentence, several gather tiles per sentence), and a width of one cell (K = 1)."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    zc = _cases.zipf()
    sents = zc.sentences(n, 400, seed=9)
    data, offs = _pack(sents)
    _, oo = bpe.encode_packed(data, offs)
    assert np.diff(oo.astype(np.int64)).min() > 20
    _, _, k = check_against_packed(bpe, m, data, offs, [KWS[0], KWS[-1], KWS[5]], [(6, 5), (6, 4), (1, 0)], dev,
                                   outs=["numpy"])
    got = call_windows(bpe, data, offs, 6, 5, {}, False, dev)
    assert PG._np(got[0]).shape[0] > 20 * n


def check_long(oracle, dev=False):
    """A word of more than LONG_W slots (the block kernel) cut by many windows, and a long sentence (about 1 MB with
    dev, 30 KB without)."""
    m = SG._model(oracle, _cases.dirty_zipf_text(60_000), 900, 0.95)
    bpe = SG._bpe(m)
    zc = _cases.zipf()
    long_word = b"".join(zc.sentences(40, 60, seed=6)).replace(b" ", b"")
    big = long_word[:700] * 2
    n_big = PG._word_ids(bpe, big)
    assert len(big) > 600 and n_big > 20
    data, offs = _pack([big, b"ab " + big + b" cd", big[:520], b"x"])
    check_against_packed(bpe, m, data, offs, KWS[::3], [(7, 3), (n_big - 1, 0), (n_big // 2, n_big // 2 - 1)], dev,
                         outs=["numpy"])
    size = 1_000_000 if dev else 30_000
    text = b" ".join(zc.sentences(size // 60, 60, seed=8))[:size]
    data, offs = _pack([text, b"", b"ab cd " + big])
    check_against_packed(bpe, m, data, offs, [KWS[0], KWS[-1]], [(510, 128), (61, 0)], dev,
                         outs=["numpy"] + (["cuda"] if dev else []))


def check_content(oracle, dev=False):
    """<UNK> runs, multi-byte and invalid UTF-8 (their spans too), with offsets[0] > 0, against encode_packed and the
    oracle's id lists."""
    m = SG._model(oracle, _cases.dirty_zipf_text(60_000), 900, 0.95)
    bpe = SG._bpe(m)
    sents = SG.ADVERSARIAL + list(_cases.EDGE_SENTENCES) + ["日本語 ёжик ☃☃☃ \U0001F600ab".encode() * 5]
    data, offs = _pack(sents)
    ids, _, _ = check_against_packed(bpe, m, data, offs, KWS, [(1, 0), (3, 1), (8, 5)], dev, outs=["numpy"])
    assert (ids == PG._special(m)[0]).any()   # <UNK> occurs
    shift = 37
    data2, offs2 = b"\xe2\x96" * shift + data + b"\xff" * shift, offs + np.uint64(2 * shift)
    check_against_packed(bpe, m, data2, offs2, KWS[::2], [(4, 2)], dev, outs=["numpy"])
    _, pad, bid, eid = PG._special(m)
    content = oracle.encoder(m).encode(sents)
    for kw in KWS[::3]:
        be = int(kw["bos"]) + int(kw["eos"])
        g = call_windows(bpe, data, offs, 4 + be, 1, kw, False, dev)
        for a, b in zip(g, windows_from_lists(content, 4 + be, 1, bid, eid, pad, **kw)):
            assert np.array_equal(PG._np(a), b), kw


def _unrow(row, n, bos, eos, reverse):
    """The content of a row of length n."""
    r = list(row[:n])
    r = r[::-1] if reverse else r
    return r[int(bos):n - int(eos)]


def check_equivalences(oracle, dev=False):
    """1. No sentence above K ids: the windows are encode_padded's rows for any S, sentence = arange(N), start = 0.
    2. The first window of every sentence is its encode_padded row.  3. The windows without their overlaps rebuild every
    sentence's encode_packed ids."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    sents = PG._mix(300, seed=7)
    data, offs = _pack(sents)
    ids, oo = bpe.encode_packed(data, offs)
    n = len(sents)
    cnt = np.diff(oo.astype(np.int64))
    for kw in (KWS[0], KWS[-1], KWS[3], KWS[4]):
        be = int(kw["bos"]) + int(kw["eos"])
        for K, Ss in ((int(cnt.max()), (0, int(cnt.max()) - 1)), (int(cnt.max()) + 4, (3,))):
            L = K + be
            pad_rows = [PG._np(x) for x in bpe.encode_padded(data, offs, max_length=L, with_spans=True, **kw)]
            for S in Ss:
                g = [PG._np(x) for x in call_windows(bpe, data, offs, L, S, kw, True, dev)]
                assert np.array_equal(g[0], pad_rows[0]) and np.array_equal(g[1], pad_rows[1]), (kw, K, S)
                assert np.array_equal(g[4], pad_rows[2]), (kw, K, S)
                assert np.array_equal(g[2], np.arange(n)) and not g[3].any()
        for K, S in ((3, 0), (5, 2), (8, 7)):
            L = K + be
            g = [PG._np(x) for x in call_windows(bpe, data, offs, L, S, kw, True, dev)]
            pad_rows = [PG._np(x) for x in bpe.encode_padded(data, offs, max_length=L, with_spans=True, **kw)]
            first = np.searchsorted(g[2], np.arange(n))
            assert np.array_equal(g[2][first], np.arange(n)) and not g[3][first].any()
            assert np.array_equal(g[0][first], pad_rows[0]) and np.array_equal(g[1][first], pad_rows[1]), (kw, K, S)
            assert np.array_equal(g[4][first], pad_rows[2]), (kw, K, S)
            rebuilt = [[] for _ in range(n)]
            for r in range(g[0].shape[0]):
                c = _unrow(g[0][r], g[1][r], kw["bos"], kw["eos"], kw["reverse"])
                i = g[2][r]
                assert g[3][r] == len(rebuilt[i]) - (S if rebuilt[i] else 0)
                rebuilt[i] += c[S:] if rebuilt[i] else c
            for i in range(n):
                assert rebuilt[i] == ids[oo[i]:oo[i + 1]].tolist(), (kw, K, S, i)


def check_dropout(oracle, p, dev=False):
    """After the same dropout_seed the windows are those of encode_packed's draws; two successive calls advance the
    sentence counter exactly as two encode_packed calls do."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    data, offs = _pack(PG._mix(400, seed=5))
    for kw in (KWS[0], KWS[-1], KWS[5]):
        check_against_packed(bpe, m, data, offs, [dict(kw, dropout_prob=p)], [(4, 1), (9, 0)], dev,
                             spans=kw["reverse"], seed=41, outs=["numpy"])
    bpe.dropout_seed(8)
    a = [bpe.encode_packed(data, offs, dropout_prob=p) for _ in range(2)]
    _, pad, bid, eid = PG._special(m)
    bpe.dropout_seed(8)
    b = [call_windows(bpe, data, offs, 6, 2, dict(dropout_prob=p), False, dev) for _ in range(2)]
    for (ids, oo), got in zip(a, b):
        want = windows_ref(ids, oo, 6, 2, bid, eid, pad)
        for x, y in zip(got, want[:4]):
            assert np.array_equal(PG._np(x), y.numpy())
    assert not np.array_equal(a[0][0], a[1][0])


def check_inputs(oracle, dev=False):
    """offsets[0] > 0, empty batches, all-empty sentences; with dev also bytes, numpy, CPU and CUDA torch inputs with
    numpy, CPU and CUDA offsets, and every out."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    sents = PG._mix(120, seed=21)
    data, offs = _pack(sents)
    shift = 11
    check_against_packed(bpe, m, b"\x00ab " * shift + data + b" zz", offs + np.uint64(4 * shift), KWS[::3],
                         [(5, 2)], dev)
    empty = np.zeros(1, dtype=np.uint64)
    for kw in (KWS[0], KWS[-1]):
        for spans in (False, True):
            g = call_windows(bpe, b"", empty, 5, 1, kw, spans, dev)
            assert PG._np(g[0]).shape == (0, 5) and all(PG._np(x).shape == (0,) for x in g[1:4])
            if spans:
                assert PG._np(g[4]).shape == (0, 5, 2)
    data0, offs0 = _pack([b"", b" ", b"\t\n", b""] * 70)
    g = call_windows(bpe, data0, offs0, 3, 2, {}, True, dev)
    assert PG._np(g[0]).shape == (280, 3) and not PG._np(g[1]).any()
    check_against_packed(bpe, m, data0, offs0, KWS, [(1, 0), (2, 1)], dev, outs=["numpy"])
    if not dev:
        return
    import torch
    _, pad, bid, eid = PG._special(m)
    ids, oo, sp = bpe.encode_packed(data, offs, with_spans=True)
    want = [x.numpy() for x in windows_ref(ids, oo, 9, 3, bid, eid, pad, True, False, True, sp, offs)]
    inputs = [data, np.frombuffer(data, dtype=np.uint8), torch.frombuffer(bytearray(data), dtype=torch.uint8),
              torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()]
    offsets = [offs, torch.from_numpy(offs.astype(np.int64)), torch.from_numpy(offs.astype(np.int64)).cuda()]
    for d in inputs:
        for o in offsets:
            for out in ("numpy", "torch", "cuda"):
                g = bpe.encode_windows(d, o, 9, stride=3, bos=True, reverse=True, with_spans=True, out=out)
                for x, y in zip(g, want):
                    assert np.array_equal(PG._np(x).astype(np.int64), y.astype(np.int64)), (type(d), type(o), out)


def check_errors(oracle, dev=False):
    """Argument errors with encode_padded's texts and types, a model without <PAD>, <BOS> / <EOS>, and the C entry's
    own checks."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    data, offs = _pack([b"ab cd", b"e"])
    call = lambda **k: bpe.encode_windows(data, offs, **k)
    for bad, kw in ((0, {}), (-3, {}), (2, dict(bos=True, eos=True)), (1, dict(bos=True)), (2**31, {})):
        with pytest.raises(ValueError, match="max_length must be at least bos \\+ eos \\+ 1, and below 2\\^31"):
            call(max_length=bad, **kw)
    for bad in (3.0, "8", True, None):
        with pytest.raises(TypeError, match="max_length must be an int"):
            call(max_length=bad)
    for bad, L, kw in ((-1, 4, {}), (4, 4, {}), (5, 4, {}), (2, 4, dict(bos=True, eos=True)), (1, 2, dict(eos=True))):
        with pytest.raises(ValueError, match="stride must be at least 0 and below max_length - bos - eos"):
            call(max_length=L, stride=bad, **kw)
    for bad in (1.0, "1", True, None):
        with pytest.raises(TypeError, match="stride must be an int"):
            call(max_length=4, stride=bad)
    for p in (-0.1, 1.5):
        with pytest.raises(ValueError, match="dropout_prob value must be in the range"):
            call(max_length=4, dropout_prob=p)
    with pytest.raises(ValueError, match="pad_id must fit in int32"):
        call(max_length=4, pad_id=2**31)
    with pytest.raises(TypeError, match="pad_id must be an int"):
        call(max_length=4, pad_id=1.5)
    with pytest.raises(ValueError, match="out must be"):
        call(max_length=4, out="list")
    m2 = SG._model(oracle, _cases.dirty_zipf_text(60_000), 700, pad=-1, unk=1, bos=2, eos=3)
    b2 = SG._bpe(m2)
    with pytest.raises(ValueError, match="Can't pad: model was trained without <PAD>"):
        call_windows(b2, data, offs, 6, 1, {}, False, dev)
    check_against_packed(b2, m2, data, offs, KWS[::3], [(3, 1)], dev, spans=False, pad_id=0, outs=["numpy"])
    for pad_id in (-100, 2**31 - 1, -2**31):
        check_against_packed(bpe, m, data, offs, [KWS[-1]], [(2, 1)], dev, spans=False, pad_id=pad_id, outs=["numpy"])
    m3 = tmp_model_path("orc")
    oracle.train(synth.readme_corpus(n_lines=200), m3, 100, 1.0, pad=0, unk=1, bos=-1, eos=-1)
    b3 = SG._bpe(m3)
    with pytest.raises(ValueError, match="Can't add <BOS> token. Model was trained without it."):
        call_windows(b3, data, offs, 4, 0, dict(bos=True), False, dev)
    with pytest.raises(ValueError, match="Can't add <EOS> token. Model was trained without it."):
        call_windows(b3, data, offs, 4, 0, dict(eos=True), False, dev)
    # the C entries check width and stride themselves
    Lb = _lib.lib()
    enc = Lb.yttm_api_device_encoder(bpe._h)
    ctx = Lb.yttm_api_device_context(bpe._h)
    buf = C.create_string_buffer(data)
    p = [C.c_void_p() for _ in range(5)]
    rows = C.c_uint64(7)
    for w, s, b, e, what in ((0, 0, 0, 0, b"width"), (2, 0, 1, 1, b"width"), (2**31, 0, 0, 0, b"width"),
                             (4, 4, 0, 0, b"stride"), (4, 3, 1, 0, b"stride")):
        assert Lb.yttm_enc_run_windows_device(enc, C.cast(buf, C.c_void_p), offs.ctypes.data, len(data), 2, b, e, 0,
                                              0.0, 0, 0, w, s, 0, 0, *[C.byref(x) for x in p], C.byref(rows)) == 1
        assert what + b" must be" in Lb.yttm_last_error(ctx) and rows.value == 0
    assert Lb.yttm_enc_run_windows_device(None, None, None, 0, 0, 0, 0, 0, 0.0, 0, 0, 4, 0, 0, 0, None, None, None,
                                          None, None, None) == 1
    assert b"null encoder handle" in Lb.yttm_last_error(None)


# ---- GPU tests -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 255, 256, 257, 600])
def test_flags(product, oracle, n):
    check_flags(oracle, n, dev=True)


def test_count_edges(product, oracle):
    check_count_edges(oracle, dev=True)


def test_many_rows(product, oracle):
    check_many_rows(oracle, 300, dev=True)


def test_long(product, oracle):
    check_long(oracle, dev=True)


def test_content(product, oracle):
    check_content(oracle, dev=True)


def test_equivalences(product, oracle):
    check_equivalences(oracle, dev=True)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout(product, oracle, p):
    check_dropout(oracle, p, dev=True)


def test_inputs(product, oracle):
    check_inputs(oracle, dev=True)


def test_errors(product, oracle):
    check_errors(oracle, dev=True)


def test_too_large_is_an_error(product, oracle):
    """A request over 2^40 cells (one sentence of about 3 M ids, step 1, L = 2^21) and one that cannot be reserved:
    the library's error, then the same BPE keeps working."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    w1 = _w1(bpe)
    data, offs = _pack([_of(w1, 3_000_000)])
    L = 2**21
    assert (3_000_000 - L + 2) * L > 2**40
    with pytest.raises(ValueError, match="rows do not fit in device memory"):
        bpe.encode_windows(data, offs, L, stride=L - 1, out="cuda")
    small, soffs = _pack(PG._mix(100, seed=2))
    with pytest.raises(ValueError, match="rows do not fit in device memory"):   # 100 x 2^31 - 1 cells of 20 bytes
        bpe.encode_windows(small, soffs, 2**31 - 1, with_spans=True, out="cuda")
    check_against_packed(bpe, m, small, soffs, [KWS[-1]], [(5, 2), (11, 0)], True)


def test_bench_shape(product, oracle):
    """The benchmark's batch (1 M x 128 B Zipf sentences): at L = 16, S = 4 and L = 24, S = 21 with every flag, the
    whole result equals the definition over encode_packed(out="cuda"), computed on the device with torch; at L = the
    longest row no sentence has a second window, so the windows are encode_padded's rows even at step 1."""
    import torch
    import youtokentome_b200 as yttm
    m = EM._model(oracle)
    bpe = yttm.BPE(m)
    buf, offs = synth.FastZipf(200_000, 1.07, 1234).packed_sentences(1_000_000, 128, seed=4321)
    data, offs = np.frombuffer(bytes(buf), dtype=np.uint8), np.asarray(offs, dtype=np.uint64)
    ids, oo = bpe.encode_packed(data, offs, out="cuda")
    _, pad, bid, eid = PG._special(m)
    for L, S, kw in ((16, 4, {}), (24, 21, dict(bos=True, eos=True, reverse=True))):
        g = bpe.encode_windows(data, offs, L, stride=S, out="cuda", **kw)
        want = windows_ref(ids, oo, L, S, bid, eid, pad, **kw)
        assert g[0].shape == want[0].shape and g[0].shape[0] > 1_000_000
        assert all(torch.equal(a, b) for a, b in zip(g, want[:4]))
        del g, want
    longest = int((oo[1:] - oo[:-1]).max())
    g = bpe.encode_windows(data, offs, longest, stride=longest - 1, out="cuda")
    p = bpe.encode_padded(data, offs, max_length=longest, out="cuda")
    assert torch.equal(g[0], p[0]) and torch.equal(g[1], p[1])
    assert torch.equal(g[2], torch.arange(1_000_000, device="cuda")) and not bool(g[3].any())
    del g, p
    torch.cuda.empty_cache()

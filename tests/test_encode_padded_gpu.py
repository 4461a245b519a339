"""Padded rows of device encode (`BPE.encode_padded`, yttm_enc_run_padded*, emit_padded_kernel in
youtokentome_b200/csrc/encode.cu).  The expectation is the definition of yttm_enc_run_padded applied with torch to
encode_packed's output for the same call (encode_packed is pinned to the oracle elsewhere); a subset is also built from
the oracle's ids directly.  The check bodies take `dev`: True also runs the CUDA interfaces, L = None through the
Python surface and the sizes only a GPU finishes quickly; tests/test_encode_padded_emul_cpu.py runs them with False
under the SIMT emulator, where L = None goes through the device C entry on host memory."""
import ctypes as C
import os

import numpy as np
import pytest

import _cases
import test_encode_emit_gpu as EM
import test_encode_spans_gpu as SG
from _bind import _pack, tmp_model_path
from youtokentome_b200 import _lib, synth

pytestmark = pytest.mark.gpu

KWS = SG.KWS
TILE = 256
PAD_FROM_MODEL = -2**63


# ---- the definition ------------------------------------------------------------------------------------------------
def padded_ref(ids, oo, L, bos_id, eos_id, pad, bos=False, eos=False, reverse=False, spans=None, offs=None):
    """Rows of encode_packed's output (ids / oo / spans of a call with bos = eos = reverse = False) as torch tensors on
    the ids' device: (ids [N, L] int32, lengths [N] int64, spans [N, L, 2] int64 or None).  L = None: the longest row."""
    import torch
    t = lambda x: x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x).astype(np.int64))
    ids, oo = t(ids).to(torch.int64), t(oo).to(torch.int64)
    dev, n, be = ids.device, oo.numel() - 1, int(bos) + int(eos)
    cnt = oo[1:] - oo[:-1]
    if L is None:
        L = int((cnt + be).max()) if n else 0
    lens = torch.clamp(cnt, max=L - be) + be
    col = torch.arange(L, device=dev)[None, :]
    last = lens[:, None] - 1
    p = last - col if reverse else col.expand(n, L)          # place in the unreversed row
    valid = col < lens[:, None]
    is_bos = valid & (p == 0) if bos else torch.zeros_like(valid)
    is_eos = valid & (p == last) if eos else torch.zeros_like(valid)
    content = valid & ~is_bos & ~is_eos
    src = (oo[:-1, None] + p - int(bos)).clamp(0, max(ids.numel() - 1, 0))
    out = torch.full((n, L), pad, dtype=torch.int64, device=dev)
    if ids.numel():
        out = torch.where(content, ids[src], out)
    out = torch.where(is_bos, torch.full_like(out, bos_id), out)
    out = torch.where(is_eos, torch.full_like(out, eos_id), out)
    sp = None
    if spans is not None:
        spans, o = t(spans).to(torch.int64).reshape(-1, 2), t(offs).to(torch.int64).to(dev)
        lo, hi = o[:-1, None, None].expand(n, L, 2), o[1:, None, None].expand(n, L, 2)
        sp = hi.clone()
        if spans.shape[0]:
            sp = torch.where(content[..., None], spans[src], sp)
        sp = torch.where(is_bos[..., None], lo, sp)
    return out.to(torch.int32), lens, sp


def rows_from_lists(content, L, bos_id, eos_id, pad, bos, eos, reverse):
    """The definition in plain Python over per-sentence id lists (the oracle's)."""
    be = int(bos) + int(eos)
    if L is None:
        L = max([len(c) + be for c in content], default=0)
    out, lens = np.full((len(content), L), pad, np.int32), np.zeros(len(content), np.int64)
    for i, c in enumerate(content):
        row = ([bos_id] if bos else []) + list(c)[:L - be] + ([eos_id] if eos else [])
        row = row[::-1] if reverse else row
        out[i, :len(row)] = row
        lens[i] = len(row)
    return out, lens


# ---- library calls -------------------------------------------------------------------------------------------------
def _np(x):
    if type(x).__module__.startswith("torch"):
        return x.cpu().numpy()
    return np.asarray(x)


def padded_abi(bpe, data, offs, width, pad, kw, spans):
    """yttm_api_encode_padded_device on HOST memory: the emulator's device memory is host memory, so this is how the
    emulator reaches the width-0 (longest row) path."""
    L = _lib.lib()
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    raw = bytes(data)
    n = len(offs) - 1
    first = int(offs[0]) if n >= 0 else 0
    buf = C.create_string_buffer(raw[first:] + b"\0")
    p = [C.c_void_p() for _ in range(3)]
    w = C.c_uint32(0)
    rc = L.yttm_api_encode_padded_device(bpe._h, C.cast(buf, C.c_void_p), offs.ctypes.data,
                                         int(offs[-1]) - first, n, int(kw.get("bos", False)), int(kw.get("eos", False)),
                                         int(kw.get("reverse", False)), float(kw.get("dropout_prob", 0.0)), width, pad,
                                         int(spans), C.byref(p[0]), C.byref(p[1]), C.byref(p[2]), C.byref(w))
    if rc != 0:
        raise ValueError(L.yttm_api_last_error(bpe._h).decode())
    W = w.value

    def arr(ptr, count, ct, shape):
        if count == 0:
            return np.zeros(shape, dtype=np.dtype(ct))
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ct)), shape=(count,)).copy().reshape(shape)
    res = [arr(p[0], n * W, C.c_int32, (n, W)), arr(p[1], n, C.c_int64, (n,))]
    if spans:
        res.append(arr(p[2], 2 * n * W, C.c_uint64, (n, W, 2)))
    return tuple(res)


def call_padded(bpe, data, offs, L, kw, spans, dev, out="numpy", pad_id=None):
    """encode_padded; L = None without a GPU goes through the device C entry on host memory."""
    if L is None and not dev:
        return padded_abi(bpe, data, offs, 0, PAD_FROM_MODEL if pad_id is None else pad_id, kw, spans)
    return bpe.encode_padded(data, offs, max_length=L, pad_id=pad_id, with_spans=spans, out=out, **kw)


def _special(m):
    from _bind import read_model
    return read_model(m)[2]   # (unk, pad, bos, eos)


def check_against_packed(bpe, m, data, offs, kws, Ls, dev, spans=True, pad_id=None, seed=None, outs=None):
    """encode_padded == the definition over encode_packed's ids (and spans) for every kw and L."""
    _, mpad, bid, eid = _special(m)
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
        for L in Ls:
            if L is not None and L < max(1, be):
                continue
            want = padded_ref(ids, oo, L, bid, eid, pad, kw.get("bos", False), kw.get("eos", False),
                              kw.get("reverse", False), sp, offs)
            for out in (outs or (["numpy"] + (["torch", "cuda"] if dev else []))):
                fresh()
                got = call_padded(bpe, data, offs, L, kw, spans, dev, out, pad_id)
                assert len(got) == (3 if spans else 2)
                if out != "numpy":
                    import torch
                    assert all(isinstance(x, torch.Tensor) and x.is_cuda == (out == "cuda") for x in got)
                g = [_np(x) for x in got]
                assert g[0].dtype == np.int32 and g[1].dtype == np.int64
                assert g[0].shape == tuple(want[0].shape), (kw, L, g[0].shape, tuple(want[0].shape))
                assert np.array_equal(g[1], want[1].cpu().numpy()), (kw, L)
                assert np.array_equal(g[0], want[0].cpu().numpy()), (kw, L)
                if spans:
                    assert g[2].shape == g[0].shape + (2,)
                    assert np.array_equal(g[2].astype(np.int64), want[2].cpu().numpy()), (kw, L)
                n_checked += 1
    return ids, oo, n_checked


def _lengths_around(oo, k=3):
    """L values at exactly some rows' content length and one on either side."""
    cnt = np.diff(np.asarray(oo, dtype=np.int64))
    pick = sorted(set(cnt[cnt > 1].tolist()))
    out = set()
    for c in pick[len(pick) // 2:len(pick) // 2 + 1] + pick[-1:] + pick[:1]:
        out |= {c - 1, c, c + 1}
    return sorted(x for x in out if x >= 1)[:3 * k]


def _mix(n, seed):
    """n sentences: Zipf sentences, the edge cases, the adversarial UTF-8, empty and all-space sentences."""
    z = _cases.zipf_sentences(max(n, 40), seed=seed)
    extra = _cases.EDGE_SENTENCES + SG.ADVERSARIAL + [b"", b" ", b"\t\n  ", b"", b"   "]
    pool = []
    for i in range(max(n, 1)):
        pool.append(extra[(i // 7) % len(extra)] if i % 7 == 3 else z[i % len(z)])
    return pool[:n]


# ---- bodies shared with the emulator test --------------------------------------------------------------------------
def check_flags_and_widths(oracle, n, dev=False, kws=KWS):
    """Every bos / eos / reverse combination with L = None, 1, bos + eos, a row's length and one on either side, and
    longer than every row, over a batch of n sentences; a subset against the oracle's ids directly."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    sents = _mix(n, seed=n)
    data, offs = _pack(sents)
    ids, oo = bpe.encode_packed(data, offs)
    longest = int(np.diff(oo.astype(np.int64)).max()) if n else 0
    for kw in kws:
        be = int(kw["bos"]) + int(kw["eos"])
        Ls = [None, 1, be] + [c + be for c in _lengths_around(oo)] + [longest + be + 5]
        check_against_packed(bpe, m, data, offs, [kw], Ls, dev, spans=kw["reverse"] or n <= 300)
    _, pad, bid, eid = _special(m)
    content = oracle.encoder(m).encode(sents)
    for kw in (KWS[0], KWS[-1]):
        for L in (None, 5):
            g = call_padded(bpe, data, offs, L, kw, False, dev)
            want = rows_from_lists(content, L, bid, eid, pad, **kw)
            assert np.array_equal(_np(g[0]), want[0]) and np.array_equal(_np(g[1]), want[1]), (kw, L)


def _word_ids(bpe, word):
    ids, _ = bpe.encode_packed(word, np.array([0, len(word)], dtype=np.uint64))
    return len(ids)


def check_cuts_inside_words(oracle, dev=False):
    """Every cut of sentences whose words have 1, 2, 3 and more ids (after id0 / id1 / id2 of a record, inside a word of
    more than 3 ids), cuts inside a word of more than 512 slots (the block kernel), and with dev a 100 KB and a 1 MB
    word at L = 128."""
    m = SG._model(oracle, _cases.dirty_zipf_text(60_000), 900, 0.95)
    bpe = SG._bpe(m)
    zc = _cases.zipf()
    long_word = b"".join(zc.sentences(40, 60, seed=6)).replace(b" ", b"")
    words = b" ".join(_cases.zipf_sentences(30, seed=4)).split() + [long_word[:30], long_word[:90]]
    by_n = {}
    for w in words:
        by_n.setdefault(min(_word_ids(bpe, w), 5), w)
    assert {1, 2, 3, 5} <= set(by_n), sorted(by_n)
    sents = [b" ".join([by_n[k] for k in (1, 2, 3, 5)]), b" ".join([by_n[5], by_n[3], by_n[1], by_n[2], by_n[5]]),
             by_n[5] + b" " + by_n[5], b"", by_n[2]]
    data, offs = _pack(sents)
    _, oo = bpe.encode_packed(data, offs)
    longest = int(np.diff(oo.astype(np.int64)).max())
    for kw in (KWS[0], KWS[3], KWS[5], KWS[6]):
        be = int(kw["bos"]) + int(kw["eos"])
        check_against_packed(bpe, m, data, offs, [kw], list(range(max(1, be), longest + be + 2)), dev, outs=["numpy"])
    big = long_word[:700] * 2   # more than 512 slots
    assert len(big) > 600
    n_big = _word_ids(bpe, big)
    assert n_big > 8
    data, offs = _pack([big, b"ab " + big + b" cd", big[:520], b"x"])
    Ls = [1, 2, 3, 4, 5, n_big // 2, n_big - 1, n_big, n_big + 1, n_big + 5]
    check_against_packed(bpe, m, data, offs, KWS[::3], Ls, dev, outs=["numpy"])
    if dev:
        rng = np.random.default_rng(3)
        giant = [bytes(rng.choice(np.frombuffer(b"abcdefghij", dtype=np.uint8), size=k).tolist()) for k in
                 (100_000, 1_000_000)]
        data, offs = _pack([giant[0], b"ab " + giant[1] + b" cd", b"ab cd", giant[1][:777]])
        check_against_packed(bpe, m, data, offs, KWS[::2], [128], dev, outs=["numpy", "cuda"])


def check_spans_shift(oracle, dev=False):
    """Spans for every flag combination with offsets[0] > 0: kept ids as encode_packed(with_spans=True), pads
    [end, end)."""
    m = SG._model(oracle, _cases.dirty_zipf_text(60_000), 900)
    bpe = SG._bpe(m)
    sents = _mix(300, seed=12)
    data, offs = _pack(sents)
    shift = 37
    data = b"\xe2\x96" * shift + data + b"\xff" * shift
    offs = offs + np.uint64(2 * shift)
    _, oo = bpe.encode_packed(data, offs)
    for kw in KWS:
        be = int(kw["bos"]) + int(kw["eos"])
        check_against_packed(bpe, m, data, offs, [kw], [None, max(1, be), 7 + be, 40], dev)


def check_dropout(oracle, p, dev=False):
    """After the same dropout_seed the rows are the padded packed output; two successive calls advance the sentence
    counter exactly as two encode_packed calls do."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    data, offs = _pack(_mix(400, seed=5))
    for kw in (KWS[0], KWS[-1], KWS[5]):
        check_against_packed(bpe, m, data, offs, [dict(kw, dropout_prob=p)], [None, 9, 30], dev, spans=kw["reverse"],
                             seed=41)
    bpe.dropout_seed(8)
    a = [bpe.encode_packed(data, offs, dropout_prob=p) for _ in range(2)]
    _, pad, bid, eid = _special(m)
    for L in (None, 12):
        bpe.dropout_seed(8)
        b = [call_padded(bpe, data, offs, L, dict(dropout_prob=p), False, dev) for _ in range(2)]
        for (ids, oo), got in zip(a, b):
            want = padded_ref(ids, oo, L, bid, eid, pad)
            assert np.array_equal(_np(got[0]), want[0].numpy()) and np.array_equal(_np(got[1]), want[1].numpy())
    assert not np.array_equal(a[0][0], a[1][0])


def check_pad_ids(oracle, dev=False):
    """The model's pad id, an explicit one, a model without <PAD> (an error without pad_id, fine with it), and custom
    special ids."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    data, offs = _pack(_mix(60, seed=3))
    for pad_id in (None, -100, 7, 2**31 - 1, -2**31):
        check_against_packed(bpe, m, data, offs, [KWS[0], KWS[-1]], [None, 6], dev, spans=False, pad_id=pad_id)
    m2 = SG._model(oracle, _cases.dirty_zipf_text(60_000), 700, pad=-1, unk=1, bos=2, eos=3)
    b2 = SG._bpe(m2)
    for L in (None, 6):
        with pytest.raises(ValueError, match="Can't pad: model was trained without <PAD>"):
            call_padded(b2, data, offs, L, {}, False, dev)
    check_against_packed(b2, m2, data, offs, KWS[::3], [None, 6], dev, spans=False, pad_id=0)
    m3 = SG._model(oracle, _cases.dirty_zipf_text(200_000), 3000, 0.95, pad=29, unk=1148, bos=2922, eos=4)
    b3 = SG._bpe(m3)
    assert _special(m3) == (1148, 29, 2922, 4)
    ids, _, _ = check_against_packed(b3, m3, data, offs, KWS, [None, 1, 2, 9], dev, spans=False)
    assert (ids == 1148).any()


def check_layouts(oracle, dev=False):
    """n_sent = 0 gives (0, L) / (0, 0); a batch of empty rows only; every row empty with L = None gives width 0
    (without bos / eos)."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    empty = np.zeros(1, dtype=np.uint64)
    for kw in (KWS[0], KWS[-1]):
        for spans in (False, True):
            g = call_padded(bpe, b"", empty, 5, kw, spans, dev)
            assert _np(g[0]).shape == (0, 5) and _np(g[1]).shape == (0,)
            g = call_padded(bpe, b"", empty, None, kw, spans, dev)
            assert _np(g[0]).shape == (0, 0) and _np(g[1]).shape == (0,)
    data, offs = _pack([b"", b" ", b"\t\n", b"\xe2\x96\x81 \xe2\x96\x81"] * 70)
    g = call_padded(bpe, data, offs, None, {}, True, dev)
    assert _np(g[0]).shape == (280, 0) and not _np(g[1]).any()
    check_against_packed(bpe, m, data, offs, KWS, [None, 2, 3], dev)


def check_chunks(oracle, monkeypatch, n_bytes, dev=False):
    """The host-buffer form over several chunks: every chunk's rows land in place."""
    m = SG._model(oracle, _cases.dirty_zipf_text(60_000), 900, 0.95)
    bpe = SG._bpe(m)
    monkeypatch.setenv("YTTM_ENC_CHUNK_MB", "1")
    data, offs = _pack(_cases.zipf().sentences(n_bytes // 100, 100, seed=11) + SG.ADVERSARIAL)
    check_against_packed(bpe, m, data, offs, [KWS[0], KWS[-1]], [23], dev, outs=["numpy"])
    L = _lib.lib()
    assert L.yttm_stage_ms(L.yttm_api_device_context(bpe._h), b"enc_chunks") >= 2


def check_errors(oracle, dev=False):
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    data, offs = _pack([b"ab cd", b"e"])
    for out in ["numpy"] + (["cuda"] if dev else []):
        call = lambda **k: bpe.encode_padded(data, offs, out=out, **k)
        for bad, kw in ((0, {}), (-3, {}), (1, dict(bos=True, eos=True)), (0, dict(bos=True))):
            with pytest.raises(ValueError, match="max_length must be at least 1 and at least bos \\+ eos"):
                call(max_length=bad, **kw)
        for bad in (3.0, "8", True):
            with pytest.raises(TypeError, match="max_length must be an int"):
                call(max_length=bad)
        for p in (-0.1, 1.5):
            with pytest.raises(ValueError, match="dropout_prob value must be in the range"):
                call(max_length=4, dropout_prob=p)
        with pytest.raises(ValueError, match="pad_id must fit in int32"):
            call(max_length=4, pad_id=2**31)
        with pytest.raises(TypeError, match="pad_id must be an int"):
            call(max_length=4, pad_id=1.5)
        with pytest.raises(ValueError, match="out must be"):
            bpe.encode_padded(data, offs, max_length=4, out="list")
    m2 = tmp_model_path("orc")
    oracle.train(synth.readme_corpus(n_lines=200), m2, 100, 1.0, pad=0, unk=1, bos=-1, eos=-1)
    b2 = SG._bpe(m2)
    with pytest.raises(ValueError, match="Can't add <BOS> token. Model was trained without it."):
        call_padded(b2, data, offs, 4, dict(bos=True), False, dev)
    with pytest.raises(ValueError, match="Can't add <EOS> token. Model was trained without it."):
        call_padded(b2, data, offs, None, dict(eos=True), False, dev)
    # the C entries check the width themselves
    Lb = _lib.lib()
    enc = Lb.yttm_api_device_encoder(bpe._h)
    ids, ln = np.zeros(8, np.int32), np.zeros(2, np.uint64)
    for w, b, e in ((0, 0, 0), (1, 1, 1), (2**31, 0, 0)):
        assert Lb.yttm_enc_run_padded(enc, data, offs.ctypes.data, 2, b, e, 0, 0.0, 0, 0, w, 0, ids.ctypes.data,
                                      ln.ctypes.data, None) == 1
        assert b"width must be" in Lb.yttm_last_error(Lb.yttm_api_device_context(bpe._h))
    assert Lb.yttm_enc_run_padded(enc, data, offs.ctypes.data, 2, 0, 0, 0, 0.0, 0, 0, 4, -5, ids.ctypes.data,
                                  ln.ctypes.data, None) == 0
    want = [min(4, len(bpe.encode_packed(s, np.array([0, len(s)], np.uint64))[0])) for s in (b"ab cd", b"e")]
    assert ln.tolist() == want
    assert all(ids.reshape(2, 4)[i, want[i]:].tolist() == [-5] * (4 - want[i]) for i in range(2))
    assert Lb.yttm_enc_run_padded(None, data, offs.ctypes.data, 2, 0, 0, 0, 0.0, 0, 0, 4, 0, None, None, None) == 1
    assert b"null encoder handle" in Lb.yttm_last_error(None)


# ---- GPU tests -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 255, 256, 257, 4000])
def test_flags_and_widths(product, oracle, n):
    check_flags_and_widths(oracle, n, dev=True, kws=KWS if n != 4000 else KWS[::3])


def test_cuts_inside_words(product, oracle):
    check_cuts_inside_words(oracle, dev=True)


def test_spans_shift(product, oracle):
    check_spans_shift(oracle, dev=True)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout(product, oracle, p):
    check_dropout(oracle, p, dev=True)


def test_pad_ids(product, oracle):
    check_pad_ids(oracle, dev=True)


def test_layouts(product, oracle):
    check_layouts(oracle, dev=True)


def test_chunks(product, oracle, monkeypatch):
    check_chunks(oracle, monkeypatch, 3_000_000, dev=True)


def test_errors(product, oracle):
    check_errors(oracle, dev=True)


def test_cuda_input_and_tensor_offsets(product, oracle):
    """CUDA torch input with int64 tensor offsets, every out."""
    import torch
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    data, offs = _pack(_mix(500, seed=21))
    ids, oo, sp = bpe.encode_packed(data, offs, with_spans=True)
    _, pad, bid, eid = _special(m)
    d_data = torch.tensor(list(data), dtype=torch.uint8).cuda()
    for d_offs in (torch.from_numpy(offs.astype(np.int64)).cuda(), torch.from_numpy(offs.astype(np.int64))):
        for L in (None, 17):
            want = padded_ref(ids, oo, L, bid, eid, pad, True, False, True, sp, offs)
            for out in ("numpy", "torch", "cuda"):
                g = bpe.encode_padded(d_data, d_offs, max_length=L, bos=True, reverse=True, with_spans=True, out=out)
                assert np.array_equal(_np(g[0]), want[0].numpy()) and np.array_equal(_np(g[1]), want[1].numpy())
                assert np.array_equal(_np(g[2]).astype(np.int64), want[2].numpy())


def test_too_large_is_an_error(product, oracle):
    """N x L that cannot be reserved on the device: the library's error, then the handle keeps working."""
    m = EM._model(oracle)
    bpe = SG._bpe(m)
    data, offs = _pack(_mix(100, seed=2))
    with pytest.raises(ValueError, match="rows do not fit in device memory"):
        bpe.encode_padded(data, offs, max_length=2**30, out="cuda")
    with pytest.raises(ValueError, match="rows do not fit in device memory"):
        bpe.encode_padded(data, offs, max_length=2**31 - 1, with_spans=True, out="cuda")
    check_against_packed(bpe, m, data, offs, [KWS[-1]], [None, 11], True)


def test_bench_shape(product, oracle):
    """The benchmark's batch (1 M x 128 B Zipf sentences) at L = 64 (many rows cut) and L = None: the whole [N, L]
    result equals the padded form of encode_packed(out="cuda"), computed on the device with torch."""
    import torch
    import youtokentome_b200 as yttm
    bpe = yttm.BPE(EM._model(oracle))
    buf, offs = synth.FastZipf(200_000, 1.07, 1234).packed_sentences(1_000_000, 128, seed=4321)
    data, offs = np.frombuffer(bytes(buf), dtype=np.uint8), np.asarray(offs, dtype=np.uint64)
    ids, oo = bpe.encode_packed(data, offs, out="cuda")
    _, pad, bid, eid = _special(EM._model(oracle))
    for L, kw in ((64, {}), (None, {}), (64, dict(bos=True, eos=True, reverse=True))):
        g = bpe.encode_padded(data, offs, max_length=L, out="cuda", **kw)
        want = padded_ref(ids, oo, L, bid, eid, pad, **kw)
        assert g[0].shape == want[0].shape
        assert torch.equal(g[0], want[0]) and torch.equal(g[1], want[1])
        if L == 64 and not kw:
            assert int((g[1] == 64).sum()) > 10_000   # many rows are cut
        del g, want
    torch.cuda.empty_cache()


def test_zzz_sanitizer_memcheck_padded(product):
    """compute-sanitizer memcheck over tools/sanitize_padded.py: no report; skips where the tool refuses the device."""
    import shutil
    import subprocess
    import sys
    from _bind import ROOT
    exe = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(exe):
        pytest.skip("compute-sanitizer is not installed")
    env = {k: v for k, v in os.environ.items() if not k.startswith(("YTTM_", "YT_EMU_"))}
    r = subprocess.run([exe, "--tool", "memcheck", sys.executable, os.path.join(ROOT, "tools", "sanitize_padded.py")],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    text = r.stdout.decode(errors="replace")
    if "Error: Device not supported" in text:
        pytest.skip("compute-sanitizer does not support this device here")
    assert "padded rows identical to the definition" in text, text[-1500:]
    assert "ERROR SUMMARY: 0 errors" in text, text[-1500:]

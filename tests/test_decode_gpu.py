"""Batch decode on the GPU (`BPE.decode_packed`, yttm_dec_run / yttm_dec_run_device) against the host `BPE.decode`
(itself checked against the reference by test_abi.py) and, at full size, against a numpy restatement of it.  The
bodies take `dev`: True runs the CUDA-tensor interfaces too; tests/test_decode_emul_cpu.py runs them with False under
the SIMT emulator, whose "device" memory is host memory."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

import _cases
from _bind import _pack, read_model, tmp_model_path
from _gpu import GpuEncoder
from youtokentome_b200 import synth

pytestmark = pytest.mark.gpu

SPACE = "▁".encode()


def _model(oracle, text, vocab, cov=1.0, **special):
    m = tmp_model_path("orc")
    oracle.train(text, m, vocab, cov, **special)
    return m


def _bpe(m):
    import youtokentome_b200 as yttm
    return yttm.BPE(m)


# ---- numpy oracle -------------------------------------------------------------------------------
def piece_table(bpe, model):
    """(flat piece bytes, start, length, leading-space flag) per id: id_to_subword(i) with a leading U+2581 turned into
    one space for non-special ids."""
    special = set(read_model(model)[2]) - {-1}
    pieces = []
    for i in range(bpe.vocab_size()):
        p = bpe.id_to_subword(i).encode()
        if i not in special and p.startswith(SPACE):
            p = b" " + p[len(SPACE):]
        pieces.append(p)
    lens = np.array([len(p) for p in pieces], dtype=np.int64)
    starts = np.zeros(len(pieces), dtype=np.int64)
    starts[1:] = np.cumsum(lens)[:-1]
    flat = np.frombuffer(b"".join(pieces), dtype=np.uint8)
    lead = np.array([p[:1] == b" " for p in pieces], dtype=bool)
    return flat, starts, lens, lead


def oracle_decode(tab, ids, offsets, ignore=()):
    """decode() of a packed batch of valid ids, vectorised: (text bytes, uint64 text offsets)."""
    flat, starts, lens, lead = tab
    offsets = np.asarray(offsets, dtype=np.int64)
    seen = np.asarray(ids, dtype=np.int64)[offsets[0]:offsets[-1]]
    sent = np.repeat(np.arange(len(offsets) - 1), np.diff(offsets))
    keep = ~np.isin(seen, np.asarray(sorted(ignore), dtype=np.int64))
    kid, ks = seen[keep], sent[keep]
    first = np.ones(len(ks), dtype=bool)
    first[1:] = ks[1:] != ks[:-1]
    strip = (first & lead[kid]).astype(np.int64)
    ln, st = lens[kid] - strip, starts[kid] + strip
    out_start = np.zeros(len(ln), dtype=np.int64)
    out_start[1:] = np.cumsum(ln)[:-1]
    idx = np.repeat(st - out_start, ln) + np.arange(int(ln.sum()), dtype=np.int64)
    per = np.bincount(ks, weights=ln, minlength=len(offsets) - 1).astype(np.int64)
    oo = np.zeros(len(offsets), dtype=np.uint64)
    oo[1:] = np.cumsum(per)
    return flat[idx], oo


def _flat(sents_ids, dtype=np.int32):
    offs = np.zeros(len(sents_ids) + 1, dtype=np.uint64)
    if sents_ids:
        offs[1:] = np.cumsum([len(s) for s in sents_ids])
    return np.array([t for s in sents_ids for t in s], dtype=dtype), offs


def _texts(text, oo):
    text, oo = np.asarray(text), np.asarray(oo).astype(np.int64)
    return [bytes(text[oo[i]:oo[i + 1]]).decode() for i in range(len(oo) - 1)]


def same_as_host(bpe, sents_ids, ignore=None, dev=False):
    """decode_packed == decode, for int32 and int64 ids (and through CUDA tensors with dev)."""
    want = bpe.decode(sents_ids, ignore_ids=ignore) if sents_ids else []
    for dt in (np.int32, np.int64):
        ids, offs = _flat(sents_ids, dt)
        assert _texts(*bpe.decode_packed(ids, offs, ignore_ids=ignore)) == want
    if dev:
        import torch
        ids, offs = _flat(sents_ids)
        t, o = bpe.decode_packed(torch.from_numpy(ids).cuda(), torch.from_numpy(offs.astype(np.int64)).cuda(),
                                 ignore_ids=ignore, out="cuda")
        assert t.is_cuda and o.is_cuda and _texts(t.cpu().numpy(), o.cpu().numpy()) == want
    return want


# ---- bodies shared with the emulator test ------------------------------------------------------------
def check_parity_stress(oracle, seed, dev=False):
    text, vocab, cov, sents = _cases.stress_case(seed)
    try:
        m = _model(oracle, text, vocab, cov)
    except ValueError:
        return
    bpe, g = _bpe(m), GpuEncoder(m)
    for kw in (dict(), dict(bos=True, eos=True), dict(reverse=True, eos=True)):
        same_as_host(bpe, g.encode(sents + _cases.EDGE_SENTENCES, **kw), dev=dev)


def check_parity_corpus(oracle, text, vocab, cov, sents, special=None, dev=False):
    special = special or {}
    m = _model(oracle, text, vocab, cov, **special)
    bpe, g = _bpe(m), GpuEncoder(m)
    kws = [dict(), dict(reverse=True)]
    if special.get("bos", 2) != -1 and special.get("eos", 3) != -1:
        kws += [dict(bos=True, eos=True), dict(bos=True, eos=True, reverse=True)]
    for kw in kws:
        ids = g.encode(sents, **kw)
        same_as_host(bpe, ids, dev=dev)
        tab = piece_table(bpe, m)
        flat, offs = _flat(ids)
        t, o = oracle_decode(tab, flat, offs)
        assert _texts(t, o) == bpe.decode(ids)
    return m, bpe


def check_ignore_ids(oracle, dev=False):
    m = _model(oracle, _cases.dirty_zipf_text(), 1200, 0.95)
    bpe, g = _bpe(m), GpuEncoder(m)
    sents = _cases.zipf_sentences(120) + _cases.EDGE_SENTENCES
    ids = g.encode(sents, bos=True, eos=True)
    V = bpe.vocab_size()
    sp = read_model(m)[0][9601]
    word_ids = sorted({i for s in ids for i in s[1:3]})
    for ign in (None, [], [2, 3], {sp}, [-5, V + 10], (2, 3, sp, -5, V + 10), [2] + word_ids, set(range(V))):
        same_as_host(bpe, ids, ign, dev=dev)
    # the first ids ignored: the strip lands on a later id
    space_first = [s for s in ids if len(s) > 3]
    same_as_host(bpe, [s[1:] for s in space_first], ignore=[s[1] for s in space_first], dev=dev)
    same_as_host(bpe, [[sp, sp] + s for s in space_first[:20]], ignore=[sp, 2], dev=dev)
    # sets that empty whole sentences
    same_as_host(bpe, [[2, 3], [2], [], [3, 2, 3]] + ids[:5], ignore=[2, 3], dev=dev)
    # the oracle with ignore sets
    tab = piece_table(bpe, m)
    flat, offs = _flat(ids)
    for ign in ([2, 3], [sp, 2, -5]):
        assert _texts(*oracle_decode(tab, flat, offs, ign)) == bpe.decode(ids, ignore_ids=ign)


def check_synthetic_lists(oracle, dev=False):
    m = _model(oracle, _cases.dirty_zipf_text(), 1500)
    bpe = _bpe(m)
    V = bpe.vocab_size()
    unk, pad, bos, eos = read_model(m)[2]
    sp = read_model(m)[0][9601]
    vocab = bpe.vocab()
    words = [i for i, p in enumerate(vocab) if p.startswith("▁") and len(p) > 2]
    inner = [i for i, p in enumerate(vocab) if i > 3 and not p.startswith("▁")]
    w, x = words[0], inner[5]
    cases = [[sp, w], [sp, sp, w], [sp], [sp, x, w], [unk, w], [bos, sp, w, eos], [pad], [eos, w], [], [w, w, sp],
             [x], [x, sp, sp]]
    same_as_host(bpe, cases, dev=dev)
    same_as_host(bpe, [[], [], []], dev=dev)
    same_as_host(bpe, [[]] + cases + [[]], dev=dev)
    text, oo = bpe.decode_packed(np.zeros(0, dtype=np.int32), np.zeros(1, dtype=np.uint64))
    assert len(text) == 0 and oo.tolist() == [0]
    rng = np.random.default_rng(5)
    big = rng.integers(0, V, size=100_000).tolist()
    same_as_host(bpe, [big], dev=dev)
    same_as_host(bpe, [big[:33], [w] * 64, big[:31], [sp] * 40 + [x]], dev=dev)


def check_long_pieces(oracle, dev=False):
    """Pieces over 1 KB (a model trained on long space-free words): one round's bytes spread over the lanes."""
    word = b"abcd" * 700
    text = b" ".join([word, word[:1500], word, b"abcdab" * 300] * 6)
    m = _model(oracle, text, 32)
    bpe, g = _bpe(m), GpuEncoder(m)
    assert max(len(p) for p in bpe.vocab()) > 1024
    ids = g.encode([word, word + b" " + word[:1001], b"x " + word[:777] + b" ab " + word, b"abcd abcd " * 5])
    assert max(len(bpe.id_to_subword(i)) for s in ids for i in s) > 1024
    same_as_host(bpe, ids, dev=dev)
    rng = np.random.default_rng(7)
    V = bpe.vocab_size()
    mixed = [rng.integers(0, V, size=int(n)).tolist() for n in rng.integers(0, 70, size=40)]
    same_as_host(bpe, mixed, dev=dev)
    same_as_host(bpe, mixed, ignore=[2, 3], dev=dev)


def check_errors(oracle, dev=False):
    m = _model(oracle, _cases.dirty_zipf_text(), 1200)
    bpe = _bpe(m)
    V = bpe.vocab_size()
    text = "id must be in the range [0, vocab_size - 1]. Current value: vocab_size = %d; id=%d;"
    for bad in (V, -1, 2**31 - 1, -2**31):
        sents = [[5, 6], [7, bad, 8]]
        with pytest.raises(ValueError) as e_host:
            bpe.decode(sents)
        assert str(e_host.value) == text % (V, bad)
        for dt in (np.int32, np.int64):
            with pytest.raises(ValueError) as e:
                bpe.decode_packed(*_flat(sents, dt))
            assert str(e.value) == str(e_host.value)
        assert _texts(*bpe.decode_packed(*_flat(sents), ignore_ids=[bad])) == bpe.decode(sents, ignore_ids=[bad])
    for big in (2**31, 2**40, -2**31 - 1):   # int64 values outside int32: never truncated
        with pytest.raises(ValueError, match=r"Current value: vocab_size = %d; id=%d;" % (V, big)):
            bpe.decode_packed(*_flat([[5], [big, 7]], np.int64))
        with pytest.raises(ValueError, match=r"id=%d;" % V):   # an earlier invalid id is reported first
            bpe.decode_packed(*_flat([[V], [big]], np.int64))
        t, o = bpe.decode_packed(*_flat([[5, big], [big]], np.int64), ignore_ids=[big])
        assert _texts(t, o) == bpe.decode([[5], []])
    # two bad ids in different sentences: the earlier one
    many = [[5] * 40] * 300 + [[6, V + 3]] + [[7] * 50] * 300 + [[-7]]
    with pytest.raises(ValueError, match=r"id=%d;" % (V + 3)):
        bpe.decode_packed(*_flat(many))
    with pytest.raises(ValueError, match=r"id=-7;"):
        bpe.decode_packed(*_flat(many), ignore_ids=[V + 3])
    assert _texts(*bpe.decode_packed(*_flat(many), ignore_ids=[V + 3, -7])) == bpe.decode(many, ignore_ids=[V + 3, -7])
    # malformed offsets: an error, never a fault
    ids = np.arange(4, 24, dtype=np.int32)
    for offs in ([0, 5, 3, 20], [0, 21], [3, 2], [0, 10, 30], [25, 30]):
        with pytest.raises(ValueError, match="offsets must be non-decreasing"):
            bpe.decode_packed(ids, np.array(offs, dtype=np.uint64))
        if dev:
            import torch
            with pytest.raises(ValueError, match="offsets must be non-decreasing"):
                bpe.decode_packed(torch.from_numpy(ids).cuda(), torch.tensor(offs).cuda(), out="cuda")
    with pytest.raises(TypeError):
        bpe.decode_packed(ids, np.array([0, 20], dtype=np.uint64), ignore_ids=5)
    with pytest.raises(TypeError):
        bpe.decode_packed(ids.astype(np.float32), np.array([0, 20], dtype=np.uint64))
    assert _texts(*bpe.decode_packed(ids, np.array([0, 20], dtype=np.uint64))) == bpe.decode([ids.tolist()])


def check_interfaces(oracle, dev=False):
    import torch
    m = _model(oracle, _cases.dirty_zipf_text(), 1200)
    bpe, g = _bpe(m), GpuEncoder(m)
    sents = _cases.zipf_sentences(200) + list(_cases.EDGE_SENTENCES)
    ids = g.encode(sents, bos=True, eos=True)
    want = bpe.decode(ids)
    flat, offs = _flat(ids)
    inputs = [flat, flat.astype(np.int64), torch.from_numpy(flat), torch.from_numpy(flat.astype(np.int64))]
    offs_in = [offs, offs.astype(np.int64), torch.from_numpy(offs.astype(np.int64))]
    if dev:
        inputs += [torch.from_numpy(flat).cuda(), torch.from_numpy(flat.astype(np.int64)).cuda()]
        offs_in += [torch.from_numpy(offs.astype(np.int64)).cuda()]
    outs = ["numpy", "torch"] + (["cuda"] if dev else [])
    for x in inputs:
        for o in offs_in:
            for out in outs:
                t, oo = bpe.decode_packed(x, o, out=out)
                if out == "numpy":
                    assert t.dtype == np.uint8 and oo.dtype == np.uint64
                else:
                    assert t.dtype == torch.uint8 and oo.dtype == torch.int64 and t.is_cuda == (out == "cuda")
                    t, oo = t.cpu().numpy(), oo.cpu().numpy()
                assert _texts(t, oo) == want
    # offsets that do not start at 0: ids in front of and behind the batch are not read
    pre = np.full(37, 10**6, dtype=np.int32)
    shifted = np.concatenate([pre, flat, pre])
    t, oo = bpe.decode_packed(shifted, offs + 37)
    assert _texts(t, oo) == want and int(oo[0]) == 0
    # two threads on one handle each get their own result
    batches = [ids[k * 37:k * 37 + 90] for k in range(4)]
    wants = [bpe.decode(b) for b in batches]
    errs = []

    def body(k):
        out = "cuda" if dev and k % 2 else "numpy"   # with a GPU, half of the threads use the device entry point
        try:
            for _ in range(5):
                t, oo = bpe.decode_packed(*_flat(batches[k]), out=out)
                if out == "cuda":
                    t, oo = t.cpu().numpy(), oo.cpu().numpy()
                assert _texts(t, oo) == wants[k]
        except BaseException as e:  # noqa: BLE001
            errs.append(e)

    th = [threading.Thread(target=body, args=(k,)) for k in range(4)]
    for t_ in th:
        t_.start()
    for t_ in th:
        t_.join()
    assert not errs, errs[0]


def _read(ptr, n, dtype, dev):
    """n values at a library-owned device (or, under the emulator, host) address."""
    if dev:
        import torch
        from youtokentome_b200.distributed import _DevView
        ts = {np.uint8: "|u1", np.int32: "<i4", np.uint64: "<i8"}[dtype]   # (torch has no uint64: read as int64)
        return torch.as_tensor(_DevView(ptr, max(n, 1), ts), device="cuda")[:n].cpu().numpy().view(dtype)
    buf = (C.c_char * max(n * np.dtype(dtype).itemsize, 1)).from_address(ptr)
    return np.frombuffer(bytes(buf), dtype=dtype)[:n].copy()


def check_abi_device(oracle, dev=False):
    """yttm_enc_run_device -> yttm_dec_run_device on the returned ids in place; the decode results survive a following
    encode on the same handle; the launch count of a call does not depend on the batch size."""
    from youtokentome_b200 import _lib
    L = _lib.lib()
    m = _model(oracle, _cases.dirty_zipf_text(), 1200)
    bpe = _bpe(m)
    sents = _cases.zipf_sentences(300) + list(_cases.EDGE_SENTENCES)
    buf, offs = _pack(sents)
    ctx, enc = L.yttm_api_device_context(bpe._h), L.yttm_api_device_encoder(bpe._h)
    if dev:
        import torch
        keep = (torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda(), torch.from_numpy(offs.astype(np.int64)).cuda())
        p_bytes, p_offs = keep[0].data_ptr(), keep[1].data_ptr()
        torch.cuda.synchronize()
    else:
        raw = np.frombuffer(buf, dtype=np.uint8).copy()
        p_bytes, p_offs = raw.ctypes.data, offs.ctypes.data
    p_ids, p_ioff, n_ids = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
    assert L.yttm_enc_run_device(enc, p_bytes, p_offs, len(buf), len(sents), 1, 1, 0, 0.0, 0, 0, C.byref(p_ids),
                                 C.byref(p_ioff), C.byref(n_ids)) == 0, L.yttm_last_error(ctx)
    ids_host = _read(p_ids.value, n_ids.value, np.int32, dev)
    ioff_host = _read(p_ioff.value, len(sents) + 1, np.uint64, dev)
    want = bpe.decode([ids_host[ioff_host[i]:ioff_host[i + 1]].tolist() for i in range(len(sents))])
    p_text, p_toff, n_text = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
    l0 = L.yttm_launch_count(ctx)
    assert L.yttm_dec_run_device(enc, p_ids, n_ids.value, p_ioff, len(sents), None, 0, C.byref(p_text), C.byref(p_toff),
                                 C.byref(n_text)) == 0, L.yttm_last_error(ctx)
    per_call = L.yttm_launch_count(ctx) - l0
    assert per_call == 5   # count, three scan launches, emit
    for st in ("decode", "dec_count", "dec_scan", "dec_emit"):
        assert L.yttm_stage_ms(ctx, st.encode()) >= 0
    text0 = _read(p_text.value, n_text.value, np.uint8, dev)
    toff0 = _read(p_toff.value, len(sents) + 1, np.uint64, dev)
    assert _texts(text0, toff0) == want
    # a following encode on the same handle leaves the decode results alone
    assert L.yttm_enc_run_device(enc, p_bytes, p_offs, len(buf), len(sents), 0, 0, 1, 0.0, 0, 0, C.byref(C.c_void_p()),
                                 C.byref(C.c_void_p()), C.byref(C.c_uint64())) == 0
    bpe.encode_packed(buf, offs)
    assert np.array_equal(_read(p_text.value, n_text.value, np.uint8, dev), text0)
    assert np.array_equal(_read(p_toff.value, len(sents) + 1, np.uint64, dev), toff0)
    # the host-buffer entry point: return code 2 with the size needed, then the same text
    ids_c = np.ascontiguousarray(ids_host)
    out = np.zeros(16, dtype=np.uint8)
    oo = np.zeros(len(sents) + 1, dtype=np.uint64)
    tot = C.c_uint64(0)
    assert L.yttm_dec_run(enc, ids_c.ctypes.data, ioff_host.ctypes.data, len(sents), None, 0, out.ctypes.data, 16,
                          oo.ctypes.data, C.byref(tot)) == 2 and tot.value == n_text.value
    out = np.zeros(tot.value, dtype=np.uint8)
    assert L.yttm_dec_run(enc, ids_c.ctypes.data, ioff_host.ctypes.data, len(sents), None, 0, out.ctypes.data, tot.value,
                          oo.ctypes.data, C.byref(tot)) == 0
    assert _texts(out, oo) == want
    # ... and leaves the results of the device entry point alone too
    assert np.array_equal(_read(p_text.value, n_text.value, np.uint8, dev), text0)
    assert np.array_equal(_read(p_toff.value, len(sents) + 1, np.uint64, dev), toff0)
    # launches per call do not depend on the batch size
    l0 = L.yttm_launch_count(ctx)
    assert L.yttm_dec_run_device(enc, p_ids, n_ids.value, p_ioff, 3, None, 0, C.byref(p_text), C.byref(p_toff),
                                 C.byref(n_text)) == 0
    assert L.yttm_launch_count(ctx) - l0 == per_call
    assert L.yttm_dec_run_device(None, None, 0, None, 0, None, 0, C.byref(p_text), C.byref(p_toff), C.byref(n_text)) == 1
    assert b"null encoder handle" in L.yttm_last_error(None)


# ---- GPU tests ----------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(8))
def test_parity_stress(product, oracle, seed):
    check_parity_stress(oracle, seed, dev=True)


@pytest.mark.parametrize("name", sorted(synth.GOLDEN_TEXTS))
def test_parity_golden_texts(product, oracle, name):
    train, test, vocab = synth.GOLDEN_TEXTS[name]
    check_parity_corpus(oracle, train.encode(), vocab, 1.0, [test.encode()] + test.encode().split(b"\n"), dev=True)


@pytest.mark.parametrize("cov", [1.0, 0.9])
def test_parity_dirty_zipf(product, oracle, cov):
    check_parity_corpus(oracle, _cases.dirty_zipf_text(), 1500, cov, _cases.zipf_sentences(1000) + _cases.EDGE_SENTENCES,
                        dev=True)


@pytest.mark.parametrize("special", [dict(pad=-1, unk=1, bos=2, eos=3), dict(pad=-1, unk=5, bos=-1, eos=-1),
                                     dict(pad=3, unk=40, bos=41, eos=1000)])
def test_parity_special_layouts(product, oracle, special):
    """"▁" with id 0 (pad = -1) and special ids between / above the others."""
    check_parity_corpus(oracle, _cases.dirty_zipf_text(), 1200, 1.0, _cases.zipf_sentences(300) + _cases.EDGE_SENTENCES,
                        special, dev=True)


def test_ignore_ids(product, oracle):
    check_ignore_ids(oracle, dev=True)


def test_synthetic_id_lists(product, oracle):
    check_synthetic_lists(oracle, dev=True)


def test_long_pieces(product, oracle):
    check_long_pieces(oracle, dev=True)


def test_errors(product, oracle):
    check_errors(oracle, dev=True)


def test_interfaces(product, oracle):
    check_interfaces(oracle, dev=True)


def test_abi_device_and_launches(product, oracle):
    check_abi_device(oracle, dev=True)


def test_encode_cuda_decode_cuda_round_trip(product, oracle):
    import torch
    m = _model(oracle, _cases.dirty_zipf_text(), 1500)
    bpe = _bpe(m)
    sents = _cases.zipf_sentences(500) + list(_cases.EDGE_SENTENCES)
    data, offs = _pack(sents)
    ids, oo = bpe.encode_packed(data, offs, out="cuda")
    text, to = bpe.decode_packed(ids, oo, out="cuda")
    assert text.is_cuda and to.is_cuda
    h_ids, h_oo = ids.cpu().numpy(), oo.cpu().numpy()
    want = bpe.decode([h_ids[h_oo[i]:h_oo[i + 1]].tolist() for i in range(len(sents))])
    assert _texts(text.cpu().numpy(), to.cpu().numpy()) == want
    text2, to2 = bpe.decode_packed(*bpe.encode_packed(torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda(),
                                                      torch.from_numpy(offs.astype(np.int64)).cuda(), out="cuda"), out="cuda")
    assert torch.equal(text, text2) and torch.equal(to, to2)


def test_scale_bench_shape(product):
    """configs[1] shape: 1 M x 128-byte FastZipf sentences, vocab 32 000 model trained on the GPU; the whole decode
    equals the numpy oracle, a sample equals BPE.decode, and a call launches as many kernels at 1 k as at 1 M."""
    import torch
    from _gpu import gpu_train
    from youtokentome_b200 import _lib
    fz = synth.FastZipf(n_words=200_000, s=1.07, seed=1234)
    m = gpu_train(fz.text(20_000_000), 32_000, 1.0)
    bpe = _bpe(m)
    buf, offs = fz.packed_sentences(1_000_000, 128, seed=4321)
    ids, oo = bpe.encode_packed(torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda(),
                                torch.from_numpy(np.asarray(offs).astype(np.int64)).cuda(), out="cuda")
    L = _lib.lib()
    ctx = L.yttm_api_device_context(bpe._h)
    launches = []
    for n in (1_000, 1_000_000):
        l0 = L.yttm_launch_count(ctx)
        text, to = bpe.decode_packed(ids, oo[:n + 1], out="cuda")
        launches.append(L.yttm_launch_count(ctx) - l0)
    assert launches[0] == launches[1]
    h_ids, h_oo = ids.cpu().numpy(), oo.cpu().numpy()
    text, to = text.cpu().numpy(), to.cpu().numpy().astype(np.uint64)
    tab = piece_table(bpe, m)
    step = 100_000
    for lo in range(0, 1_000_000, step):
        t_o, o_o = oracle_decode(tab, h_ids, h_oo[lo:lo + step + 1])
        a, b = int(to[lo]), int(to[lo + step])
        assert np.array_equal(text[a:b], t_o) and np.array_equal(to[lo:lo + step + 1] - to[lo], o_o), lo
    sample = np.random.default_rng(1).choice(1_000_000, 5_000, replace=False)
    want = bpe.decode([h_ids[h_oo[i]:h_oo[i + 1]].tolist() for i in sample])
    assert [bytes(text[to[i]:to[i + 1]]).decode() for i in sample] == want


def test_zzz_sanitizer_memcheck_decode(product):
    """compute-sanitizer memcheck over tools/sanitize_decode.py: no report; skips where the tool refuses the device."""
    import shutil
    import subprocess
    import sys
    from _bind import ROOT
    exe = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(exe):
        pytest.skip("compute-sanitizer is not installed")
    env = {k: v for k, v in os.environ.items() if not k.startswith(("YTTM_", "YT_EMU_"))}
    r = subprocess.run([exe, "--tool", "memcheck", sys.executable, os.path.join(ROOT, "tools", "sanitize_decode.py")],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    text = r.stdout.decode(errors="replace")
    if "Error: Device not supported" in text:
        pytest.skip("compute-sanitizer does not support this device here")
    assert "checks identical to the host decode" in text, text[-1500:]
    assert "ERROR SUMMARY: 0 errors" in text, text[-1500:]

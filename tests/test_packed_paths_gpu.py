"""The staging, run and read-out that the packed methods of `BPE` (encode_packed with and without spans, encode_padded,
encode_subwords_packed, decode_packed) share, and the checks and result epilogue that the yttm_enc_run* entry points
share: the first offset of a batch, empty batches through every method and output form, argument errors, an empty
device call after a full one, and the <BOS> / <EOS> check of every layer.  tests/test_packed_paths_emul_cpu.py runs the
same bodies with dev=False under the SIMT emulator, where only the host outputs exist and device memory is host
memory."""
import ctypes as C

import numpy as np
import pytest

import test_encode_padded_gpu as PG
from _bind import _pack, tmp_model_path
from youtokentome_b200 import _lib, synth

pytestmark = pytest.mark.gpu

SENTS = [b"abc dab", b"", b" a  bcd dd", b"cab\xff", "é abc".encode(), b"dcba abcd abcd", b"   "]
NO_BOS = dict(pad=-1, unk=0, bos=-1, eos=-1)
FLAG_TEXT = {"bos": "Can't add <BOS> token. Model was trained without it.",
             "eos": "Can't add <EOS> token. Model was trained without it."}

_models = {}


def _model(oracle, **special):
    key = tuple(sorted(special.items()))
    if key not in _models:
        m = tmp_model_path("orc")
        oracle.train(synth.readme_corpus(n_lines=200), m, 100, 1.0, **special)
        _models[key] = m
    return _models[key]


def _bpe(m):
    import youtokentome_b200 as yttm
    return yttm.BPE(m)


def _outs(dev):
    return ["numpy", "torch"] + (["cuda"] if dev else [])


def _np(x):
    return x.cpu().numpy() if type(x).__module__.startswith("torch") else np.asarray(x)


def _check_result(got, out, want):
    """got: a method's result for `out`; want: [(numpy array, numpy dtype for out="numpy")]: torch results are the
    same values as int64 where numpy has uint64."""
    assert len(got) == len(want)
    for g, (w, dt) in zip(got, want):
        if out == "numpy":
            assert isinstance(g, np.ndarray) and g.dtype == dt, (out, g.dtype, dt)
        else:
            import torch
            assert isinstance(g, torch.Tensor) and g.is_cuda == (out == "cuda"), out
            assert g.dtype == {np.uint8: torch.uint8, np.int32: torch.int32}.get(dt, torch.int64), (out, g.dtype, dt)
        assert _np(g).shape == w.shape and np.array_equal(_np(g).astype(np.int64), w.astype(np.int64)), (out, g, w)


def device_ids_abi(bpe, data, offs, dev):
    """yttm_api_encode_device (yttm_enc_run_device) without flags: (ids pointer, ids, id offsets).  The input is CUDA
    memory on the GPU and host memory (the emulator's device memory) under the emulator."""
    L = _lib.lib()
    offs = np.ascontiguousarray(offs, dtype=np.uint64)
    n = len(offs) - 1
    if dev:
        import torch
        from youtokentome_b200.distributed import _DevView
        keep = (torch.frombuffer(bytearray(data + b"\0"), dtype=torch.uint8).cuda(),
                torch.from_numpy(offs.astype(np.int64)).cuda())
        ptrs = [t.data_ptr() for t in keep]
        get = lambda p, k, ts: torch.as_tensor(_DevView(p, k, ts), device="cuda").cpu().numpy()
    else:
        keep = (C.create_string_buffer(data + b"\0"), offs)
        ptrs = [C.cast(keep[0], C.c_void_p).value, offs.ctypes.data]
        get = lambda p, k, ts: np.ctypeslib.as_array(C.cast(p, C.POINTER(np.ctypeslib.as_ctypes_type(ts))),
                                                     shape=(k,)).copy()
    p_ids, p_off, total = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
    rc = L.yttm_api_encode_device(bpe._h, ptrs[0], ptrs[1], len(data), n, 0, 0, 0, 0.0, C.byref(p_ids), C.byref(p_off),
                                  C.byref(total))
    assert rc == 0, L.yttm_api_last_error(bpe._h).decode()
    ids = get(p_ids.value, total.value, "<i4") if total.value else np.zeros(0, np.int32)
    return p_ids.value, ids, get(p_off.value, n + 1, "<i8")


# ---- bodies shared with the emulator test --------------------------------------------------------------------------
def check_first_offset(oracle):
    """encode_packed(out="cuda") reads sentence i at data[offsets[i]:offsets[i+1]] when offsets[0] > 0, from host
    bytes and from CUDA tensors, with host or CUDA offsets: the host path's ids and offsets."""
    import torch
    bpe = _bpe(_model(oracle))
    data, offs = _pack(SENTS)
    prefix = b"dd a\xe2\x96 bc"
    data, offs = prefix + data + b" abc", offs + np.uint64(len(prefix))
    for kw in (dict(), dict(bos=True, eos=True, reverse=True)):
        ids, oo = bpe.encode_packed(data, offs, **kw)
        assert oo[-1] == len(ids) > 0
        d_data = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
        d_offs = torch.from_numpy(offs.astype(np.int64)).cuda()
        for src in (data, np.frombuffer(data, np.uint8), d_data):
            for o in (offs, d_offs):
                got = bpe.encode_packed(src, o, out="cuda", **kw)
                _check_result(got, "cuda", [(ids, np.int32), (oo, np.uint64)])


def check_empty_batches(oracle, dev=False):
    """No sentence, and sentences that are all empty, through every packed method and output form: no ids, no
    pieces, no text, and offsets of zeros, in each method's documented dtypes."""
    m = _model(oracle)
    bpe = _bpe(m)
    pad = PG._special(m)[1]
    for n in (0, 3):
        offs = np.zeros(n + 1, np.uint64)
        zeros = np.zeros(n + 1, np.uint64)
        for data in (b"", np.zeros(0, np.uint8)):
            for out in _outs(dev):
                _check_result(bpe.encode_packed(data, offs, out=out), out,
                              [(np.zeros(0, np.int32), np.int32), (zeros, np.uint64)])
                _check_result(bpe.encode_packed(data, offs, out=out, with_spans=True), out,
                              [(np.zeros(0, np.int32), np.int32), (zeros, np.uint64), (np.zeros((0, 2)), np.uint64)])
                for L in [4] + ([None] if dev else []):
                    W = L or 0
                    for spans in (False, True):
                        want = [(np.full((n, W), pad), np.int32), (np.zeros(n), np.int64)]
                        want += [(np.zeros((n, W, 2)), np.uint64)] if spans else []
                        _check_result(bpe.encode_padded(data, offs, max_length=L, out=out, with_spans=spans), out, want)
                _check_result(bpe.encode_subwords_packed(data, offs, out=out), out,
                              [(np.zeros(0, np.uint8), np.uint8), (np.zeros(1), np.uint64), (zeros, np.uint64)])
                _check_result(bpe.decode_packed(np.zeros(0, np.int32), offs, out=out), out,
                              [(np.zeros(0, np.uint8), np.uint8), (zeros, np.uint64)])


def check_argument_errors(oracle, dev=False):
    """encode_packed checks its offsets and dropout_prob like its sibling methods do, for every output form."""
    bpe = _bpe(_model(oracle))
    data, offs = _pack(SENTS)
    for out in _outs(dev):
        for bad in (np.zeros(0, np.uint64), []):
            with pytest.raises(ValueError) as e:
                bpe.encode_packed(data, bad, out=out)
            assert str(e.value) == "offsets must hold at least one value"
        for p in (1.5, -0.5):
            with pytest.raises(ValueError) as e:
                bpe.encode_packed(data, offs, dropout_prob=p, out=out)
            assert str(e.value) == ("dropout_prob value must be in the range [0, 1]. Current value of dropout_prob = "
                                    + str(p))
            with pytest.raises(ValueError):
                bpe.encode_packed(data, offs, dropout_prob=p, out=out, with_spans=True)


def check_empty_after_full(oracle, dev=False):
    """yttm_enc_run_device with no sentence hands out a non-null ids pointer and offsets [0]: on a handle that has
    encoded nothing yet, after an ids call and after a padded call whose row lengths share the offsets buffer."""
    m = _model(oracle)
    bpe = _bpe(m)
    data, offs = _pack(SENTS)

    def empty():
        p_ids, ids, oo = device_ids_abi(bpe, b"", [0], dev)
        assert p_ids and len(ids) == 0 and oo.tolist() == [0]

    empty()
    _, ids, oo = device_ids_abi(bpe, data, offs, dev)
    want_ids, want_oo = bpe.encode_packed(data, offs)
    assert np.array_equal(ids, want_ids) and np.array_equal(oo.astype(np.uint64), want_oo)
    empty()
    if dev:
        lengths = _np(bpe.encode_padded(data, offs, out="cuda")[1])
    else:  # the width-0 device entry on host memory
        lengths = PG.padded_abi(bpe, data, offs, 0, PG.PAD_FROM_MODEL, {}, False)[1]
    assert lengths[0] > 0
    empty()


def check_flags_without_tokens(oracle, dev=False):
    """bos / eos on a model without <BOS> / <EOS> (and without <PAD>): every packed method of BPE in every output
    form, and every yttm_enc_run* entry point, report the same text."""
    bpe = _bpe(_model(oracle, **NO_BOS))
    L = _lib.lib()
    data, offs = _pack(SENTS)
    for flag, text in FLAG_TEXT.items():
        kw = {flag: True}
        calls = [lambda **k: bpe.encode_packed(data, offs, **k),
                 lambda **k: bpe.encode_packed(data, offs, with_spans=True, **k),
                 lambda **k: bpe.encode_padded(data, offs, max_length=4, **k),
                 lambda **k: bpe.encode_subwords_packed(data, offs, **k)]
        if dev:
            calls.append(lambda **k: bpe.encode_padded(data, offs, **k))
        for call in calls:
            for out in _outs(dev):
                with pytest.raises(ValueError) as e:
                    call(out=out, **kw)
                assert str(e.value) == text, (flag, out)
        if not dev:  # the width-0 padded rows of the device entry, on host memory
            with pytest.raises(ValueError) as e:
                PG.padded_abi(bpe, data, offs, 0, PG.PAD_FROM_MODEL, kw, False)
            assert str(e.value) == text
        check_entry_points(L, bpe, flag, text)


def check_entry_points(L, bpe, flag, text):
    """Every yttm_enc_run* entry point refuses `flag` with `text` before it reads its arguments (all null here)."""
    enc, ctx = L.yttm_api_device_encoder(bpe._h), L.yttm_api_device_context(bpe._h)
    assert enc and ctx
    b, e = int(flag == "bos"), int(flag == "eos")
    n, p = C.c_uint64(0), None
    P = lambda: C.byref(C.c_void_p())
    runs = {
        "yttm_enc_run": lambda: L.yttm_enc_run(enc, p, p, 1, b, e, 0, 0.0, 0, 0, p, 0, p, C.byref(n)),
        "yttm_enc_run_device": lambda: L.yttm_enc_run_device(enc, p, p, 0, 1, b, e, 0, 0.0, 0, 0, P(), P(), C.byref(n)),
        "yttm_enc_run_spans": lambda: L.yttm_enc_run_spans(enc, p, p, 1, b, e, 0, 0.0, 0, 0, p, 0, p, p, C.byref(n)),
        "yttm_enc_run_spans_device": lambda: L.yttm_enc_run_spans_device(enc, p, p, 0, 1, b, e, 0, 0.0, 0, 0, P(), P(),
                                                                         P(), C.byref(n)),
        "yttm_enc_run_padded": lambda: L.yttm_enc_run_padded(enc, p, p, 1, b, e, 0, 0.0, 0, 0, 4, 0, p, p, p),
        "yttm_enc_run_padded_device": lambda: L.yttm_enc_run_padded_device(enc, p, p, 0, 1, b, e, 0, 0.0, 0, 0, 4, 0, 0,
                                                                           P(), P(), P(), C.byref(C.c_uint32())),
        "yttm_enc_run_subwords": lambda: L.yttm_enc_run_subwords(enc, p, p, 1, b, e, 0, 0.0, 0, 0, p, 0, p, 0, p,
                                                                 C.byref(n), C.byref(n)),
        "yttm_enc_run_subwords_device": lambda: L.yttm_enc_run_subwords_device(enc, p, p, 0, 1, b, e, 0, 0.0, 0, 0, P(),
                                                                               P(), P(), C.byref(n), C.byref(n)),
    }
    for name, run in runs.items():
        assert run() == 1, name
        assert L.yttm_last_error(ctx).decode() == text, name


# ---- tests ---------------------------------------------------------------------------------------------------------
def test_first_offset(product, oracle):
    check_first_offset(oracle)


def test_empty_batches(product, oracle):
    check_empty_batches(oracle, dev=True)


def test_argument_errors(product, oracle):
    check_argument_errors(oracle, dev=True)


def test_empty_after_full(product, oracle):
    check_empty_after_full(oracle, dev=True)


def test_flags_without_tokens(product, oracle):
    check_flags_without_tokens(oracle, dev=True)

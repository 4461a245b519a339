"""The padded output kernel of device encode (emit_padded_kernel: row lengths, pad cells, kept ids and spans of every
tile of EMIT_T = 256 sentences, and the counting form for L = None) on the SIMT emulator with 1, 2 and 5 SMs, through
the bodies of tests/test_encode_padded_gpu.py at small sizes.  L = None reaches the device C entry on host memory (the
emulator's device memory).  Also, with the real library: without a GPU encode_padded fails loudly.

TEST HARNESS ONLY, like tests/test_simt_emul_cpu.py."""
import pytest

import test_encode_padded_gpu as PG
from _bind import _pack, tmp_model_path
from youtokentome_b200 import _lib


@pytest.fixture(params=["1", "2", "5"])
def emu(monkeypatch, request):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


@pytest.mark.parametrize("n", [1, 255, 256, 257, 600])
def test_flags_and_widths(emu, oracle, n):
    PG.check_flags_and_widths(oracle, n, kws=PG.KWS if n in (1, 257) else PG.KWS[::3])


def test_cuts_inside_words(emu, oracle):
    PG.check_cuts_inside_words(oracle)


def test_spans_shift(emu, oracle):
    PG.check_spans_shift(oracle)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout(emu, oracle, p):
    PG.check_dropout(oracle, p)


def test_pad_ids(emu, oracle):
    PG.check_pad_ids(oracle)


def test_layouts(emu, oracle):
    PG.check_layouts(oracle)


def test_chunks(emu, oracle, monkeypatch):
    PG.check_chunks(oracle, monkeypatch, 2_200_000)


def test_errors(emu, oracle):
    PG.check_errors(oracle)


def test_padded_without_gpu_fails_loudly(product, oracle):
    if product.yttm_device_count() != 0:
        pytest.skip("a GPU is present")
    import youtokentome_b200 as yttm
    m = tmp_model_path()
    oracle.train(b"ab ab abc abd", m, 14)
    data, offs = _pack([b"ab abc", b"abd"])
    with pytest.raises(ValueError, match="no CUDA device"):
        yttm.BPE(m).encode_padded(data, offs, max_length=4)

"""The window kernels of device encode (win_count_kernel, the row-base scan and win_gather_kernel: rows of every
sentence, tiles of rows, cells from the packed ids and spans) on the SIMT emulator with 1, 2 and 5 SMs, through the
bodies of tests/test_encode_windows_gpu.py at small sizes and the device C entry on host memory (the emulator's device
memory).  Also, with the real library: without a GPU encode_windows fails loudly.

TEST HARNESS ONLY, like tests/test_simt_emul_cpu.py."""
import pytest

import test_encode_windows_gpu as WG
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
def test_flags(emu, oracle, n):
    WG.check_flags(oracle, n, kws=WG.KWS if n in (1, 257) else WG.KWS[::3])


def test_count_edges(emu, oracle):
    WG.check_count_edges(oracle)


def test_many_rows(emu, oracle):
    WG.check_many_rows(oracle, 260)


def test_long(emu, oracle):
    WG.check_long(oracle)


def test_content(emu, oracle):
    WG.check_content(oracle)


def test_equivalences(emu, oracle):
    WG.check_equivalences(oracle)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout(emu, oracle, p):
    WG.check_dropout(oracle, p)


def test_inputs(emu, oracle):
    WG.check_inputs(oracle)


def test_errors(emu, oracle):
    WG.check_errors(oracle)


def test_windows_without_gpu_fails_loudly(product, oracle):
    if product.yttm_device_count() != 0:
        pytest.skip("a GPU is present")
    import youtokentome_b200 as yttm
    m = tmp_model_path()
    oracle.train(b"ab ab abc abd", m, 14)
    data, offs = _pack([b"ab abc", b"abd"])
    for kw in ({}, dict(with_spans=True, out="cuda"), dict(stride=2, out="torch")):
        with pytest.raises(ValueError, match="no CUDA device"):
            yttm.BPE(m).encode_windows(data, offs, 4, **kw)

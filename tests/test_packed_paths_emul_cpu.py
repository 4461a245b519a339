"""The shared staging and result paths of the packed methods and the yttm_enc_run* entry points on the CPU under the SIMT
emulator with 1, 2 and 5 SMs, through the bodies of tests/test_packed_paths_gpu.py with the host outputs only.  Also,
with the real library: without a GPU the device entries of BaseEncoder report a missing <BOS> / <EOS> before the
missing device.

TEST HARNESS ONLY, like tests/test_simt_emul_cpu.py."""
import ctypes as C

import pytest

import test_packed_paths_gpu as PP
from _bind import tmp_model_path
from youtokentome_b200 import _lib


@pytest.fixture(params=["1", "2", "5"])
def emu(monkeypatch, request):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


def test_empty_batches(emu, oracle):
    PP.check_empty_batches(oracle)


def test_argument_errors(emu, oracle):
    PP.check_argument_errors(oracle)


def test_empty_after_full_abi(emu, oracle):
    PP.check_empty_after_full(oracle)


def test_flags_without_tokens(emu, oracle):
    PP.check_flags_without_tokens(oracle)


def test_device_entries_without_gpu_report_flags_first(product, oracle):
    if product.yttm_device_count() != 0:
        pytest.skip("a GPU is present")
    import youtokentome_b200 as yttm
    m = tmp_model_path()
    oracle.train(b"ab ab abc abd", m, 14, **PP.NO_BOS)
    bpe = yttm.BPE(m)
    L = _lib.lib()
    p, n, P = None, C.c_uint64(0), lambda: C.byref(C.c_void_p())
    for flag, text in PP.FLAG_TEXT.items():
        b, e = int(flag == "bos"), int(flag == "eos")
        calls = [lambda: L.yttm_api_encode_device(bpe._h, p, p, 0, 1, b, e, 0, 0.0, P(), P(), C.byref(n)),
                 lambda: L.yttm_api_encode_spans_device(bpe._h, p, p, 0, 1, b, e, 0, 0.0, P(), P(), P(), C.byref(n)),
                 lambda: L.yttm_api_encode_padded_device(bpe._h, p, p, 0, 1, b, e, 0, 0.0, 4, 0, 0, P(), P(), P(),
                                                         C.byref(C.c_uint32())),
                 lambda: L.yttm_api_encode_subwords_device(bpe._h, p, p, 0, 1, b, e, 0, 0.0, P(), P(), P(), C.byref(n),
                                                           C.byref(n))]
        for i, call in enumerate(calls):
            assert call() == 1, i
            assert L.yttm_api_last_error(bpe._h).decode() == text, i

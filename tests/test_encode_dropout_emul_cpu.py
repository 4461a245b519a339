"""BPE-dropout of device encode against the reference's own DropoutQueue replaying the same draws, on the CPU under the
SIMT emulator with 1, 2 and 5 SMs: the bodies of tests/test_encode_dropout_gpu.py at small sizes.

TEST HARNESS ONLY, like tests/test_simt_emul_cpu.py."""
import pytest

import test_encode_dropout_gpu as DG
from youtokentome_b200 import _lib


@pytest.fixture(params=["1", "2", "5"])
def emu(monkeypatch, request):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


def test_packed_ids(emu, oracle):
    DG.check_packed(oracle, small=True)


def test_skip_boundary(emu, oracle):
    DG.check_boundary(oracle)


def test_keys(emu, oracle):
    DG.check_keys(oracle, small=True)


def test_space_id_zero(emu, oracle):
    DG.check_space_id_zero(oracle)


def test_chunk_pipeline(emu, oracle, monkeypatch):
    DG.check_chunks(oracle, monkeypatch, n_mb=2)


def test_api_counter_spans_padded_subwords(emu, oracle):
    DG.check_api_counter(oracle, small=True)


def test_two_threads_one_handle(emu, oracle):
    DG.check_threads(oracle, small=True)

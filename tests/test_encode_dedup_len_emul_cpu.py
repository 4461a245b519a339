"""Word lengths from the finder in the word dedup (tests/test_encode_dedup_len_gpu.py) on the SIMT emulator with 1, 2
and 5 SMs, at emulator sizes.  The emulator runs the blocks of a launch one after the other, so occurrences that claim
table slots at the same time from different blocks only meet on the GPU.

TEST HARNESS ONLY, like tests/test_simt_emul_cpu.py."""
import pytest

import test_encode_dedup_len_gpu as DL
import test_encode_words_gpu as WG
from youtokentome_b200 import _lib


def _emu(monkeypatch, sms):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", sms)
    monkeypatch.setattr(WG, "_cache", {})   # encoders belong to the library that made them
    return L


@pytest.fixture(params=["1", "2", "5"])
def emu(monkeypatch, request):
    return _emu(monkeypatch, request.param)


@pytest.fixture
def emu2(monkeypatch):
    return _emu(monkeypatch, "2")


def test_piece_edges(emu2, oracle):
    DL.check_piece_edges(oracle, edges=(1,))


def test_long_groups(emu, oracle):
    DL.check_long_groups(oracle, small=True)


def test_escape_lengths(emu2, oracle):
    DL.check_escape_lengths(oracle)


def test_misaligned_batches(emu2, oracle):
    DL.check_misaligned_batches(oracle, dev=False)


@pytest.mark.parametrize("slots", [0, 1, 8])
@pytest.mark.parametrize("weak", [False, True])
def test_last_byte_pairs(emu, oracle, monkeypatch, slots, weak):
    DL.check_last_byte_pairs(oracle, monkeypatch, slots, weak)

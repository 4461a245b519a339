"""The word dedup (tests/test_encode_dedup_gpu.py) on the SIMT emulator with 1, 2 and 5 SMs.  The emulator runs the
blocks of a launch one after the other, so two occurrences of a word that claim a table slot at the same time from
different blocks only meet on the GPU.

TEST HARNESS ONLY, like tests/test_simt_emul_cpu.py."""
import pytest

import test_encode_dedup_gpu as DG
from youtokentome_b200 import _lib


@pytest.fixture(params=["1", "2", "5"])
def emu(monkeypatch, request):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


def test_repeated_and_distinct(emu, oracle):
    DG.check_repeated_and_distinct(oracle)


def test_pairs(emu, oracle):
    DG.check_pairs(oracle)


def test_long_leader(emu, oracle):
    DG.check_long_leader(oracle)


@pytest.mark.parametrize("slots", [1, 8, 64])
@pytest.mark.parametrize("weak", [False, True])
def test_small_tables(emu, oracle, monkeypatch, slots, weak):
    DG.check_small_tables(oracle, monkeypatch, slots, weak)

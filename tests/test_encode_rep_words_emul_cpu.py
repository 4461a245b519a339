"""The representative merge's shared-memory path and its edges (tests/test_encode_rep_words_gpu.py) on the SIMT emulator
with 1 and 2 SMs.

TEST HARNESS ONLY, like tests/test_simt_emul_cpu.py."""
import os
import re

import pytest

import test_encode_rep_words_gpu as RG
import test_encode_words_gpu as WG
from _bind import ROOT
from youtokentome_b200 import _lib


@pytest.fixture(params=["1", "2"])
def emu(monkeypatch, request):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    monkeypatch.setattr(WG, "_cache", {})   # encoders belong to the library that made them
    return L


def test_constants_match_the_source():
    src = open(os.path.join(ROOT, "youtokentome_b200", "csrc", "encode.cu")).read()
    value = lambda name: re.findall(r"constexpr \w+ %s = (\d+);" % name, src)   # noqa: E731
    assert value("SHARED_W") == [str(RG.SHARED_W)] and value("SHARED_B") == [str(RG.SHARED_B)]


def test_token_counts(emu, oracle):
    RG.check_token_counts(oracle)


def test_byte_counts(emu, oracle):
    RG.check_byte_counts(oracle)


def test_unknown_runs(emu, oracle):
    RG.check_unknown_runs(oracle)


def test_equal_ranks(emu, oracle):
    RG.check_equal_ranks(oracle)


def test_space_id_zero(emu, oracle):
    RG.check_space_id_zero(oracle)


def test_record_boundary(emu, oracle):
    RG.check_record_boundary(oracle)


def test_unknown_lengths(emu, oracle):
    RG.check_unknown_lengths(oracle)

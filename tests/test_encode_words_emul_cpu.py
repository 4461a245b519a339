"""The word finder, the word-merge kernels, the rule table and the chunk cutter (tests/test_encode_words_gpu.py) on the
SIMT emulator with 1, 2 and 5 SMs, at emulator sizes; and the test that makes the plain restatement of
tests/_encode_ref.py trustworthy: it equals the oracle wherever the oracle is pinned to the reference (trained models).

The emulator runs the blocks of a launch one after the other and a thread until its next barrier, so the order in
which groups reserve their work items and hazards between the warps of a block only show on the GPU.

TEST HARNESS ONLY, like tests/test_simt_emul_cpu.py."""
import os
import re

import pytest

import test_encode_words_gpu as WG
from _bind import ROOT
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
    """The bodies whose paths do not depend on the number of blocks run once."""
    return _emu(monkeypatch, "2")


def test_constants_match_the_source():
    src = open(os.path.join(ROOT, "youtokentome_b200", "csrc", "encode.cu")).read()
    value = lambda name: re.findall(r"constexpr \w+ %s = ([^;]+);" % name, src)   # noqa: E731
    assert value("LOCAL_W") == [str(WG.LOCAL_W)] * 2          # both thread-per-word kernels
    assert value("LONG_W") == [str(WG.LONG_W)] and value("LONG_T") == [str(WG.LONG_T)]
    assert value("FIND_GMAX") == [str(WG.FIND_GMAX)]
    assert value("FIND_TILE") == ["FIND_T * FIND_BPT"] and int(value("FIND_T")[0]) * int(value("FIND_BPT")[0]) == WG.FIND_TILE


def test_restatement_equals_oracle(oracle):
    WG.check_restatement_equals_oracle(oracle)


def test_wrap_model(emu2, oracle):
    WG.check_wrap_model(oracle)


def test_big_model(emu2, oracle):
    WG.check_big_model(oracle, n_words=2000)


def test_duplicate_pair(emu2, oracle):
    WG.check_duplicate_pair(oracle)


def test_piece_edges(emu, oracle, request):
    sms = request.node.callspec.params["emu"]
    WG.check_piece_edges(oracle, 2 if sms == "2" else 1, step=3 if sms == "5" else 4)


def test_many_groups(emu, oracle, request):
    WG.check_many_groups(oracle, int(request.node.callspec.params["emu"]), small=True)


def test_misaligned_device_batches(emu, oracle):
    WG.check_misaligned_device_batches(oracle, dev=False)


def test_local_boundary(emu2, oracle):
    WG.check_local_boundary(oracle)


def test_long_boundary(emu, oracle):
    WG.check_long_boundary(oracle)


def test_token_counts(emu2, oracle):
    WG.check_token_counts(oracle)


def test_run_rule_across_chunks(emu, oracle):
    WG.check_run_rule_across_chunks(oracle, small=True)


def test_id0_long_words(emu2, oracle):
    WG.check_id0_long_words(oracle, small=True)


def test_more_long_words_than_blocks(emu, oracle, request):
    WG.check_more_long_words_than_blocks(oracle, int(request.node.callspec.params["emu"]), small=True)


def test_giant_words(emu2, oracle):
    WG.check_giant_words(oracle, [40_000])


def test_dropout_long_words(emu2, oracle):
    WG.check_dropout_long_words(oracle)


def test_chunk_cutter(emu2, oracle, monkeypatch):
    WG.check_chunk_cutter(oracle, monkeypatch, small=True)

"""Subword file encodes (tests/test_encode_file_subword_gpu.py 1 - 4) on the CPU under the SIMT emulator with 1, 2 and
5 SMs, at small sizes in 1 - 7 KB pieces: the subword layout kernel with its warp-wide copy of long pieces, <UNK> runs,
the dropout counter, the C ABI, misuse and failed calls run here."""
import pytest

import test_encode_file_subword_gpu as S
from youtokentome_b200 import _lib

SMS = ["1", "2", "5"]


@pytest.fixture(params=SMS, ids=["%s_sm" % s for s in SMS])
def lib(request, monkeypatch):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


def test_line_edges(lib):
    S.edges(lib, (1, 7), small=True)


def test_bos_eos_reverse(lib):
    S.flags(lib, (1,))


def test_unk_runs(lib):
    S.unk_runs(lib, (1, 7), small=True)


def test_long_pieces(lib):
    S.long_pieces(lib, (1,), small=True)


def test_special_ids_and_wide_model(lib):
    S.special_and_wide(lib, 1)


def test_dropout_counter(lib):
    S.dropout(lib, (1, 7), small=True)


def test_inputs(lib):
    S.inputs(lib, 1)


def test_abi_blocks(lib):
    S.abi_blocks(lib, small=True)


def test_abi_misuse(lib):
    S.abi_misuse(lib)


def test_failed_calls_leave_nothing(lib):
    S.failed_calls(lib)

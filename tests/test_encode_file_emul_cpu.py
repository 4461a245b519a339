"""File encodes (tests/test_encode_file_gpu.py 1 - 4) on the CPU under the SIMT emulator with 1, 2 and 5 SMs, at small
sizes in 1 - 7 KB pieces: the line split and its tile scan, the pieces that grow to hold a long line, the 16-bit and
text forms, the pipelined slots, the sink, the .npy writer and every misuse case run here."""
import pytest

import test_encode_file_gpu as F
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
    F.edges(lib, (1, 7), small=True)


def test_bos_eos_reverse(lib):
    F.flags(lib, 1)


def test_dropout_counter(lib):
    F.dropout(lib, (1, 7), small=True)


def test_wide_model_int32(lib):
    F.wide_ids(lib, 1)


def test_fifo_file_object_and_fd(lib):
    F.fifo(lib, 1)


def test_abi_blocks(lib):
    F.abi_blocks(lib, small=True)


def test_abi_misuse(lib):
    F.abi_misuse(lib)


def test_failed_calls_leave_nothing(lib):
    F.failed_calls(lib)

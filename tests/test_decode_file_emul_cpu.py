"""File decodes (tests/test_decode_file_gpu.py 1 - 3) on the CPU under the SIMT emulator with 1, 2 and 5 SMs, at small
sizes in 1 - 7 KB pieces: the id-text parser against `yttm decode`, the 16-bit widening, the newline-terminated decode,
the shared piece pipeline of both streams, the sink, the .npy reader and every misuse case run here."""
import pytest

import test_decode_file_gpu as F
from youtokentome_b200 import _lib

SMS = ["1", "2", "5"]


@pytest.fixture(params=SMS, ids=["%s_sm" % s for s in SMS])
def lib(request, monkeypatch):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


def test_parser_edges(lib):
    F.parser(lib, (1, 7), small=True)


def test_round_trips(lib):
    F.round_trips(lib, 1, small=True)


def test_inputs(lib):
    F.inputs(lib, 1)


def test_rejected_npy(lib):
    F.rejected(lib)


def test_out_of_range_ids(lib):
    F.out_of_range(lib, 1)


def test_abi_blocks(lib):
    F.abi(lib, small=True)


def test_abi_misuse(lib):
    F.abi_misuse(lib)

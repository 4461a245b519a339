"""Part A of tests/test_large_index_gpu.py under the SIMT emulator: every encode entry point on a batch of a few KB
whose offsets start at 2^31 - 3 ... 2^63 - 2^20 and cross 2^31 and 2^32 inside a word, against the same batch at base 0,
the span restatement, the padded and window definitions and the reference's dropout replay; with 1, 2 and 5 emulated
SMs."""
import pytest

import test_large_index_gpu as LI
from youtokentome_b200 import _lib


@pytest.fixture(params=["1", "2", "5"])
def emu(monkeypatch, request):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)  # what _lib.lib() hands to the Python BPE class
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


def test_absolute_offsets(emu, oracle):
    LI.check_bases(oracle)


def test_dropout_key_at_absolute_offsets(emu, oracle):
    LI.check_dropout_key(oracle)

"""The single-pass output kernel of device encode (emit_ids_kernel: per-tile id counts, a decoupled look-back over the
earlier tiles of EMIT_T = 256 sentences, then offsets, ids and spans) on the SIMT emulator with 1, 2 and 5 SMs.  Batch
shapes are chosen around the tile edges: one sentence, exactly one, two and many tiles, runs of empty and wordless
sentences across tile edges, sentences of more than 32 and more than 256 words, every bos / eos / reverse combination
in ids and spans mode, offsets[0] != 0 and dropout.

The emulator runs the blocks of a normal launch one after the other, so every look-back finds the tile right in front
of it published with its inclusive prefix.  Three branches of the look-back are therefore never taken here: the wait
for a tile that is not published yet, the sum over tiles that published only their own count, and a second window of
32 tiles further back.  Only the GPU tests (tests/test_encode_emit_gpu.py, many tiles running at once) reach them.
The emulated SM count does not change the output kernel's grid (one block per tile); it changes the grids of the
word finder and the dedup that produce the output kernel's input.

TEST HARNESS ONLY, like tests/test_simt_emul_cpu.py."""
import pytest

import test_encode_emit_gpu as EM
from youtokentome_b200 import _lib


@pytest.fixture(params=["1", "2", "5"])
def emu(monkeypatch, request):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


@pytest.mark.parametrize("n", [1, 255, 256, 257, 512, 1100])
def test_tile_counts(emu, oracle, n):
    EM.check_tile_counts(oracle, n)


def test_empty_runs_across_tile_edges(emu, oracle):
    EM.check_empty_runs(oracle)


def test_many_words_per_sentence(emu, oracle):
    EM.check_many_words(oracle)


def test_spans_all_flags_and_shift(emu, oracle):
    EM.check_spans(oracle, 300)


def test_dropout(emu, oracle):
    EM.check_dropout(oracle, 600)

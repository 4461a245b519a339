"""Fed trainings (tests/test_train_feed_gpu.py 1 - 3) on the CPU under the SIMT emulator with 1, 2 and 5 SMs, in pieces
of 1 - 4 KB: the per-piece word split and its overflow retry, the merge of each piece's words into the persistent table
(lookup, scan, insert), the arena and table growth and the final compaction all run here."""
import pytest

import test_train_feed_gpu as F
from _cases import zipf
from youtokentome_b200 import _lib, synth

SMS = ["1", "2", "5"]


@pytest.fixture(params=SMS, ids=["%s_sm" % s for s in SMS])
def lib(request, monkeypatch):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


@pytest.mark.parametrize("name", ["readme_small", "stress_17", "special_ids"])
def test_golden_corpora_fed(lib, name):
    F.parity(lib, [p for p in F.GOLDEN if p.endswith(name + ".json")][0], (1, 3))


@pytest.mark.parametrize("case", range(len(F.edge_corpora(small=True))), ids=[c[0] for c in F.edge_corpora(small=True)])
def test_edges_against_the_oracle(lib, oracle, case):
    _, text, vocab, cov, pieces = F.edge_corpora(small=True)[case]
    F.check_oracle(lib, oracle, text, vocab, cov, 1, pieces)


def test_fifo(lib):
    F.fifo(lib, synth.readme_corpus(n_lines=150), 250)


def test_memory_api_above_the_threshold(lib):
    F.memory_api(lib, zipf().text(20_000), 300)


def test_abi_blocks(lib):
    F.abi_blocks(lib, F.abi_text(small=True)[:12_000], 1)


def test_abi_misuse(lib):
    F.abi_misuse(lib)

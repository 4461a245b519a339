"""Word-count tables (tests/test_word_counts_gpu.py 1 - 3 and 5) on the CPU under the SIMT emulator with 1, 2 and 5
SMs, at small sizes: the weighted character pass and layout of word lists, their pieces, the per-piece insert and its
overflow retry, the merge into the persistent table, and the export of the fed words.  Device lists are host memory
here, which is what the emulated device reads."""
import numpy as np
import pytest

import test_train_feed_gpu as F
import test_word_counts_gpu as W
from youtokentome_b200 import _lib

SMS = ["1", "2", "5"]


@pytest.fixture(params=SMS, ids=["%s_sm" % s for s in SMS])
def lib(request, monkeypatch):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


@pytest.mark.parametrize("name", ["readme_small", "stress_17", "special_ids", "dirty_zipf_cov98"])
def test_round_trip_golden(lib, name):
    text, vocab, cov, special, _ = F.golden([p for p in F.GOLDEN if p.endswith(name + ".json")][0])
    W.round_trip(text, vocab, cov, piece_kbs=(None, 1), **W.special_ids(special))


@pytest.mark.parametrize("case", range(len(F.edge_corpora(small=True))), ids=[c[0] for c in F.edge_corpora(small=True)])
def test_round_trip_edges(lib, case):
    _, text, vocab, cov, _ = F.edge_corpora(small=True)[case]
    W.round_trip(text, vocab, cov, piece_kbs=(1,))


def test_counting_against_the_restatement(lib):
    for text in W.counting_corpora(small=True):
        W.check_counting(text, piece_kbs=(None, 1))


def test_tables_not_from_a_text(lib, oracle):
    W.tables_not_from_text(oracle, small=True)


def test_mixed_feed_at_the_abi(lib):
    W.abi_mixed(lib, np.ascontiguousarray, small=True)


def test_abi_misuse(lib):
    W.abi_misuse(lib)

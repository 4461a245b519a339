"""The training path of bench.py (tests/test_train_dist_gpu.py A - D) on the CPU under the SIMT emulator with 1, 2 and 5
SMs, at small sizes: the one-rank front through dist_export_words / dist_import_words, the export at 2, 3, 5 and 8 ranks
with every owner's import, crafted word lists (the freq x tokens limit included) and whole trainings through
train_distributed.  Also the restated owner balance on more than 10 000 unique words, which is deterministic."""
import os

import pytest

import _cases
import test_train_dist_gpu as TD
import test_train_front_gpu as FG
from youtokentome_b200 import _lib

SMS = ["1", "2", "5"]


@pytest.fixture(params=SMS, ids=["%s_sm" % s for s in SMS])
def lib(request, monkeypatch):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


def test_front_pieces_and_edges(lib):
    TD.check_front(lib, FG.corpus("chunk"), "chunk")
    TD.check_front(lib, FG.corpus("soup", small=True), "soup")
    TD.front_edges(lib, small=True)


@pytest.mark.parametrize("piece_kb", ["1", "3"])
def test_front_pipelined(lib, piece_kb):
    TD.front_pipelined(lib, piece_kb, small=True)


def test_front_word_table_overflow(lib):
    TD.front_overflow(lib, False)
    TD.front_overflow(lib, True)


def test_front_fed_shard(lib):
    TD.front_fed(lib, small=True)


@pytest.mark.parametrize("world", TD.WORLDS)
def test_export_and_owner_imports(lib, world):
    for name, text, fed in TD.export_corpora(small=True):
        TD.check_exports(lib, text, world, False, feed_rank=fed if fed is None else world - 1)


def test_owner_balance(lib):
    """More than 10 000 unique words: every owner gets between U/(2W) and 2U/W of them, at every world size."""
    text = FG.overflow_corpus()
    for world in TD.WORLDS:
        TD.check_exports(lib, text, world, False, balance=True)


def test_crafted_lists(lib, oracle):
    TD.crafted_duplicates(lib, False)
    TD.crafted_large_counts(lib, oracle, False)
    TD.crafted_edges(lib, oracle, False)


def test_crafted_count_limit(lib, oracle):
    TD.crafted_limits(lib, oracle, False)


@pytest.mark.parametrize("name", ["readme_small", "stress_17", "special_ids", "manual_japanese"])
def test_training_golden(lib, name):
    path = [p for p in TD.F.GOLDEN if os.path.basename(p) == name + ".json"][0]
    TD.golden_training(lib, path, sharded=name != "stress_17")


def test_training_stress_and_coverage(lib, oracle):
    for seed in range(4):
        text, vocab, cov, _ = _cases.stress_case(seed)
        TD.check_training(lib, text, vocab, cov, oracle=oracle)
    for cov in (1.0, 0.98, 0.9, 0.9999):
        TD.check_training(lib, _cases.dirty_zipf_text(30_000), 400, cov, oracle=oracle)


def test_training_special_layouts(lib, oracle):
    TD.special_layouts(lib, oracle, small=True)


@pytest.mark.parametrize("knob", TD.KNOBS, ids=["_".join(k) for k in TD.KNOBS])
def test_training_knobs(lib, oracle, knob):
    TD.knob_training(lib, oracle, knob, small=True)


def test_training_edges_and_errors(lib, oracle):
    TD.edge_trainings(lib, oracle, small=True)
    TD.error_texts(lib)


def test_sanitizer_script_dry_run():
    """tools/sanitize_train_dist.py on the emulator: the workload the GPU test runs under memcheck and racecheck."""
    import subprocess
    import sys
    from _bind import ROOT
    env = {k: v for k, v in os.environ.items() if not k.startswith(("YTTM_", "YT_EMU_"))}
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sanitize_train_dist.py"), "--emulate"], cwd=ROOT,
                       env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=900)
    out = r.stdout.decode(errors="replace")
    assert r.returncode == 0 and "checks identical to the restatement" in out, out[-1500:]

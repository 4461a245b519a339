"""Training contexts used again (tests/test_train_reuse_gpu.py (a) - (e)) on the CPU under the SIMT emulator, with
smaller inputs and 2 SMs.  The wrap of the exchange stamps (f) needs a million merges and stays on the GPU."""
import pytest

import test_train_reuse_gpu as RG
from test_train_reuse_gpu import kept  # noqa: F401 - the fixture, on this module's `lib`
from youtokentome_b200 import _lib


@pytest.fixture
def lib(monkeypatch):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", "2")
    return L


def test_kept_context_corpus_sizes(kept, oracle):  # noqa: F811
    RG.seq_sizes(kept, oracle, small=True)


def test_kept_context_alphabets(kept, oracle):  # noqa: F811
    RG.seq_alphabets(kept, oracle, small=True)


def test_kept_context_special_ids(kept, oracle):  # noqa: F811
    RG.seq_special_ids(kept, oracle, small=True)


def test_kept_context_resident_streaming(kept, oracle, monkeypatch):  # noqa: F811
    RG.seq_resident_streaming(kept, oracle, monkeypatch, small=True)


def test_kept_context_pair_table_growth(kept, oracle, monkeypatch):  # noqa: F811
    RG.seq_pair_table_growth(kept, oracle, monkeypatch, small=True)


def test_kept_context_compaction(kept, oracle):  # noqa: F811
    RG.seq_compaction(kept, oracle, small=True)


def test_kept_context_pipelined_and_plain(kept, oracle, monkeypatch):  # noqa: F811
    RG.seq_pipelined(kept, oracle, monkeypatch, small=True)


def test_error_after_pipelined_load_releases(lib, oracle, monkeypatch):
    RG.error_after_pipelined_load(lib, oracle, monkeypatch)


def test_error_on_exiting_thread_releases(lib, monkeypatch):
    monkeypatch.delenv(RG.KEEP, raising=False)
    RG.error_on_exiting_thread(lib)


def test_abi_two_corpora_on_one_context(lib, oracle):
    RG.abi_two_corpora(lib, oracle, small=True)


def test_abi_import_twice_on_one_context(lib, oracle):
    RG.abi_import_twice(lib, oracle, small=True)


def test_abi_calls_before_build_fail(lib, oracle):
    RG.abi_calls_before_build(lib, oracle)


def test_abi_device_load_after_abandoned_pipelined_load(lib):
    RG.abi_abandoned_pipelined_load(lib, dev=False)


def test_kept_context_seg_cap_and_geometry(kept, oracle, monkeypatch):  # noqa: F811
    RG.knob_seg_cap(kept, oracle, monkeypatch, small=True)


def test_kept_context_stage_times(kept, monkeypatch):  # noqa: F811
    RG.stage_times_training(kept, monkeypatch, small=True)


def test_encoder_handle_stage_times(lib, oracle):
    RG.stage_times_encoder(lib, oracle)

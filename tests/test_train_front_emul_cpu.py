"""The byte passes of training (tests/test_train_front_gpu.py) on the CPU under the SIMT emulator, at small sizes: the
adversarial pieces at every window offset, across warp and block boundaries and at the corpus ends, every length 0..70,
byte soup, device-resident corpora at base offsets 1..15, pipelined ingest, word-table overflow and pair-table growth.
Also the restatement itself: its scalar and vectorised decoders against each other, and against Python's decoder on
valid UTF-8."""
import collections

import numpy as np
import pytest

import _cases
import _front_ref as R
import test_train_front_gpu as FG
from youtokentome_b200 import _lib


@pytest.fixture
def emu(monkeypatch):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", "2")
    return L


# ---- the restatement ------------------------------------------------------------------------------------------------
def _small_inputs():
    return (FG.PIECES + FG.length_corpora() + FG.edge_corpora() + [FG.chunk_corpus(), FG.soup(30_000, seed=3)] +
            [bytes(np.random.default_rng(s).integers(0, 256, size=500, dtype=np.uint8)) for s in range(20)])


def test_scalar_and_vectorised_decoders_agree():
    for text in _small_inputs():
        units = R.decode_units(text)
        starts, cps = R.decode_units_np(text)
        assert starts.tolist() == [u[0] for u in units], text[:80]
        assert cps.tolist() == [-1 if u[2] is None else u[2] for u in units], text[:80]
        assert all(s + n == t for (s, n, _), (t, _, _) in zip(units, units[1:]))


def test_decoders_match_python_on_valid_utf8():
    rng = np.random.default_rng(4)
    cps = np.concatenate([rng.integers(0, 0xD800, 3000), rng.integers(0xE000, 0x110000, 3000),
                          [0x7F, 0x80, 0x7FF, 0x800, 0xD7FF, 0xE000, 0xFFFF, 0x10000, 0x10FFFF, 0x2581, 9, 10, 13, 32]])
    texts = ["".join(map(chr, cps.tolist())), _cases.zipf().text(50_000).decode()]
    for s in texts:
        b = s.encode()
        units = R.decode_units(b)
        assert [u[2] for u in units] == [ord(c) for c in s]
        _, np_cps = R.decode_units_np(b)
        assert np_cps.tolist() == [ord(c) for c in s]
        data_len, hist = R.char_hist(b)
        assert data_len == len(s)
        assert hist == dict(collections.Counter(ord(c) for c in s if ord(c) not in R.SPACE_CPS))
        assert R.byte_words(b) == [w.encode() for w in _split_words(s)]


def _split_words(s):
    """Maximal runs of non-space characters of a str."""
    out, cur = [], []
    for c in s:
        if ord(c) in R.SPACE_CPS:
            if cur:
                out.append("".join(cur))
            cur = []
        else:
            cur.append(c)
    if cur:
        out.append("".join(cur))
    return out


def test_restated_words_from_the_units():
    """byte_words (bytes.split after E2 96 81 -> space) against the definition: maximal runs of non-space units."""
    for text in _small_inputs():
        units = R.decode_units(text)
        words, cur = [], None
        for s, n, cp in units:
            if cp in R.SPACE_CPS:
                if cur is not None:
                    words.append(text[cur:s])
                cur = None
            elif cur is None:
                cur = s
        if cur is not None:
            words.append(text[cur:])
        assert R.byte_words(text) == words, text[:80]


# ---- the kernels on the emulator ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["chunk", "warp", "block", "soup"])
def test_adversarial_pieces(emu, name):
    FG.check_pieces(emu, name, small=True)


def test_pieces_at_the_corpus_ends(emu):
    FG.check_edges(emu)


def test_corpus_lengths_0_to_70(emu):
    FG.check_lengths(emu)


def test_prefix_word_with_an_equal_tag(emu):
    FG.check_prefix_with_equal_tag(emu)


@pytest.mark.parametrize("off", range(1, 16))
def test_device_corpus_at_a_misaligned_base(emu, off):
    FG.check_misaligned(emu, off, ["chunk"], lengths=off in (1, 7, 15))


@pytest.mark.parametrize("piece_kb", ["1", "3", "64"])
def test_pipelined_ingest(emu, piece_kb):
    FG.check_pipelined(emu, piece_kb, ["chunk", "soup"], small=True)


def test_pipelined_no_space(emu):
    FG.check_no_space(emu)


@pytest.mark.parametrize("pipelined", [False, True])
def test_word_table_overflow(emu, pipelined):
    FG.check_overflow(emu, pipelined)


def test_initial_pair_table(emu):
    FG.check_pair_table(emu)


def test_pair_table_grown_from_a_small_floor(emu):
    FG.check_pair_table(emu, "16")


def test_sanitizer_script_dry_run():
    """tools/sanitize_train_front.py on the emulator: the workload the GPU test runs under memcheck."""
    import os
    import subprocess
    import sys
    from _bind import ROOT
    env = {k: v for k, v in os.environ.items() if not k.startswith(("YTTM_", "YT_EMU_"))}
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sanitize_train_front.py"), "--emulate"], cwd=ROOT,
                       env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    out = r.stdout.decode(errors="replace")
    assert r.returncode == 0 and "checks identical to the restatement" in out, out[-1500:]

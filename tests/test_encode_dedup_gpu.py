"""The word dedup of device encode (dedup_words_kernel in youtokentome_b200/csrc/encode.cu): an open-addressed claim
table elects one representative occurrence per distinct word, and a tag match is verified byte by byte against the
representative.  The check bodies build batches that hit each path: one word repeated thousands of times, thousands
of distinct words, tables forced small with YTTM_ENC_DEDUP_SLOTS (1, 8, 64 slots) so that most words find no room and
represent themselves, equal tags everywhere (YTTM_ENC_DEDUP_WEAKTAG: every probe ends in the byte compare), pairs that
differ only after byte 16 or 32 and prefix pairs, and repeats of a representative of more than LONG_W slots.  The ids
are compared with the oracle; tests/test_encode_dedup_emul_cpu.py runs the same bodies under the SIMT emulator."""
import numpy as np
import pytest

import _cases
import test_encode_gpu as EG
from _gpu import GpuEncoder

pytestmark = pytest.mark.gpu

N = 1024
SP = b"\xe2\x96\x81"
_models = {}
KWS = [dict(), dict(bos=True, eos=True, reverse=True)]


def _model(oracle):
    if "zipf" not in _models:
        _models["zipf"] = EG._model(oracle, _cases.dirty_zipf_text(), 1500)
    return _models["zipf"]


def _same(oracle, sents, kws=KWS):
    m = _model(oracle)
    g, o = GpuEncoder(m), oracle.encoder(m)
    for kw in kws:
        assert g.encode(sents, **kw) == o.encode(sents, **kw), kw


def _word(rng, n):
    parts = [b"a", b"b", b"c", b"d", "ж".encode(), "☃".encode(), b"\xff"]
    return b"".join(parts[i] for i in rng.integers(0, len(parts), n))[:n]


def _distinct(rng, k):
    out = set()
    while len(out) < k:
        out.add(_word(rng, int(rng.integers(3, 20))))
    return sorted(out)


def check_repeated_and_distinct(oracle):
    """One word repeated, every word distinct, and both in one batch."""
    rng = np.random.default_rng(1)
    one = [b" ".join([b"abcab"] * 3 * N)]
    _same(oracle, one)
    d = _distinct(rng, 3 * N)
    _same(oracle, [b" ".join(d[i:i + 50]) for i in range(0, len(d), 50)] + one + [b" ".join(d[:N])])


def check_pairs(oracle):
    """Words that equal another word up to byte 15 / 16 / 17 / 31 / 32 / 33 / 47 / 48, prefix pairs that end at the
    sentence end, before a space or before U+2581, and repeats of words at every alignment mod 16."""
    rng = np.random.default_rng(5)
    sents = []
    for k in (15, 16, 17, 31, 32, 33, 47, 48):
        w = _word(rng, k + 9)
        x, y = w[:k] + b"x" + w[k + 1:], w[:k] + b"y" + w[k + 1:]
        sents += [x + b" " + y, b"z" + y + b" " + x, b"zz " + x + SP + y, y, x, b" ".join([x, y] * 9)]
    for k in (1, 2, 15, 16, 17, 31, 32, 33):
        w = _word(rng, k)
        sents += [w, w + b"z " + w, w + b" " + w + b"z", w + SP + w + b"z" + SP, w + b"z", b"q" + SP + w,
                  w + b"\xe2\x96", w + b"\xe2\x96 " + w, b"  " + w + b"z" + SP[:2]]
    for n in range(1, 40):
        w = _word(rng, n)
        sents.append(b" ".join(b" " * (i % 16) + w for i in range(6)))
    _same(oracle, sents + sents[::-1] + sents)


def check_long_leader(oracle):
    """Repeats, near and far, of a representative of more than LONG_W = 512 slots, and a long word next to one that
    differs in its last byte."""
    rng = np.random.default_rng(7)
    big = _word(rng, 700)
    other = big[:-1] + (b"a" if big[-1:] != b"a" else b"b")
    fill = [b" ".join(_cases.zipf_sentences(40, seed=3))]
    _same(oracle, [big + b" " + big, b"x " + big, other + b" " + big] + fill + [big, other, b" ".join([big] * 5)])


def check_small_tables(oracle, monkeypatch, slots, weak):
    """The table capped by YTTM_ENC_DEDUP_SLOTS (1, 8, 64 slots): most words find no room and represent themselves;
    with weak tags every probe compares bytes."""
    monkeypatch.setenv("YTTM_ENC_DEDUP_SLOTS", str(slots))
    if weak:
        monkeypatch.setenv("YTTM_ENC_DEDUP_WEAKTAG", "1")
    rng = np.random.default_rng(slots)
    d = _distinct(rng, 300)
    sents = _cases.zipf_sentences(200, seed=slots) + [b" ".join(d[i:i + 30]) for i in range(0, 300, 30)]
    sents += [b" ".join([b"abcab"] * 200), b" ".join(d[:20] * 10)]
    _same(oracle, sents)


def test_repeated_and_distinct(product, oracle):
    check_repeated_and_distinct(oracle)


def test_pairs(product, oracle):
    check_pairs(oracle)


def test_long_leader(product, oracle):
    check_long_leader(oracle)


@pytest.mark.parametrize("slots", [1, 8, 64])
@pytest.mark.parametrize("weak", [False, True])
def test_small_tables(product, oracle, monkeypatch, slots, weak):
    check_small_tables(oracle, monkeypatch, slots, weak)

"""BPE-dropout pinned to the unmodified reference.  The reference draws its dropout decisions from a global mt19937
(bpe.cpp:1415); oracle/_ref/libyttm_ref_replay.so is the reference with that generator replaced by one that hands out
the product's Philox draws (oracle/replay_rng.h), so its own DropoutQueue decides given the same draws
(tests/_dropout_ref.py).  Here the replay checks itself, and the oracle (oracle/bpe_oracle.cpp, which the GPU tests of
older dropout paths compare with) is compared with it: stress cases, the golden texts, dirty Zipf text, both layouts
that give U+2581 the id 0, and the boundary of the skip test, where the draw r sits just below p * 2^32."""
import numpy as np
import pytest

import _cases
import _dropout_ref as DR
from _bind import read_model, replay_engine, tmp_model_path
from _front_ref import SPACE_CP
from youtokentome_b200 import synth

P = [0.125, 0.5, 0.1, 0.9, 1.0]
KWS = [dict(), dict(bos=True, eos=True), dict(reverse=True, eos=True), dict(bos=True, reverse=True)]


def _model(oracle, text, vocab, cov=1.0, **special):
    m = tmp_model_path("orc")
    oracle.train(text, m, vocab, cov, **special)
    return m


def _same(reference, oracle, m, sents, p, seed, first, kw):
    want = DR.replayed(reference, m, sents, p, seed, first, **kw)
    got = oracle.encoder(m).encode(sents, dropout=p, seed=seed, first_index=first, **kw)
    assert got == want, (p, seed, first, kw)
    return want


# ---- the replay itself ---------------------------------------------------------------------------------------------

def test_python_philox_known_answers():
    """Random123's published answers for Philox4x32-10 (kat_vectors)."""
    assert DR.philox4x32_10((0, 0, 0, 0), (0, 0)) == (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)
    f = 0xFFFFFFFF
    assert DR.philox4x32_10((f, f, f, f), (f, f)) == (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)
    assert DR.philox4x32_10((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0)) == \
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)


def test_engine_is_python_philox():
    """The engine the reference draws from answers 0, r_0, 0, r_1, ..., and uniform_real_distribution<>(0, 1) makes
    exactly r_k / 2^32 of it: the reference skips iff r_k / 2^32 < p."""
    rng = np.random.default_rng(5)
    keys = [(0, 0, 0), (2**64 - 1, 2**64 - 1, 2**32 - 1), (0xa4093822299f31d0, 0x03707344_13198a2e, 0x85a308d3)]
    keys += [(int(rng.integers(0, 2**63)) * 2 + 1, int(rng.integers(0, 2**63)), int(rng.integers(0, 2**32)))
             for _ in range(6)]
    for seed, sent, off in keys:
        words, canon = replay_engine(seed, sent, off, 6)
        want = [DR.draw(seed, sent, off, k) for k in range(6)]
        assert words[0::2] == [0] * 6 and words[1::2] == want
        assert canon == [r / 2**32 for r in want]
    seed, sent, off = 0x299f31d0a4093822, 0x85a308d3243f6a88, 0x13198a2e
    assert DR.draw(seed, sent, off, 0x03707344) == 0xd16cfe09   # the third known answer, as a draw


def test_sentence_words_keys():
    s = b"\xc0\xafab  c\xe2\x96\x81d\xffe\t\xff \xf0\x9f\x98\x80"
    assert DR.sentence_words(s) == [(0, b"\xc0\xafab"), (6, b"c"), (10, b"d\xffe"), (14, b"\xff"), (16, s[16:])]
    assert DR.sentence_words(b"") == [] and DR.sentence_words(b" \n ") == []


def test_p1_gives_characters(reference, oracle):
    """p = 1 skips every event: every word is its characters, and it takes one draw per pair that has a rule."""
    text = synth.stress_text(3)
    m = _model(oracle, text, len(set(text) | {32}) + 4 + 30)
    c2i, rules, _ = read_model(m)
    rule_of = {(x, y) for x, y, _ in rules}
    sents = [synth.stress_text(3 * 7 + k, 300) for k in range(6)]
    words = DR.replay_batch(reference, m, sents, 1.0, 7, 0)
    n = 0
    for s, ws in zip(sents, words):
        for (_, w), got in zip(DR.sentence_words(s), ws):
            chars = [c2i[SPACE_CP]] + [c2i[ord(ch)] for ch in w.decode()]
            assert got["ids"] == chars
            assert got["draws"] == sum((a, b) in rule_of for a, b in zip(chars, chars[1:]))
            n += got["draws"] > 1
    assert n > 20


@pytest.mark.parametrize("name", sorted(synth.GOLDEN_TEXTS))
def test_tiny_p_is_the_reference_without_dropout(reference, name):
    """p = 2^-40 skips only at r = 0: the replay equals the reference at dropout 0."""
    train, test, vocab = synth.GOLDEN_TEXTS[name]
    m = tmp_model_path("ref")
    reference.train(train.encode(), m, vocab, 1.0)
    sents = [test.encode()] + _cases.EDGE_SENTENCES
    for kw in KWS:
        assert DR.replayed(reference, m, sents, 2.0**-40, 11, 0, **kw) == reference.encoder(m).encode(sents, **kw)


# ---- the oracle against the replayed reference ---------------------------------------------------------------------

@pytest.mark.parametrize("seed", range(60))
def test_stress(reference, oracle, seed):
    text, vocab, cov, sents = _cases.stress_case(seed)
    try:
        m = _model(oracle, text, vocab, cov)
    except ValueError:
        return
    sents = sents + _cases.EDGE_SENTENCES
    for j, p in enumerate([P[seed % 5], P[(seed + 2) % 5]]):
        _same(reference, oracle, m, sents, p, (seed << 33) + 17 * j, seed * 1000, KWS[(seed + j) % 4])


@pytest.mark.parametrize("name", sorted(synth.GOLDEN_TEXTS))
def test_golden_texts(reference, oracle, name):
    train, test, vocab = synth.GOLDEN_TEXTS[name]
    m = _model(oracle, train.encode(), vocab)
    for j, p in enumerate(P):
        _same(reference, oracle, m, [test.encode()] * 3, p, 2**40 + j, 2**32 - 2, KWS[j % 4])


@pytest.mark.parametrize("cov", [1.0, 0.98, 0.9])
def test_dirty_zipf(reference, oracle, cov):
    m = _model(oracle, _cases.dirty_zipf_text(), 1500, cov)
    sents = _cases.zipf_sentences(60) + _cases.EDGE_SENTENCES
    for j, p in enumerate(P):
        _same(reference, oracle, m, sents, p, 99 + j, 5 * j, KWS[j % 4])


@pytest.mark.parametrize("special", [dict(pad=-1, unk=1, bos=2, eos=3), dict(pad=-1, unk=5, bos=-1, eos=-1)])
def test_space_id_zero(reference, oracle, special):
    """U+2581 at id 0: a word whose leading "▁" is never merged loses it, with dropout too."""
    text = _cases.zipf().text(60_000) + b" zab zab ab z zz z q"
    vocab = len(set(text.decode().replace("\n", " ").replace(" ", ""))) + 5 + 25
    m = _model(oracle, text, vocab, **special)
    assert read_model(m)[0][SPACE_CP] == 0
    sents = _cases.zipf_sentences(40) + list(_cases.EDGE_SENTENCES) + [b"zab", b"z", b"q z zz", "▁▁z".encode()]
    for j, p in enumerate(P):
        kw = KWS[j % 4] if special["bos"] != -1 else dict(reverse=bool(j % 2))
        _same(reference, oracle, m, sents, p, 3 + j, 0, kw)


# ---- the boundary of the skip test ---------------------------------------------------------------------------------

def boundary_cases(reference, m, words, want_r):
    """For each target in want_r ("low", "mid", "high"), a one-word sentence and a sentence index whose first draw r
    lies in that range, such that the reference's ids at p = (r + 0.5) / 2^32 (first event skipped) differ from those at
    p = r / 2^32 (not skipped).  Returns [(word, index, seed, r, ids at p = (r + 0.5) / 2^32, ids at p = r / 2^32)]."""
    ranges = {"low": (0, 2**24), "mid": (2**31 - 2**24, 2**31 + 2**24), "high": (2**32 - 2**24, 2**32 - 1)}
    seed, out = 0x5eed_0000_0001, []
    for target in want_r:
        lo, hi = ranges[target]
        found = None
        for idx in range(1 << 16):
            r = DR.draw(seed, idx, 0, 0)
            if not lo <= r < hi:
                continue
            for w in words:
                skip = DR.replayed(reference, m, [w], (r + 0.5) / 2**32, seed, idx)
                keep = DR.replayed(reference, m, [w], r / 2**32, seed, idx)
                if skip != keep:
                    found = (w, idx, seed, r, skip, keep)
                    break
            if found:
                break
        assert found, target
        out.append(found)
    return out


def boundary_model(oracle):
    text = b"abc abc abc bcd bcd abcd abcd abcd aab aab aaab " * 20 + b"xyzw xyz yzw " * 9
    return _model(oracle, text, 4 + 1 + 8 + 14)


BOUNDARY_WORDS = [b"abcd", b"aaab", b"xyzw", b"abcabcd"]


def test_skip_boundary(reference, oracle):
    """r = the first draw of a word and p = (r + 0.5) / 2^32: the reference skips (r / 2^32 < p) while a threshold of
    floor(p * 2^32) = r does not.  At p = r / 2^32 exactly it does not skip (a skip test of r <= threshold would).
    Draws small, middling and close to 2^32."""
    m = boundary_model(oracle)
    enc = oracle.encoder(m)
    for w, idx, seed, r, skip, keep in boundary_cases(reference, m, BOUNDARY_WORDS, ["low", "mid", "high"]):
        assert enc.encode([w], dropout=(r + 0.5) / 2**32, seed=seed, first_index=idx) == skip, (w, idx, r)
        assert enc.encode([w], dropout=r / 2**32, seed=seed, first_index=idx) == keep, (w, idx, r)

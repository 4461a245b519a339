"""Word lengths from the finder in the word dedup of device encode (youtokentome_b200/csrc/encode.cu): find_words_vec_kernel
records each word's length, or WORD_LEN_ESC when the word's end lies beyond the staged piece, and dedup_words_kernel
hashes and compares exactly that many bytes against the position and length kept in the claimed table slot.  Every
case repeats its words in short sentences, so that occurrences whose length the finder knew meet occurrences that
scanned for their end, in both orders, and the ids are compared with the oracle:
  words ending one byte before, at and one byte after a piece edge, and U+2581 straddling the edge;
  groups longer than a piece and single sentences of 100 KB;
  words of WORD_LEN_ESC - 1 .. WORD_LEN_ESC + 1 bytes;
  device batches at base addresses 1 .. 15 mod 16 whose offsets start above 0;
  words of equal length that differ only in their last byte, with equal tags everywhere and with 1- and 8-slot tables.
tests/test_encode_dedup_len_emul_cpu.py runs the same bodies under the SIMT emulator, at smaller sizes."""
import numpy as np
import pytest

import _cases
import test_encode_words_gpu as WG
from _bind import _pack

pytestmark = pytest.mark.gpu

FIND_TILE = WG.FIND_TILE
WORD_LEN_ESC = 0xFFFF  # the escape length of encode.cu
SP = b"\xe2\x96\x81"
KWS = [dict(), dict(bos=True, eos=True, reverse=True)]


def same(case, sents, kws=KWS):
    for kw in kws:
        assert case.g.encode(sents, **kw) == case.o.encode(sents, **kw), kw


def _filler(n, seed):
    return WG._zipf_text(n, seed)


def check_piece_edges(oracle, edges=(1, 2)):
    """A word that ends 2 bytes before .. 2 bytes after the `edge`-th piece edge of a group of one long sentence (the
    group starts at batch byte 0, aligned: the edges are the multiples of 16 384), before a space, before U+2581 whose
    bytes straddle the edge, or at the sentence end; the same words again in short sentences after it."""
    case = WG.zipf_case(oracle)
    rng = np.random.default_rng(3)
    for edge in edges:
        for d in range(-2, 3):
            w = WG._word(rng, int(rng.integers(5, 40)))
            at = edge * FIND_TILE + d - len(w)  # the word is bytes [at, at + len(w)) of the long sentence
            head = _filler(at - 1, 100 + d) + b" "
            short = [b"x " + w + b" y", w]
            for after in (b" z", SP + b"z", b""):
                same(case, [head + w + after] + short + [w + after])
            for k in (1, 2):  # U+2581 whose first k bytes lie in front of the edge
                hk = _filler(edge * FIND_TILE - k - len(w) - 1, 200 + k) + b" "
                same(case, [hk + w + SP + w, w + SP] + short)


def check_long_groups(oracle, small=False):
    """Groups longer than a piece: single sentences of 100 KB (40 KB on the emulator), a group of 1 - 3 KB sentences,
    and the words of all of them in short sentences."""
    case = WG.zipf_case(oracle)
    n = 40_000 if small else 100_000
    big = [_filler(n, 7), _filler(n, 8)]
    words = sorted(set(b" ".join(big).split()))
    short = [b" ".join(words[i:i + 20]) for i in range(0, len(words), 20)]
    rng = np.random.default_rng(9)
    many = [_filler(int(k), 30 + i) for i, k in enumerate(rng.integers(1000, 3000, 12 if small else 40))]
    same(case, short[:40] + big + short + many + big[:1], kws=KWS[:1])
    same(case, big[::-1] + short[::-1], kws=KWS[1:])


def check_escape_lengths(oracle):
    """Words of WORD_LEN_ESC - 1, WORD_LEN_ESC and WORD_LEN_ESC + 1 bytes (longer than a piece, so their occurrences
    find their ends by the scan), each twice, and the same words with one more byte."""
    case = WG.abcd_case(oracle)
    rng = np.random.default_rng(11)
    base = bytes(rng.choice(list(b"abcd"), size=WORD_LEN_ESC + 2).tolist())
    for n in (WORD_LEN_ESC - 1, WORD_LEN_ESC, WORD_LEN_ESC + 1):
        w = base[:n]
        same(case, [w + b" " + w, b"ab " + w, base[:n + 1] + b" " + w], kws=KWS[:1])


def check_misaligned_batches(oracle, dev):
    """Device batches whose base address is 1 .. 15 mod 16 and whose offsets start above 0: words of 1 .. 40 bytes
    repeated at every alignment, and a word that ends at the batch's last byte."""
    case = WG.zipf_case(oracle)
    rng = np.random.default_rng(13)
    for shift in range(1, 16):
        words = [WG._word(rng, n) for n in range(1, 41)]
        sents = [b" " * (i % 16) + b" ".join(words[i:] + words[:i]) for i in range(0, 40, 3)]
        sents += _cases.zipf_sentences(20, seed=shift) + [b"q " + words[shift]]
        buf, offs = _pack(sents)
        for kw in KWS:
            got = WG._device(case.g, buf, offs, shift, 5 * shift, dev, kw)
            WG._equal(got, case.o.encode(sents, **kw), sents, (shift, kw))


def check_last_byte_pairs(oracle, monkeypatch, slots, weak):
    """Words of 1 .. 48 bytes that equal another word of the same length up to their last byte, each repeated; with
    equal tags everywhere every probe that meets the other word compares all of its bytes."""
    if slots:
        monkeypatch.setenv("YTTM_ENC_DEDUP_SLOTS", str(slots))
    if weak:
        monkeypatch.setenv("YTTM_ENC_DEDUP_WEAKTAG", "1")
    case = WG.zipf_case(oracle)
    rng = np.random.default_rng(17)
    sents = []
    for n in range(1, 49):
        w = WG._word(rng, n, (b"a", b"b", b"c", b"d"))
        x, y = w[:-1] + b"x", w[:-1] + b"y"
        sents += [x + b" " + y, y + b" " + x + b" " + x, b" " * (n % 16) + y, x + SP + y]
    same(case, sents + sents[::-1])


def test_piece_edges(product, oracle):
    check_piece_edges(oracle)


def test_long_groups(product, oracle):
    check_long_groups(oracle)


def test_escape_lengths(product, oracle):
    check_escape_lengths(oracle)


def test_misaligned_batches(product, oracle):
    check_misaligned_batches(oracle, dev=True)


@pytest.mark.parametrize("slots", [0, 1, 8])
@pytest.mark.parametrize("weak", [False, True])
def test_last_byte_pairs(product, oracle, monkeypatch, slots, weak):
    check_last_byte_pairs(oracle, monkeypatch, slots, weak)

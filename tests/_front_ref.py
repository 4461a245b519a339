"""A plain restatement of the two byte passes at the start of training: the code-point histogram with `data_len`
(char_hist_kernel) and the word split / dedup / tokenisation (word_insert_kernel, word_compact_kernel,
word_tokens_kernel), plus the initial pair table built from the unique words (pair_hist_kernel).

It restates the serial semantics of decode_unit / space_at / word_start_at (csrc/bpe_core.cuh: utf8.cpp's iterator
and compute_word_count of bpe.cpp) without any of the kernels' position-parallel tricks: `decode_units` walks the bytes
one unit at a time, `decode_units_np` is a vectorised form of the same walk for inputs of many MB, and the words come
from `bytes.split`."""
import collections

import numpy as np

SPACE_CP = 0x2581                     # U+2581, the word separator of the model files
SPACE_CPS = frozenset([0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x20, SPACE_CP])
U2581 = b"\xe2\x96\x81"
_MIN_CP = {2: 0x80, 3: 0x800, 4: 0x10000}   # smaller values are overlong encodings


def _seq_len(b0):
    """Length a lead byte announces (0: not a lead byte)."""
    if b0 < 0x80:
        return 1
    if 0xC0 <= b0 <= 0xDF:
        return 2
    if 0xE0 <= b0 <= 0xEF:
        return 3
    if 0xF0 <= b0 <= 0xF7:
        return 4
    return 0


def decode_units(data):
    """The serial decode: a list of (start, length, code point or None) per unit.  A valid sequence advances by its
    length; anything else (overlong, surrogate, above U+10FFFF, truncated, a lead without its continuations, a stray
    continuation, 0xF8..0xFF) is one invalid unit of one byte."""
    out, i, n = [], 0, len(data)
    while i < n:
        b0 = data[i]
        L = _seq_len(b0)
        cp, size = None, 1
        if L == 1:
            cp = b0
        elif L and i + L <= n and all(0x80 <= data[i + k] <= 0xBF for k in range(1, L)):
            v = b0 & (0x7F >> L)
            for k in range(1, L):
                v = (v << 6) | (data[i + k] & 0x3F)
            if v >= _MIN_CP[L] and v <= 0x10FFFF and not 0xD800 <= v <= 0xDFFF:
                cp, size = v, L
        out.append((i, size, cp))
        i += size
    return out


def decode_units_np(data):
    """decode_units for inputs of many MB: (unit start positions, code point per unit or -1 for an invalid unit).

    Valid multi-byte sequences consist of one lead byte followed by continuation bytes only, so a byte that is not a
    continuation always starts a unit (no valid sequence can swallow it), and the valid sequences are exactly those
    that start at such a byte.  Hence the units are the bytes that no valid multi-byte sequence covers beyond its
    lead, which needs no serial walk."""
    b = np.frombuffer(bytes(data), dtype=np.uint8)
    n = len(b)
    x = np.concatenate([b, np.zeros(3, dtype=np.uint8)]).astype(np.uint32)   # bytes past the end: no continuation
    c1, c2, c3 = x[1:n + 1], x[2:n + 2], x[3:n + 3]
    is_c = lambda v: (v & 0xC0) == 0x80                                        # noqa: E731
    b0 = x[:n]
    cp2 = ((b0 & 0x1F) << 6) | (c1 & 0x3F)
    cp3 = ((b0 & 0x0F) << 12) | ((c1 & 0x3F) << 6) | (c2 & 0x3F)
    cp4 = ((b0 & 0x07) << 18) | ((c1 & 0x3F) << 12) | ((c2 & 0x3F) << 6) | (c3 & 0x3F)
    ok2 = (b0 >= 0xC0) & (b0 <= 0xDF) & is_c(c1) & (cp2 >= 0x80)
    ok3 = (b0 >= 0xE0) & (b0 <= 0xEF) & is_c(c1) & is_c(c2) & (cp3 >= 0x800) & ((cp3 < 0xD800) | (cp3 > 0xDFFF))
    ok4 = (b0 >= 0xF0) & (b0 <= 0xF7) & is_c(c1) & is_c(c2) & is_c(c3) & (cp4 >= 0x10000) & (cp4 <= 0x10FFFF)
    # (a sequence "valid" at a continuation byte cannot exist: the lead byte ranges above exclude 0x80..0xBF)
    covered = np.zeros(n + 3, dtype=bool)
    for ok, L in ((ok2, 2), (ok3, 3), (ok4, 4)):
        at = np.nonzero(ok)[0]
        for k in range(1, L):
            covered[at + k] = True
    starts = np.nonzero(~covered[:n])[0]
    cp = np.full(n, -1, dtype=np.int64)
    ascii_ = b0 < 0x80
    cp[ascii_] = b0[ascii_]
    for ok, v in ((ok2, cp2), (ok3, cp3), (ok4, cp4)):
        cp[ok] = v[ok]
    return starts, cp[starts]


def char_hist(data):
    """(data_len, {code point: count}): data_len counts every unit (spaces and invalid units too); the histogram
    counts the valid code points that are not spaces (0x09..0x0D, 0x20, U+2581)."""
    _, cps = decode_units_np(data)
    keep = cps >= 0
    for s in SPACE_CPS:
        keep &= cps != s
    cnt = np.bincount(cps[keep], minlength=0)
    nz = np.nonzero(cnt)[0]
    return len(cps), dict(zip(nz.tolist(), cnt[nz].tolist()))


def byte_words(data):
    """Word occurrences as raw byte strings.  A word is a maximal run of non-space units.  `bytes.split()` splits at
    exactly the six ASCII space bytes, and every such byte is a space unit of its own (an ASCII byte never belongs to a
    multi-byte sequence); E2 96 81 is always the unit U+2581 (E2 is no continuation byte, so a unit starts there, and
    the three bytes are its valid encoding) and is the only encoding of U+2581.  So turning each E2 96 81 into one
    space and splitting on whitespace cuts at the space units and nowhere else.  No unit crosses a cut either: the byte
    after a word is ASCII or E2, neither of which continues a sequence."""
    return bytes(data).replace(U2581, b" ").split()


def word_tokens(word, cp2id, space_id):
    """[space_id] + the id of each kept code point of one byte-word; invalid and removed units vanish.  None when no
    unit is kept (the word is dropped)."""
    ids = [cp2id[cp] for _, _, cp in decode_units(word) if cp is not None and cp in cp2id]
    return (space_id, *ids) if ids else None


def run_pairs(tokens, freq, out):
    """Add a word's pairs to `out` under the run rule: a run a^L gives floor(L/2) pairs (a, a) and every run boundary
    one cross pair (key = a << 32 | b), each weighted by the word's frequency."""
    i = 0
    while i < len(tokens):
        j = i
        while j < len(tokens) and tokens[j] == tokens[i]:
            j += 1
        if j - i >= 2:
            out[(tokens[i] << 32) | tokens[i]] += (j - i) // 2 * freq
        if j < len(tokens):
            out[(tokens[i] << 32) | tokens[j]] += freq
        i = j


def expected_front(data, cp2id, space_id):
    """Everything the byte passes and the initial pair table give, for an alphabet cp2id ({code point: id})."""
    data_len, hist = char_hist(data)
    return dict(expected_words(collections.Counter(byte_words(data)), cp2id, space_id), data_len=data_len, hist=hist)


def expected_words(uniq, cp2id, space_id):
    """The word fields of expected_front for a set of byte-words with counts ({byte-word: count})."""
    words = []
    for w, f in uniq.items():
        t = word_tokens(w, cp2id, space_id)
        if t is not None:
            words.append((t, f))
    words.sort()
    pairs = collections.Counter()
    for t, f in words:
        run_pairs(t, f, pairs)
    return dict(n_words=sum(uniq.values()), n_unique=len(words), n_tokens=sum(len(t) for t, _ in words), words=words,
                pairs=dict(pairs))

"""The two byte passes at the start of training on the GPU — the code-point histogram with data_len (char_hist_kernel)
and the word split / dedup / tokenisation (word_insert_kernel, word_compact_kernel, word_tokens_kernel) with the
initial pair table built from their words — against the plain restatement of tests/_front_ref.py, field by field:
histogram, data_len, word occurrences, the multiset of (tokens, frequency) of the unique words and the pair table.

Inputs: adversarial UTF-8 pieces at every offset around a 16-byte chunk, across 512-byte warp and 8 KB block
boundaries and at both ends of the corpus; every corpus length 0..70; random byte soup; device-resident corpora at
base offsets 1..15; pipelined ingest with 1, 3 and 64 KB pieces and one corpus of 80 MB at the default 32 MB pieces;
a word table that overflows (plain and pipelined); a pair table that has to grow.  The bodies take the library and
`dev`: tests/test_train_front_emul_cpu.py runs them on the SIMT emulator with dev=False (device memory is host memory
there) and smaller inputs."""
import collections
import contextlib
import ctypes as C
import functools
import os

import numpy as np
import pytest

import _cases
import _front_ref as R
from youtokentome_b200 import _lib, synth

pytestmark = pytest.mark.gpu

SPACE_ID = 4

# ---- adversarial pieces --------------------------------------------------------------------------------------------
PIECES = [
    # valid characters at the length boundaries of UTF-8 and around the surrogates
    b"\x7f", b"\xc2\x80", b"\xdf\xbf", b"\xe0\xa0\x80", b"\xed\x9f\xbf", b"\xee\x80\x80", b"\xef\xbf\xbf",
    b"\xf0\x90\x80\x80", b"\xf4\x8f\xbf\xbf", b"\xc3\xa9\xe2\x82\xac\xf0\x9f\x98\x80",
    # overlong, surrogate, above U+10FFFF, leads that are never valid
    b"\xc0\xaf", b"\xc1\xbf", b"\xe0\x80\xaf", b"\xe0\x9f\xbf", b"\xf0\x80\x80\xaf", b"\xf0\x8f\xbf\xbf", b"\xed\xa0\x80",
    b"\xed\xbf\xbf", b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xf7\xbf\xbf\xbf", b"\xf8\x88\x80\x80\x80",
    b"\xfc\x84\x80\x80\x80\x80", b"\xfe", b"\xff",
    # stray continuations, continuations behind a complete sequence, truncated sequences
    b"\x80", b"\xbf\xbf", b"\x80\x80\x80\x80\x80", b"\xc3\xa9\x80", b"\xe2\x82\xac\xbf", b"\xf0\x9f\x98\x80\x80\x80",
    b"\xc3", b"\xe0\xa0", b"\xe2\x96", b"\xf0", b"\xf0\x9f", b"\xf0\x9f\x98", b"\xf4\x8f\xbf",
    # a lead followed by a space or by U+2581
    b"\xc3 ", b"\xe2\x96 ", b"\xf0\x9f\x98\n", b"\xc3\xe2\x96\x81", b"\xf0\x9f\xe2\x96\x81", b"\xe2\xe2\x96\x81",
    b"\xe2\x96\x81\x81", b"\x96\x81",
    # the space units
    b" ", b"\t", b"\n", b"\x0b", b"\x0c", b"\r", b"\xe2\x96\x81", b"\xe2\x96\x81\xe2\x96\x81x",
]
MAX_PIECE = max(map(len, PIECES))


def _filler(n, seed):
    """ASCII letters (some removed by the alphabet) and spaces."""
    rng = np.random.default_rng(seed)
    return bytes(rng.choice(np.frombuffer(b"abcdefghijkl   ", dtype=np.uint8), size=n))


def chunk_corpus():
    """Each piece at each of the 24 positions of a thread's register window: 4 bytes before its 16-byte chunk, the
    chunk, 4 bytes after (cells of 48 bytes, chunks at cell offsets 0, 16, 32)."""
    buf = bytearray(_filler(48 * 24 * len(PIECES), 1))
    cell = 0
    for p in PIECES:
        for k in range(24):
            at = 48 * cell + 12 + k
            buf[at:at + len(p)] = p
            cell += 1
    return bytes(buf)


def boundary_corpus(period, shifts=range(-7, 4)):
    """Each piece starting 7 bytes before to 3 bytes after a multiple of `period` (512: the bytes of one warp, 8192:
    of one block of char_hist_kernel), one placement per period."""
    n_pl = len(PIECES) * len(shifts)
    buf = bytearray(_filler(period * (n_pl + 1), 2))
    i = 0
    for p in PIECES:
        for d in shifts:
            i += 1
            at = period * i + d
            buf[at:at + len(p)] = p
    return bytes(buf)


def soup(n, seed=5):
    """Random bytes that lean toward 0x80..0xFF and the space units, mixed with the pieces and valid characters."""
    rng = np.random.default_rng(seed)
    high = [bytes([b]) for b in range(0x80, 0x100)]
    spaces = [b" ", b"\n", b"\t", b"\r", b"\x0b", b"\x0c", R.U2581]
    valid = [b"a", b"b", b"c", b"d", "é".encode(), "ж".encode(), "ߋ".encode(), "ࠀ".encode(), "語".encode(), "😀".encode()]
    groups = [(high, 0.45), (PIECES, 0.15), (spaces, 0.15), (valid, 0.25)]
    items = [x for g, _ in groups for x in g]
    w = np.concatenate([np.full(len(g), p / len(g)) for g, p in groups])
    idx = rng.choice(len(items), size=n // 2 + 16, p=w / w.sum())
    return b"".join(items[i] for i in idx)[:n]


def edge_corpora():
    """Each piece as the first and the last bytes of a corpus, and alone."""
    out = []
    for k, p in enumerate(PIECES):
        out += [p + _filler(40, 10 + k) + p, p]
    # byte-words that tokenise alike stay separate words; a word of removed characters only vanishes
    out.append(b"ab ab\xff a\x80b \xffab ab\xe2\x96 ab a\xc3 aaa jjj jj\xff j ab")
    return out


LENGTH_BASES = [b"".join(PIECES[::-1]), soup(80, seed=9)]


def length_corpora():
    return [base[:n] for base in LENGTH_BASES for n in range(71)]


# ---- the alphabet: code points removed on both sides of U+0800 --------------------------------------------------------
def alphabet(hist):
    """Keep a code point unless cp % 3 == 1 (this removes e.g. 'a', U+07FF and U+10000); ids from 5 on in code-point
    order, U+2581 = SPACE_ID."""
    kept = sorted(cp for cp in hist if cp % 3 != 1)
    cp2id = {cp: 5 + i for i, cp in enumerate(kept)}
    cp2id[R.SPACE_CP] = SPACE_ID
    return cp2id


@functools.lru_cache(maxsize=64)
def expected(text):
    _, hist = R.char_hist(text)
    cp2id = alphabet(hist)
    return R.expected_front(text, cp2id, SPACE_ID), cp2id


@contextlib.contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ---- the device side: the phase-by-phase ABI ------------------------------------------------------------------------
def _device_buffer(text, off, dev):
    """A buffer whose last byte is the corpus' last byte, the corpus at byte `off` of it: (pointer, keep-alive)."""
    if dev:
        import torch
        buf = torch.empty(len(text) + off, dtype=torch.uint8, device="cuda")
        if text:
            buf[off:] = torch.frombuffer(bytearray(text), dtype=torch.uint8).cuda()
        torch.cuda.synchronize()
        return buf.data_ptr() + off, buf
    raw = np.empty(len(text) + off, dtype=np.uint8)
    raw[off:] = np.frombuffer(text, dtype=np.uint8)
    return raw.ctypes.data + off, raw


def device_front(L, text, cp2id, off=None, dev=False, ctx=None):
    """load_corpus (host bytes, or device-resident at base offset `off`), char_hist, set_alphabet, build,
    export_words, dump_pairs -> the fields of _front_ref.expected_front.  ctx: run on this context (it stays open)
    instead of a new one."""
    own = ctx is None
    if own:
        ctx = C.c_void_p()
        assert L.yttm_ctx_create(0, C.byref(ctx)) == 0
    keep = None
    try:
        if off is None:
            assert L.yttm_train_load_corpus(ctx, C.cast(C.c_char_p(text), C.c_void_p), len(text), 0) == 0, L.yttm_last_error(ctx)
        else:
            ptr, keep = _device_buffer(text, off, dev)
            assert L.yttm_train_load_corpus(ctx, ptr, len(text), 1) == 0, L.yttm_last_error(ctx)
        dl, nd = C.c_uint64(0), C.c_uint64(0)
        assert L.yttm_train_char_hist(ctx, C.byref(dl), C.byref(nd)) == 0, L.yttm_last_error(ctx)
        cps = np.zeros(nd.value, dtype=np.uint32)
        cnt = np.zeros(nd.value, dtype=np.uint64)
        L.yttm_train_get_char_hist(ctx, cps.ctypes.data, cnt.ctypes.data)
        kc = np.array(list(cp2id), dtype=np.uint32)
        ki = np.array(list(cp2id.values()), dtype=np.uint32)
        assert L.yttm_train_set_alphabet(ctx, kc.ctypes.data, ki.ctypes.data, len(kc), SPACE_ID) == 0
        st = _lib.TrainStats()
        assert L.yttm_train_build(ctx, C.byref(st)) == 0, L.yttm_last_error(ctx)
        nw, nt = C.c_uint64(0), C.c_uint64(0)
        assert L.yttm_train_export_words(ctx, None, 0, None, None, 0, C.byref(nw), C.byref(nt)) == 0
        tok = np.zeros(nt.value + 1, dtype=np.uint32)
        offs = np.zeros(nw.value + 1, dtype=np.uint32)
        freq = np.zeros(nw.value + 1, dtype=np.uint64)
        assert L.yttm_train_export_words(ctx, tok.ctypes.data, len(tok), offs.ctypes.data, freq.ctypes.data, len(freq),
                                         C.byref(nw), C.byref(nt)) == 0, L.yttm_last_error(ctx)
        tl = tok.tolist()
        o = offs.tolist()
        words = sorted((tuple(tl[o[i]:o[i + 1]]), int(freq[i])) for i in range(nw.value))
        keys = np.zeros(st.n_pairs + 16, dtype=np.uint64)
        cts = np.zeros(st.n_pairs + 16, dtype=np.uint64)
        n = C.c_uint64(0)
        assert L.yttm_train_dump_pairs(ctx, keys.ctypes.data, cts.ctypes.data, len(keys), C.byref(n)) == 0
        pairs = dict(zip(keys[:n.value].tolist(), cts[:n.value].tolist()))
        return dict(data_len=dl.value, hist=dict(zip(cps.tolist(), cnt.tolist())), n_words=st.n_words,
                    n_unique=st.n_unique, n_tokens=st.n_tokens, words=words, pairs=pairs, n_pairs=st.n_pairs,
                    table_capacity=st.table_capacity)
    finally:
        if own:
            L.yttm_ctx_destroy(ctx)
        del keep


def _first_difference(a, b):
    if isinstance(a, dict):
        ks = sorted(set(a) | set(b))
        k = next(k for k in ks if a.get(k) != b.get(k))
        return "key %r: %r vs %r" % (k, a.get(k), b.get(k))
    k = next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
    return "%d vs %d entries, first difference at %d: %r vs %r" % (len(a), len(b), k, a[k:k + 1], b[k:k + 1])


FIELDS = ("data_len", "hist", "n_words", "n_unique", "n_tokens", "words", "pairs")


def assert_same(got, want, what=""):
    for f in FIELDS:
        if got[f] != want[f]:
            detail = _first_difference(got[f], want[f]) if f in ("hist", "words", "pairs") else "%r vs %r" % (got[f], want[f])
            raise AssertionError("%s: %s differs (device vs restatement): %s" % (what, f, detail))
    assert got["n_pairs"] == len(want["pairs"]), what


def check(L, text, what, off=None, dev=False):
    want, cp2id = expected(text)
    got = device_front(L, text, cp2id, off, dev)
    assert_same(got, want, "%s (%d bytes%s)" % (what, len(text), "" if off is None else ", base offset %d" % off))
    return got


# ---- bodies shared with the emulator test ------------------------------------------------------------------------------
def corpus(name, small=False):
    if name == "chunk":
        return chunk_corpus()
    if name == "warp":
        return boundary_corpus(512)
    if name == "block":
        return boundary_corpus(8192, shifts=(-3, -1) if small else range(-7, 4))
    if name == "soup":
        return soup(200_000 if small else 3_000_000)
    raise KeyError(name)


def check_pieces(L, name, small=False, dev=False):
    check(L, corpus(name, small), name, dev=dev)


def check_edges(L, dev=False):
    for k, text in enumerate(edge_corpora()):
        check(L, text, "edge corpus %d" % k, dev=dev)


def check_lengths(L, dev=False):
    for k, text in enumerate(length_corpora()):
        check(L, text, "length corpus %d" % k, dev=dev)


def check_misaligned(L, off, names, lengths=True, dev=False):
    for name in names:
        check(L, corpus(name, small=not dev), name, off=off, dev=dev)
    if lengths:
        for k, text in enumerate(length_corpora()):
            check(L, text, "length corpus %d" % k, off=off, dev=dev)


def check_pipelined(L, piece_kb, names, small=False, dev=False):
    """Pieces of piece_kb KB: the same results as the restatement and as the unpipelined run, field by field."""
    for name in names:
        text = corpus(name, small)
        with env(YTTM_TRAIN_PIPELINE=1, YTTM_TRAIN_PIPELINE_PIECE_KB=piece_kb):
            piped = check(L, text, "%s, pipelined in %s KB pieces" % (name, piece_kb), dev=dev)
        with env(YTTM_TRAIN_PIPELINE=0):
            plain = check(L, text, name, dev=dev)
        for f in FIELDS + ("n_pairs",):
            assert piped[f] == plain[f], (name, f)


def check_no_space(L, dev=False):
    """No ASCII space or newline anywhere (tabs and U+2581 only): one piece."""
    text = soup(150_000, seed=13).replace(b" ", b"\t").replace(b"\n", b"\xe2\x96\x81")
    assert b" " not in text and b"\n" not in text
    with env(YTTM_TRAIN_PIPELINE=1, YTTM_TRAIN_PIPELINE_PIECE_KB=1):
        check(L, text, "no space, pipelined", dev=dev)


def _word_hash(w):
    """The word table's hash of a byte-word (word_table_insert): FNV-1a, then mix64 of it xor (length << 1); the top
    24 bits are the slot's tag, the low bits its home slot."""
    m = (1 << 64) - 1
    h = 0xcbf29ce484222325
    for b in w:
        h = ((h ^ b) * 0x100000001b3) & m
    h ^= len(w) << 1
    h ^= h >> 33
    h = (h * 0xff51afd7ed558ccd) & m
    h ^= h >> 33
    h = (h * 0xc4ceb9fe1a85ec53) & m
    return h ^ (h >> 33)


def check_prefix_with_equal_tag(L, dev=False):
    """"we" and "wehvfqceze" have the same tag, and the home slot of the longer word is 4 slots after the shorter
    one's (65 536-slot table); ksmkp, kmzkm, nmxtu and kykot fill the 4 slots in between.  So when the longer word is
    in the table first, the shorter one's probe reaches it with an equal tag and equal first bytes: only the check that
    the stored word ends where the new one does keeps them apart."""
    short, long_, fill = b"we", b"wehvfqceze", [b"ksmkp", b"kmzkm", b"nmxtu", b"kykot"]
    hs, hl = _word_hash(short), _word_hash(long_)
    assert hs >> 40 == hl >> 40 and (hl - hs) & 0xffff == len(fill)
    assert sorted(_word_hash(f) & 0xffff for f in fill) == [(hs + k) & 0xffff for k in range(len(fill))]
    for text in (b" ".join([long_] * 3 + fill + [short, long_, short]), b" ".join(fill + [short, long_, short])):
        check(L, text, "prefix word with an equal tag", dev=dev)


def overflow_corpus():
    """About 40 000 distinct 4-letter words (plus repeats) in 220 KB: corpora up to 1 MB get a 65 536-slot word table
    that takes 32 768 unique words, so the first pass overflows and the build starts over with a larger table."""
    rng = np.random.default_rng(17)
    ids = rng.choice(26 ** 4, size=40_000, replace=False)
    ids = np.concatenate([ids, rng.choice(ids, size=4_000)])
    rng.shuffle(ids)
    letters = np.stack([(ids // 26 ** k) % 26 for k in range(4)], axis=1).astype(np.uint8) + ord("a")
    rows = np.concatenate([letters, np.full((len(ids), 1), ord(" "), dtype=np.uint8)], axis=1)
    text = rows.tobytes()
    assert len(text) < 1 << 20 and len(set(text.split())) > 32_768
    return text


def check_overflow(L, pipelined, dev=False):
    text = overflow_corpus()
    if pipelined:
        with env(YTTM_TRAIN_PIPELINE=1, YTTM_TRAIN_PIPELINE_PIECE_KB=64):
            check(L, text, "word table overflow, pipelined", dev=dev)
    else:
        with env(YTTM_TRAIN_PIPELINE=0):
            check(L, text, "word table overflow", dev=dev)


def check_pair_table(L, floor=None, dev=False):
    """The clean 100 KB Zipf text (valid UTF-8): also the histogram against Python's decoder; with a small
    YTTM_PAIR_CAP_FLOOR the build starts at that floor and grows the table until it is accepted."""
    text = _cases.zipf().text(100_000)
    want, _ = expected(text)
    s = text.decode()
    assert want["data_len"] == len(s)
    assert want["hist"] == dict(collections.Counter(ord(ch) for ch in s if ord(ch) not in R.SPACE_CPS))
    if floor is None:
        check(L, text, "zipf", dev=dev)
    else:
        with env(YTTM_PAIR_CAP_FLOOR=floor):
            got = check(L, text, "zipf, pair table floor %s" % floor, dev=dev)
        assert got["table_capacity"] > int(floor) and got["n_pairs"] > int(floor)


# ---- GPU tests ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["chunk", "warp", "block", "soup"])
def test_adversarial_pieces(product, name):
    check_pieces(product, name, dev=True)


def test_pieces_at_the_corpus_ends(product):
    check_edges(product, dev=True)


def test_corpus_lengths_0_to_70(product):
    check_lengths(product, dev=True)


def test_prefix_word_with_an_equal_tag(product):
    check_prefix_with_equal_tag(product, dev=True)


@pytest.mark.parametrize("off", range(1, 16))
def test_device_corpus_at_a_misaligned_base(product, off):
    check_misaligned(product, off, ["chunk", "warp", "soup"], dev=True)


@pytest.mark.parametrize("piece_kb", ["1", "3", "64"])
def test_pipelined_ingest(product, piece_kb):
    check_pipelined(product, piece_kb, ["chunk", "warp", "soup"], dev=True)


def test_pipelined_no_space(product):
    check_no_space(product, dev=True)


def test_pipelined_80mb_at_the_default_pieces(product):
    """About 80 MB of Zipf text at the default settings (pipelined, 32 MB pieces), adversarial bytes right before and
    right after each end the host chooses (the last ASCII space or newline of the piece's 32 MB)."""
    piece = 32 << 20
    text = bytearray(synth.FastZipf(n_words=50_000, seed=7).text(80 << 20))
    ends = _piece_ends(text, piece)
    assert len(ends) == 2
    before = [b"\xf0\x9f\x98", b"\xe2\x96", b"\xc3", b"\x80\xbf", b"\xe2\x96\x81", b"\xed\xa0\x80"]
    after = [b"\x80\x80\xbf", b"\x96\x81x", b"\xe2\x96\x81\t", b"\xf4\x90\x80\x80", b"\xbf\xe0\x9f\xbf", b"\xc0\xafz"]
    for k, e in enumerate(ends):
        a, b = before[k::2], after[k::2]
        pa, pb = b"".join(a), b"".join(b)
        text[e - 1 - len(pa):e - 1] = pa            # e - 1 is the space / newline the piece ends with
        text[e:e + len(pb)] = pb                    # no ' ' / '\n' in pb: the end stays where it is
    text = bytes(text)
    assert _piece_ends(text, piece) == ends
    assert len(text) >= 64 << 20                    # pipelined at the default threshold
    check(product, text, "80 MB, default pieces", dev=True)


def _piece_ends(text, piece):
    ends, lo, n = [], 0, len(text)
    while lo < n:
        hi = min(n, lo + piece)
        if hi < n:
            q = max(text.rfind(b" ", lo, hi), text.rfind(b"\n", lo, hi))
            hi = q + 1 if q >= 0 else n
            if hi < n:
                ends.append(hi)
        lo = hi
    return ends


@pytest.mark.parametrize("pipelined", [False, True])
def test_word_table_overflow(product, pipelined):
    check_overflow(product, pipelined, dev=True)


def test_initial_pair_table(product):
    check_pair_table(product, dev=True)


def test_pair_table_grown_from_a_small_floor(product):
    check_pair_table(product, "16", dev=True)


def test_zzz_sanitizer_memcheck_device_corpus(product):
    """compute-sanitizer memcheck over tools/sanitize_train_front.py (device-resident corpora at base offsets 1..15,
    each at the end of its own cudaMalloc): no report; skips where the tool refuses the device."""
    import shutil
    import subprocess
    import sys
    from _bind import ROOT
    exe = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(exe):
        pytest.skip("compute-sanitizer is not installed")
    env = {k: v for k, v in os.environ.items() if not k.startswith(("YTTM_", "YT_EMU_"))}
    env["PYTORCH_NO_CUDA_MEMORY_CACHING"] = "1"
    r = subprocess.run([exe, "--tool", "memcheck", sys.executable, os.path.join(ROOT, "tools", "sanitize_train_front.py")],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    text = r.stdout.decode(errors="replace")
    if "Error: Device not supported" in text:
        pytest.skip("compute-sanitizer does not support this device here")
    assert "checks identical to the restatement" in text, text[-1500:]
    assert "ERROR SUMMARY: 0 errors" in text, text[-1500:]

"""Training on a FED corpus on the GPU: the text goes through the byte passes in pieces (yttm_train_feed_begin / feed /
feed_end), its unique words gather in one device table whose bytes live in a word arena, and the corpus itself never
sits on the device.  train_bpe / learn_bpe_from_string feed above a size threshold (YTTM_TRAIN_FEED_ABOVE forces it
here) in pieces of YTTM_TRAIN_FEED_PIECE_KB.

  1. parity: the golden corpora fed in many pieces give the reference's model, byte for byte the in-memory model, and
     the same report sizes;
  2. edges against the oracle: long words, tab / vertical-tab / form-feed / CRLF separators, multi-byte sequences and
     invalid UTF-8 around the cuts, empty and blank files, a rare character in one piece, all-new and all-repeated
     pieces (insert and lookup paths, arena and table growth);
  3. inputs: a FIFO, yttm_api_train_memory, and the C ABI fed in blocks of 1, 7 and random sizes from one reused
     buffer (same histogram, words and pairs as load_corpus + build); misuse fails with a message;
  4. the memory bound: the device peak of a fed corpus does not grow with the corpus;
  5. a forced STREAMING merge loop after a feed.

The bodies take the library: tests/test_train_feed_emul_cpu.py runs 1 - 3 on the SIMT emulator at small sizes."""
import base64
import ctypes as C
import glob
import json
import os
import tempfile
import threading

import numpy as np
import pytest

import test_train_front_gpu as FG
from _bind import read_model, tmp_model_path
from youtokentome_b200 import _lib, synth

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "*.json")))
REPORT = ["n_bytes", "data_len", "n_words", "n_unique", "n_tokens", "n_pairs", "n_merges", "read_s", "h2d_ms",
          "char_hist_ms", "word_count_ms", "tokenise_ms", "pair_hist_ms", "merge_loop_ms", "total_s", "launches",
          "loop_launches", "feed_pieces", "device_peak_bytes"]
SIZES = ("n_words", "n_unique", "data_len", "n_tokens", "n_pairs")
_tmp = tempfile.mkdtemp(prefix="yttm_feed_")


def report(L):
    out = (C.c_double * len(REPORT))()
    n = L.yttm_api_train_report(out, len(REPORT))
    return dict(zip(REPORT[:n], list(out)[:n]))


def corpus_file(text):
    fd, path = tempfile.mkstemp(dir=_tmp, suffix=".txt")
    with os.fdopen(fd, "wb") as f:
        f.write(text)
    return path


def train_file(L, path, vocab, cov=1.0, pad=0, unk=1, bos=2, eos=3, piece_kb=None):
    """train_bpe on a file (fed when piece_kb is given) -> (model path, report); ValueError(message) on failure."""
    model = tmp_model_path("feed")
    knobs = dict(YTTM_TRAIN_FEED_ABOVE=0, YTTM_TRAIN_FEED_PIECE_KB=piece_kb) if piece_kb else {}
    with FG.env(**knobs):
        if L.yttm_api_train(path.encode(), model.encode(), vocab, cov, 1, pad, unk, bos, eos) != 0:
            raise ValueError(L.yttm_api_last_error(None).decode())
    return model, report(L)


def same_file(a, b):
    with open(a, "rb") as f, open(b, "rb") as g:
        return f.read() == g.read()


def golden(path):
    with open(path) as f:
        g = json.load(f)
    want = ({int(k): int(v) for k, v in g["model"]["char2id"]}, [tuple(r) for r in g["model"]["rules"]],
            tuple(g["model"]["special_line"]))
    return base64.b64decode(g["train_b64"]), g["vocab_size"], g["coverage"], g["special"], want


# ---- 1. parity with the reference ------------------------------------------------------------------------------------
def parity(L, path, pieces_kb):
    text, vocab, cov, special, want = golden(path)
    f = corpus_file(text)
    m_mem, r_mem = train_file(L, f, vocab, cov, **special)
    assert read_model(m_mem) == want
    assert r_mem["feed_pieces"] == 0
    for kb in pieces_kb:
        m, r = train_file(L, f, vocab, cov, piece_kb=kb, **special)
        assert same_file(m, m_mem), "%s in %d KB pieces: the model differs from the in-memory one" % (path, kb)
        assert {k: r[k] for k in SIZES} == {k: r_mem[k] for k in SIZES}, (kb, r, r_mem)
        assert r["n_bytes"] == len(text)
        assert r["feed_pieces"] >= (2 if len(text) > 2 * kb * 1024 else 1), (kb, len(text), r["feed_pieces"])


# ---- 2. edges against the oracle --------------------------------------------------------------------------------------
def check_oracle(L, oracle, text, vocab, cov=1.0, piece_kb=1, min_pieces=1):
    """A fed training of `text` equals the oracle's (or fails with the same message) -> the report."""
    m_o = tmp_model_path("orc")
    f = corpus_file(text)
    try:
        oracle.train(text, m_o, vocab, cov)
    except ValueError as e:
        with pytest.raises(ValueError) as ei:
            train_file(L, f, vocab, cov, piece_kb=piece_kb)
        assert str(ei.value) == str(e)
        return None
    m, r = train_file(L, f, vocab, cov, piece_kb=piece_kb)
    a, b = read_model(m_o), read_model(m)
    assert a == b, "fed model differs from the oracle (%d bytes, %d KB pieces)" % (len(text), piece_kb)
    assert r["feed_pieces"] >= min_pieces, r
    return r


def _words(rng, n, lo=2, hi=9, letters=b"abcdefghijklmnop"):
    lens = rng.integers(lo, hi, n)
    al = np.frombuffer(letters, dtype=np.uint8)
    return [al[rng.integers(0, len(al), k)].tobytes() for k in lens]


def edge_corpora(small=False):
    """(name, text, vocab, coverage, least number of pieces at 1 KB)"""
    rng = np.random.default_rng(17)
    base = b" ".join(_words(rng, 1500 if small else 6000)) + b"\n"
    out = [("long word", b"ab cd " + b"xy" * 1800 + b" ab ef\n" + base[:3000], 120, 1.0, 3)]
    for name, sep in (("tabs", b"\t"), ("vertical tabs", b"\x0b"), ("form feeds", b"\x0c"), ("crlf", b"\r\n")):
        out.append((name, sep.join(_words(rng, 1200 if small else 3000)), 150, 1.0, 2))
    cjk = "日本▁語 テキスト▁a ▁▁ 𝄞x ".encode()
    out.append(("multi-byte at the cuts", b"".join(cjk[:k] + b" " + base[k * 7:k * 7 + 97] for k in range(len(cjk))) * 4,
                200, 1.0, 2))
    bad = b"\x80\xbfab \xff\xfeab\xe2\x96 \xc0\xaf \xed\xa0\x80 \xf0\x9f\x98 \x80\x80 "
    out.append(("invalid UTF-8 after the cuts", b"".join(bad[k:] + base[k * 11:k * 11 + 211] for k in range(len(bad))) * 3,
                150, 1.0, 2))
    out.append(("empty", b"", 10, 1.0, 0))
    out.append(("only spaces", b" " * 5000, 10, 1.0, 0))
    out.append(("no trailing newline", base[:4000].rstrip() + b" lastword", 150, 1.0, 3))
    rare = base[:2500] + " ζζζζ ".encode() + base[2500:6000]
    out.append(("rare character in one piece", rare, 150, 0.9995, 3))
    out.append(("words only in the first piece", b"QQQ RRR QQQRRR " * 60 + base[:5000], 150, 1.0, 3))
    out.append(("words only in the last piece", base[:5000] + b" QQQ RRR QQQRRR" * 60, 150, 1.0, 3))
    new = b" ".join(_words(rng, 4000 if small else 20000, 5, 9, b"abcdefghijklmnopqrstuvwxyz")) + b"\n"
    out.append(("every piece all-new words", new, 300, 1.0, 10))
    out.append(("every piece the same words", b"the cat sat on a mat and ran off\n" * (200 if small else 800), 100,
                1.0, 5))
    return out


# ---- 3. inputs -------------------------------------------------------------------------------------------------------
def fifo(L, text, vocab):
    """A corpus written into a FIFO by a thread: no size, so it is fed without any knob; equals the in-memory model."""
    path = os.path.join(tempfile.mkdtemp(dir=_tmp), "fifo")
    os.mkfifo(path)

    def writer():
        with open(path, "wb") as f:
            f.write(text)
    t = threading.Thread(target=writer)
    t.start()
    try:
        with FG.env(YTTM_TRAIN_FEED_PIECE_KB=4):
            m, r = train_file(L, path, vocab)
    finally:
        t.join()
    m_mem, r_mem = train_file(L, corpus_file(text), vocab)
    assert same_file(m, m_mem)
    assert r["feed_pieces"] > 1 and r_mem["feed_pieces"] == 0
    assert {k: r[k] for k in SIZES} == {k: r_mem[k] for k in SIZES}


def memory_api(L, text, merges):
    """yttm_api_train_memory above the threshold: fed, and the model of the in-memory path."""
    vocab = len(set(text.decode("utf-8", "ignore"))) + 5 + merges
    m_mem, m = tmp_model_path("mem"), tmp_model_path("fed")
    assert L.yttm_api_train_memory(text, len(text), m_mem.encode(), vocab, 1.0, 0, 1, 2, 3) == 0
    r_mem = report(L)
    with FG.env(YTTM_TRAIN_FEED_ABOVE=len(text) - 1, YTTM_TRAIN_FEED_PIECE_KB=2):
        assert L.yttm_api_train_memory(text, len(text), m.encode(), vocab, 1.0, 0, 1, 2, 3) == 0
    r = report(L)
    assert same_file(m, m_mem)
    assert r["feed_pieces"] > 1 and r_mem["feed_pieces"] == 0
    assert {k: r[k] for k in SIZES} == {k: r_mem[k] for k in SIZES}


def feed_blocks(L, ctx, text, blocks):
    """feed_begin, then `text` in blocks of the sizes `blocks` yields, each copied into ONE reused caller buffer."""
    assert L.yttm_train_feed_begin(ctx) == 0, L.yttm_last_error(ctx)
    buf = C.create_string_buffer(max(len(text), 1))
    at = 0
    while at < len(text):
        k = min(next(blocks), len(text) - at)
        C.memmove(buf, text[at:at + k], k)
        assert L.yttm_train_feed(ctx, buf, k) == 0, L.yttm_last_error(ctx)
        C.memset(buf, 0x41, k)   # the library copied the block: overwriting it changes nothing
        at += k
    dl, nd = C.c_uint64(0), C.c_uint64(0)
    assert L.yttm_train_feed_end(ctx, C.byref(dl), C.byref(nd)) == 0, L.yttm_last_error(ctx)


def fed_front(L, text, cp2id, blocks, piece_kb):
    """The fields of _front_ref.expected_front from a fed context (as FG.device_front from a loaded one)."""
    ctx = C.c_void_p()
    assert L.yttm_ctx_create(0, C.byref(ctx)) == 0
    try:
        with FG.env(YTTM_TRAIN_FEED_PIECE_KB=piece_kb):
            feed_blocks(L, ctx, text, blocks)
        pieces = L.yttm_stage_ms(ctx, b"feed_pieces")
        got = _front_after_load(L, ctx, cp2id)
        got["feed_pieces"] = pieces
        assert got["n_bytes"] == len(text)
        return got
    finally:
        L.yttm_ctx_destroy(ctx)


def _front_after_load(L, ctx, cp2id):
    """FG.device_front's steps after the load (char_hist .. dump_pairs), on a context whose corpus is in place."""
    dl, nd = C.c_uint64(0), C.c_uint64(0)
    assert L.yttm_train_char_hist(ctx, C.byref(dl), C.byref(nd)) == 0, L.yttm_last_error(ctx)
    cps = np.zeros(nd.value, dtype=np.uint32)
    cnt = np.zeros(nd.value, dtype=np.uint64)
    L.yttm_train_get_char_hist(ctx, cps.ctypes.data, cnt.ctypes.data)
    kc = np.array(list(cp2id), dtype=np.uint32)
    ki = np.array(list(cp2id.values()), dtype=np.uint32)
    assert L.yttm_train_set_alphabet(ctx, kc.ctypes.data, ki.ctypes.data, len(kc), FG.SPACE_ID) == 0
    st = _lib.TrainStats()
    assert L.yttm_train_build(ctx, C.byref(st)) == 0, L.yttm_last_error(ctx)
    return dict(words_and_pairs(L, ctx, st), data_len=dl.value, hist=dict(zip(cps.tolist(), cnt.tolist())))


def words_and_pairs(L, ctx, st):
    """The word and pair fields of _front_ref.expected_front from a context that has built its words (st: the
    statistics the build returned)."""
    nw, nt = C.c_uint64(0), C.c_uint64(0)
    assert L.yttm_train_export_words(ctx, None, 0, None, None, 0, C.byref(nw), C.byref(nt)) == 0
    tok = np.zeros(nt.value + 1, dtype=np.uint32)
    offs = np.zeros(nw.value + 1, dtype=np.uint32)
    freq = np.zeros(nw.value + 1, dtype=np.uint64)
    assert L.yttm_train_export_words(ctx, tok.ctypes.data, len(tok), offs.ctypes.data, freq.ctypes.data, len(freq),
                                     C.byref(nw), C.byref(nt)) == 0, L.yttm_last_error(ctx)
    tl, o = tok.tolist(), offs.tolist()
    words = sorted((tuple(tl[o[i]:o[i + 1]]), int(freq[i])) for i in range(nw.value))
    n = C.c_uint64(0)
    keys = np.zeros(st.n_pairs + 16, dtype=np.uint64)
    cts = np.zeros(st.n_pairs + 16, dtype=np.uint64)
    assert L.yttm_train_dump_pairs(ctx, keys.ctypes.data, cts.ctypes.data, len(keys), C.byref(n)) == 0
    return dict(n_words=st.n_words, n_unique=st.n_unique, n_tokens=st.n_tokens, words=words,
                pairs=dict(zip(keys[:n.value].tolist(), cts[:n.value].tolist())), n_pairs=st.n_pairs,
                n_bytes=st.n_bytes)


def _sizes(kind, seed=5):
    rng = np.random.default_rng(seed)
    while True:
        yield kind if isinstance(kind, int) else int(rng.integers(1, 5000))


def abi_blocks(L, text, piece_kb=1):
    want, cp2id = FG.expected(text)
    loaded = FG.device_front(L, text, cp2id)
    FG.assert_same(loaded, want, "loaded")
    for kind in (1, 7, "random"):
        got = fed_front(L, text, cp2id, _sizes(kind), piece_kb)
        FG.assert_same(got, want, "fed in blocks of %s bytes" % kind)
        assert got["feed_pieces"] > 1


def abi_misuse(L):
    """feed / feed_end before feed_begin, char_hist and build between begin and end fail and say why; a load_corpus
    after an abandoned feed trains its own corpus."""
    a = FG.soup(30_000, seed=3)
    b = FG.corpus("chunk")
    want, cp2id = FG.expected(b)
    ctx = C.c_void_p()
    assert L.yttm_ctx_create(0, C.byref(ctx)) == 0
    err = lambda: L.yttm_last_error(ctx).decode()   # noqa: E731
    try:
        assert L.yttm_train_feed(ctx, a, 10) != 0 and "feed_begin" in err()
        dl, nd = C.c_uint64(0), C.c_uint64(0)
        assert L.yttm_train_feed_end(ctx, C.byref(dl), C.byref(nd)) != 0 and "feed_begin" in err()
        with FG.env(YTTM_TRAIN_FEED_PIECE_KB=1):
            assert L.yttm_train_feed_begin(ctx) == 0
            assert L.yttm_train_feed(ctx, a, len(a)) == 0, err()
        assert L.yttm_train_char_hist(ctx, C.byref(dl), C.byref(nd)) != 0 and "feed_end" in err()
        assert L.yttm_train_build(ctx, None) != 0 and "feed_end" in err()
        got = FG.device_front(L, b, cp2id, ctx=ctx)   # load_corpus after the abandoned feed
        FG.assert_same(got, want, "loaded corpus after an abandoned feed")
        assert L.yttm_stage_ms(ctx, b"feed_pieces") == 0
        assert L.yttm_train_feed(ctx, a, 10) != 0 and "feed_begin" in err()
    finally:
        L.yttm_ctx_destroy(ctx)


def abi_text(small=False):
    return FG.soup(20_000 if small else 200_000, seed=9) + b"\t" + FG.chunk_corpus()[:30_000]


# ---- GPU tests -------------------------------------------------------------------------------------------------------
@pytest.fixture
def lib(product):
    return product


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-5] for p in GOLDEN])
def test_golden_corpora_fed(lib, path):
    parity(lib, path, (1, 4, 13, 1 << 16))


@pytest.mark.parametrize("case", range(len(edge_corpora())), ids=[c[0] for c in edge_corpora()])
def test_edges_against_the_oracle(lib, oracle, case):
    _, text, vocab, cov, pieces = edge_corpora()[case]
    check_oracle(lib, oracle, text, vocab, cov, 1, pieces)


def test_fifo(lib):
    fifo(lib, synth.readme_corpus(n_lines=600), 400)


def test_memory_api_above_the_threshold(lib):
    memory_api(lib, FG.soup(100_000, seed=4), 500)


def test_abi_blocks(lib):
    abi_text_ = abi_text()
    abi_blocks(lib, abi_text_[:60_000], 1)
    abi_blocks(lib, abi_text_, 13)


def test_abi_misuse(lib):
    abi_misuse(lib)


def test_streaming_merge_loop_after_a_feed(lib, oracle):
    text = synth.readme_corpus(n_lines=800)
    with FG.env(YTTM_FORCE_STREAM=1, YTTM_STREAM_Q=64):
        check_oracle(lib, oracle, text, 600, 1.0, 4, 2)


def test_device_memory_does_not_grow_with_the_corpus(lib):
    """Zipf corpora of 256 MB and 1 GB (one lexicon) fed in 16 MB pieces: their device peaks differ by less than 10 %
    and stay below half of the smaller corpus, while the in-memory path on 256 MB reports more than the corpus; the
    models are equal.  The fed peak is mostly fixed costs that no corpus size changes: the merge loop's exchange buffer
    (about 36 MB on one GPU), the dense code-point histogram and id table (13 MB) and two piece buffers (measured on an
    H100 80GB HBM3, 700 W: 77.0 MB for both corpora, against 651 MB and 2379 MB in memory)."""
    z = synth.FastZipf(n_words=100_000, seed=11)
    small, big = z.text(256 << 20), z.text(1 << 30)
    peaks = []
    for text in (small, big):
        f = corpus_file(text)
        m, r = train_file(lib, f, 5000, piece_kb=16 << 10)
        m_mem, r_mem = train_file(lib, f, 5000)
        assert same_file(m, m_mem)
        assert {k: r[k] for k in SIZES} == {k: r_mem[k] for k in SIZES}
        peaks.append(r["device_peak_bytes"])
        if text is small:
            assert r_mem["device_peak_bytes"] > len(text), r_mem
        os.remove(f)
        print("%d MB: fed peak %.1f MB in %d pieces, in-memory peak %.1f MB" %
              (len(text) >> 20, r["device_peak_bytes"] / 2 ** 20, r["feed_pieces"], r_mem["device_peak_bytes"] / 2 ** 20))
    assert abs(peaks[1] - peaks[0]) < 0.1 * peaks[0], peaks
    assert max(peaks) < (256 << 20) / 2, peaks

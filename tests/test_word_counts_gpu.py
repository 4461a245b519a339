"""Word-count tables on the GPU: BPE.count_words counts a corpus's words once, and BPE.train_from_counts trains from
such a table (yttm_train_feed_words / yttm_train_fed_words of include/yttm_b200.h).  A model depends on the text only
through its words with their counts, its code points and data_len, so a table must train to the model file of the
text, byte for byte, and fail with its errors.

  1. round trip: every golden corpus and every feed edge corpus -> count_words -> train_from_counts (as a WordCounts
     and through the TSV, at the default pieces and at 1 KB pieces) writes BPE.train's model file or fails alike;
  2. counting against a restatement on tests/_front_ref.py: words, counts, data_len and separators; the TSV is
     byte-identical across piece sizes and sorted by count descending, then bytes ascending;
  3. tables that no text wrote: duplicates, zero counts, multi-byte and invalid UTF-8, words above a tile, with and
     without separators, characters removed by coverage -> the model of the expanded text and of the oracle;
  4. counts beyond any text: all counts x 2^20, the 2^43 freq x tokens limit, data_len past 2^64;
  5. the C ABI: text blocks and word lists interleaved in one feed, host and device lists, misuse;
  6. inputs: every form of `counts`, rejected words, TSV errors with their line, type errors;
  7. scale: a 256 MB corpus at vocab 32k, and the device peak of the table training below the text training's;
  8. the CLI: `yttm count_words` (stdin) then `yttm bpe_counts` write `yttm bpe`'s model.

The bodies take the library (and a function that puts a numpy array where the library reads device lists), so
tests/test_word_counts_emul_cpu.py runs 1 - 3 and 5 on the SIMT emulator."""
import collections
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import _front_ref as R
import test_train_feed_gpu as F
import test_train_front_gpu as FG
from _bind import ROOT, read_model, tmp_model_path
from youtokentome_b200 import synth
from youtokentome_b200.youtokentome import BPE, WordCounts

pytestmark = pytest.mark.gpu
_tmp = tempfile.mkdtemp(prefix="yttm_counts_")
LIMIT_ERROR = "fed corpus: a word's frequency x tokens must stay below 2^43"


def read(path):
    with open(path, "rb") as f:
        return f.read()


def special_ids(special):
    return dict(pad_id=special["pad"], unk_id=special["unk"], bos_id=special["bos"], eos_id=special["eos"])


def train_text(text, vocab, cov=1.0, **ids):
    """BPE.train on `text` written to a file -> (model file bytes, None) or (None, error message)."""
    model = tmp_model_path("txt")
    try:
        BPE.train(F.corpus_file(text), model, vocab, cov, **ids)
    except ValueError as e:
        return None, str(e)
    return read(model), None


def train_table(counts, vocab, cov=1.0, **ids):
    model = tmp_model_path("tab")
    try:
        BPE.train_from_counts(counts, model, vocab, cov, **ids)
    except ValueError as e:
        return None, str(e)
    return read(model), None


def write_tsv(table):
    """A WordCounts as the TSV count_words writes."""
    fd, path = tempfile.mkstemp(dir=_tmp, suffix=".tsv")
    b = table.word_bytes.tobytes()
    o = table.word_offsets.tolist()
    with os.fdopen(fd, "wb") as f:
        f.write(b"\t%d\n" % table.separators)
        for i, c in enumerate(table.counts.tolist()):
            f.write(b[o[i]:o[i + 1]] + b"\t%d\n" % c)
    return path


def entries(table):
    b, o = table.word_bytes.tobytes(), table.word_offsets.tolist()
    return [(b[o[i]:o[i + 1]], c) for i, c in enumerate(table.counts.tolist())]


def expand(words, counts, separators=None):
    """The text a table stands for: every occurrence joined by one space, then the separators left over."""
    occ = [w for w, c in zip(words, counts) for _ in range(int(c))]
    seps = len(occ) if separators is None else separators
    assert seps >= len(occ) - 1
    return b" ".join(occ) + b" " * (seps - max(len(occ) - 1, 0))


# ---- 1. round trip ---------------------------------------------------------------------------------------------------
def round_trip(text, vocab, cov=1.0, piece_kbs=(None, 1), **ids):
    want, err = train_text(text, vocab, cov, **ids)
    tsvs = []
    for kb in piece_kbs:
        with FG.env(**({"YTTM_TRAIN_FEED_PIECE_KB": kb} if kb else {})):
            table = BPE.count_words(text)
            path = os.path.join(_tmp, "t%d.tsv" % len(tsvs))
            BPE.count_words(F.corpus_file(text), output=path)
            tsvs.append(read(path))
            for form in (table, path):
                got, got_err = train_table(form, vocab, cov, **ids)
                assert got_err == err, (kb, got_err, err)
                assert got == want, "%d bytes, %s KB pieces, %s: the model differs from BPE.train's" % (
                    len(text), kb, type(form).__name__)
    assert len(set(tsvs)) == 1, "the TSV depends on the piece size"
    return table


# ---- 2. counting against a restatement ------------------------------------------------------------------------------
def restated(text):
    units = R.decode_units(text)
    seps = sum(1 for _, _, cp in units if cp is not None and cp in R.SPACE_CPS)
    words = collections.Counter(R.byte_words(text))
    return sorted(words.items(), key=lambda kv: (-kv[1], kv[0])), seps, len(units)


def check_counting(text, piece_kbs=(None, 1, 3)):
    want, seps, data_len = restated(text)
    tsvs = set()
    for kb in piece_kbs:
        with FG.env(**({"YTTM_TRAIN_FEED_PIECE_KB": kb} if kb else {})):
            for run in range(2):
                path = os.path.join(_tmp, "c.tsv")
                t = BPE.count_words(text, output=path)
                assert entries(t) == want
                assert (t.separators, t.data_len) == (seps, data_len)
                assert t.word_bytes.dtype == np.uint8 and t.word_offsets.dtype == np.uint64 and t.counts.dtype == np.uint64
                tsv = read(path)
                assert tsv == b"\t%d\n" % seps + b"".join(w + b"\t%d\n" % c for w, c in want)
                tsvs.add(tsv)
    assert len(tsvs) == 1


def counting_corpora(small=False):
    bad = b"\x80\xbfab \xff\xfeab\xe2\x96 \xc0\xaf \xed\xa0\x80 \xf0\x9f\x98 \x80\x80 x\xe2\x96\x81y\r\n\x0b\x0c"
    return [synth.readme_corpus(n_lines=60 if small else 300), bad * 20, b"", b"   ", b"single",
            "日本▁語 テキスト▁a ▁▁ 𝄞x ".encode() * 30]


# ---- 3. tables that no text wrote -----------------------------------------------------------------------------------
def random_table(seed, n=300, long_word=False):
    rng = np.random.default_rng(seed)
    alpha = [b"a", b"b", b"c", b"d", "é".encode(), "ж".encode(), "日".encode(), "𝄞".encode(), b"\xff", b"\x80",
             b"\xe2\x96", b"\xc0\xaf", "ζ".encode()]
    p = np.array([20, 15, 12, 10, 6, 6, 4, 2, 1, 1, 1, 1, 0.3])
    p /= p.sum()
    words = []
    for _ in range(n):
        k = int(rng.integers(1, 8))
        words.append(b"".join(alpha[i] for i in rng.choice(len(alpha), k, p=p)))
    words += words[:40]                        # duplicates add up
    if long_word:
        words.append(b"ab" * 10_000)             # 20 000 tokens: above a tile of the merge loop
    counts = rng.integers(0, 50, len(words)).astype(np.uint64)
    counts[::17] = 0                           # count 0 contributes nothing
    return words, counts


def check_table(oracle, words, counts, vocab, cov, separators=None):
    text = expand(words, counts.tolist(), separators)
    want, err = train_text(text, vocab, cov)
    table = (words, counts) if separators is None else WordCounts(*_packed(words), counts, separators, None)
    got, got_err = train_table(table, vocab, cov)
    assert (got, got_err) == (want, err)
    if oracle is not None and want is not None:
        m_o = tmp_model_path("orc")
        oracle.train(text, m_o, vocab, cov)
        assert read_model(m_o) == read_model(_written(got))


def _packed(words):
    offs = np.zeros(len(words) + 1, dtype=np.uint64)
    np.cumsum([len(w) for w in words], out=offs[1:])
    return np.frombuffer(b"".join(words), dtype=np.uint8), offs


def _written(model_bytes):
    path = tmp_model_path("cmp")
    with open(path, "wb") as f:
        f.write(model_bytes)
    return path


def tables_not_from_text(oracle, small=False):
    for seed, long_word, cov, seps in ((1, False, 1.0, None), (2, True, 1.0, 5000), (3, False, 0.999, None),
                                       (4, False, 0.97, 9000)):
        words, counts = random_table(seed, 120 if small else 300, long_word and not small)
        total = int(counts.sum())
        check_table(oracle, words, counts, 200, cov, None if seps is None else max(seps, total - 1))
    # every character of some words removed by coverage: they vanish or become equal
    words = [b"ab", b"a\xc2\xbfb", "aζb".encode(), "ζ".encode(), "ζζ".encode(), b"cd"]
    check_table(oracle, words, np.array([50, 1, 1, 1, 1, 40], dtype=np.uint64), 30, 0.98)


# ---- 5. the C ABI ----------------------------------------------------------------------------------------------------
def feed_mixed(L, blocks, to_device):
    """feed_begin, then text blocks (bytes) and word lists ((words, counts, separators)) in order, feed_end, and the
    front fields of the context."""
    text_all = b"".join(b if isinstance(b, bytes) else expand(*b) for b in blocks)
    want, cp2id = FG.expected(text_all)
    ctx = C.c_void_p()
    assert L.yttm_ctx_create(0, C.byref(ctx)) == 0
    keep = []
    try:
        with FG.env(YTTM_TRAIN_FEED_PIECE_KB=1):
            assert L.yttm_train_feed_begin(ctx) == 0
            for b in blocks:
                if isinstance(b, bytes):
                    assert L.yttm_train_feed(ctx, b, len(b)) == 0, L.yttm_last_error(ctx)
                    continue
                words, counts, seps = b
                wb, wo = _packed(words)
                arrs = [to_device(wb), to_device(wo), to_device(np.asarray(counts, dtype=np.uint64))]
                keep.append(arrs)
                ptrs = [a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data for a in arrs]
                assert L.yttm_train_feed_words(ctx, *ptrs, len(words), 2 ** 64 - 1 if seps is None else seps,
                                               int(to_device is not np.asarray)) == 0, L.yttm_last_error(ctx)
            dl, nd = C.c_uint64(0), C.c_uint64(0)
            assert L.yttm_train_feed_end(ctx, C.byref(dl), C.byref(nd)) == 0, L.yttm_last_error(ctx)
        got = F._front_after_load(L, ctx, cp2id)
        FG.assert_same(got, want, "mixed feed")
    finally:
        L.yttm_ctx_destroy(ctx)
    return got


def abi_mixed(L, to_device, small=False):
    rng = np.random.default_rng(7)
    base = b" ".join(F._words(rng, 800 if small else 3000)) + b"\n"
    words, counts = random_table(11, 150 if small else 600)
    lst = (words, counts.tolist(), None)
    blocks = [base[:1500] + b"\n", lst, base[1500:] + b"\n", (words[:30], [3] * 30, 100), b"tail words\n"]
    host = feed_mixed(L, blocks, np.asarray)
    dev = feed_mixed(L, blocks, to_device)
    assert host == dev


def abi_misuse(L):
    ctx = C.c_void_p()
    assert L.yttm_ctx_create(0, C.byref(ctx)) == 0
    err = lambda: L.yttm_last_error(ctx).decode()   # noqa: E731
    try:
        wb, wo = _packed([b"ab"])
        cnt = np.array([1], dtype=np.uint64)
        assert L.yttm_train_feed_words(ctx, wb.ctypes.data, wo.ctypes.data, cnt.ctypes.data, 1, 1, 0) != 0
        assert "feed_begin" in err()
        u = C.c_uint64(0)
        assert L.yttm_train_fed_words(ctx, None, 0, None, None, 0, C.byref(u), C.byref(u), None) == 1
        assert "feed_end" in err()
        assert L.yttm_train_feed_begin(ctx) == 0
        wb, wo = _packed([b"ab", b"c d"])
        cnt = np.array([1, 2], dtype=np.uint64)
        assert L.yttm_train_feed_words(ctx, wb.ctypes.data, wo.ctypes.data, cnt.ctypes.data, 2, 2 ** 64 - 1, 0) != 0
        assert "entry 1" in err() and "separator" in err()
        assert L.yttm_train_feed(ctx, b"x", 1) != 0 and "feed_begin" in err()   # a failed list ended the feed
    finally:
        L.yttm_ctx_destroy(ctx)


# ---- GPU tests -------------------------------------------------------------------------------------------------------
def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64 if a.dtype == np.uint64 else a.dtype)).cuda()


@pytest.fixture
def lib(product):
    return product


@pytest.mark.parametrize("path", F.GOLDEN, ids=[os.path.basename(p)[:-5] for p in F.GOLDEN])
def test_round_trip_golden(lib, path):
    text, vocab, cov, special, _ = F.golden(path)
    round_trip(text, vocab, cov, **special_ids(special))


@pytest.mark.parametrize("case", range(len(F.edge_corpora())), ids=[c[0] for c in F.edge_corpora()])
def test_round_trip_edges(lib, case):
    _, text, vocab, cov, _ = F.edge_corpora()[case]
    round_trip(text, vocab, cov)


def test_round_trip_vocab_too_small(lib):
    round_trip(synth.readme_corpus(n_lines=100), 20)


def test_counting_against_the_restatement(lib):
    for text in counting_corpora():
        check_counting(text)


def test_tables_not_from_a_text(lib, oracle):
    tables_not_from_text(oracle)


def test_counts_times_2_20(lib):
    """Every count and the separators x 2^20 change no order and no coverage ratio, so the model is the same.  data_len
    stays below 2^53, where the coverage test's doubles hold every value exactly."""
    text = synth.readme_corpus(n_lines=400) + " ζζ ζ ξ ".encode()
    t = BPE.count_words(text)
    assert t.data_len << 20 < 2 ** 53
    big = WordCounts(t.word_bytes, t.word_offsets, t.counts << np.uint64(20), t.separators << 20, None)
    for cov in (1.0, 0.9999):
        assert train_table(big, 500, cov) == train_table(t, 500, cov) == train_text(text, 500, cov)


def test_freq_x_tokens_limit(lib):
    ok = 2 ** 43 // 3 - 1                       # "ab": [space, a, b], 3 tokens
    got, err = train_table(([b"ab", b"cd"], np.array([ok, 5], dtype=np.uint64)), 20)
    assert err is None
    got, err = train_table(([b"ab", b"cd"], np.array([ok + 1, 5], dtype=np.uint64)), 20)
    assert err == LIMIT_ERROR


def test_data_len_past_2_64(lib):
    _, err = train_table(([b"a", b"b"], np.array([2 ** 63, 2 ** 63], dtype=np.uint64)), 20)
    assert "2^64" in err
    _, err = train_table(WordCounts(*_packed([b"a"]), np.array([5], dtype=np.uint64), 2 ** 64 - 2, None), 20)
    assert "2^64" in err


def test_mixed_feed_at_the_abi(lib):
    abi_mixed(lib, _cuda)


def test_abi_misuse(lib):
    abi_misuse(lib)


def test_every_form_of_counts(lib):
    import torch
    text = synth.readme_corpus(n_lines=200)
    t = BPE.count_words(text)
    want = train_text(text, 300)
    ws = [w for w, _ in entries(t)]
    cnt = t.counts
    forms = [t, write_tsv(t),
             dict([(w.decode("utf-8", "surrogateescape"), int(c)) for w, c in zip(ws, cnt)] + [("", t.separators)]),
             dict([(w, int(c)) for w, c in zip(ws, cnt)] + [(b"", t.separators)]),
             WordCounts(_cuda(t.word_bytes), _cuda(t.word_offsets), _cuda(t.counts), t.separators, None),
             WordCounts(torch.from_numpy(t.word_bytes), torch.from_numpy(t.word_offsets.astype(np.int64)),
                        torch.from_numpy(t.counts.astype(np.int64)), t.separators, None)]
    for form in forms:
        assert train_table(form, 300) == want, type(form).__name__
    # without separators: one per occurrence, the text "w w w ... " with a space after every occurrence
    assert train_table((ws, cnt), 300) == train_table((ws, torch.from_numpy(cnt.astype(np.int64))), 300) == \
        train_text(expand(ws, cnt.tolist()), 300)


@pytest.mark.parametrize("word", [b"a b", b"a\tb", b"a\rb", "a▁b".encode(), b"a\nb"])
def test_words_with_a_separator_are_rejected(lib, word):
    with pytest.raises(ValueError, match=r"entry 1 .*separator"):
        BPE.train_from_counts(([b"ok", word], np.array([1, 1])), tmp_model_path("x"), 50)


@pytest.mark.parametrize("body, line", [(b"\t3\nab\t2\ncd 4\n", 3), (b"ab\t2\ncd\tx\n", 2), (b"ab\t-3\n", 1),
                                        (b"ab\t2\n\t1\n\t1\n", 3), (b"ab\t\n", 1)])
def test_tsv_errors_name_the_line(lib, body, line):
    path = os.path.join(_tmp, "bad.tsv")
    with open(path, "wb") as f:
        f.write(body)
    with pytest.raises(ValueError, match="line %d:" % line):
        BPE.train_from_counts(path, tmp_model_path("x"), 50)


def test_type_errors(lib):
    m = tmp_model_path("x")
    for bad in (5, [b"a"], ([1, 2], np.array([1, 1])), {b"a": 1.5}, {1: 2}, ([b"a"], [1]),
                ([b"a"], np.array([1.0]))):
        with pytest.raises(TypeError):
            BPE.train_from_counts(bad, m, 50)
    with pytest.raises(ValueError):
        BPE.train_from_counts({b"a": -1}, m, 50)
    with pytest.raises(TypeError):
        BPE.count_words(3.5)


def test_scale_256mb(lib):
    """A 256 MB synthetic corpus at the default pieces, vocab 32k: the table's model is BPE.train's, and the table
    training needs less device memory than the text training (the table is far smaller than the corpus)."""
    from youtokentome_b200.youtokentome import train_report
    text = synth.FastZipf(n_words=200_000, seed=3).text(256 << 20)
    path = F.corpus_file(text)
    del text
    m_text, m_tab = tmp_model_path("big"), tmp_model_path("bigt")
    with FG.env(YTTM_TRAIN_FEED_ABOVE=0):
        BPE.train(path, m_text, 32000)
    peak_text = train_report()["device_peak_bytes"]
    t = BPE.count_words(path)
    BPE.train_from_counts(t, m_tab, 32000)
    r = train_report()
    assert read(m_tab) == read(m_text)
    assert r["n_words"] == int(t.counts.sum()) and r["n_unique"] <= len(t.counts) and r["data_len"] == t.data_len
    assert r["device_peak_bytes"] < peak_text, (r["device_peak_bytes"], peak_text)
    os.remove(path)


def test_cli(lib):
    text = synth.readme_corpus(n_lines=300)
    corpus = F.corpus_file(text)
    tsv, m_a, m_b = os.path.join(_tmp, "cli.tsv"), tmp_model_path("cli_a"), tmp_model_path("cli_b")
    cli = [sys.executable, "-m", "youtokentome_b200.yttm_cli"]
    r = subprocess.run(cli + ["count_words", "--data", "-", "--output", tsv], input=text, cwd=ROOT,
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.returncode == 0, r.stderr.decode()
    assert b"count_words:" in r.stderr.splitlines()[-1]
    for args in (["bpe_counts", "--data", tsv, "--model", m_a], ["bpe", "--data", corpus, "--model", m_b]):
        r = subprocess.run(cli + args + ["--vocab_size", "400"], cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        assert r.returncode == 0, r.stderr.decode()
    assert read(m_a) == read(m_b)

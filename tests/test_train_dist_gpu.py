"""Training as bench.py times it, on the GPU: youtokentome_b200.distributed.train_distributed at one rank (LocalComm)
and the calls it makes — dist_init / connect, load or feed, char_hist, set_alphabet, dist_word_table,
dist_export_words (word_export_kernel, two passes) and dist_import_words (word_insert_list_kernel: a second word table
built from a list of words with counts), then the tokens, the pair table and the merge loop.

  A. the one-rank front: the export's pointers passed straight to the import, as LocalComm.all_to_all does; words,
     counts, pair table, n_words / n_unique / n_tokens against the restatement of tests/_front_ref.py;
  B. the export at 2, 3, 5 and 8 ranks on one device, one rank after the other and never connected, checked buffer by
     buffer (owner = the restated hash, positions, one space behind each word, each rank's words with their counts);
     then every destination's list imported at one rank, where equal words from several sources, with counts > 1,
     race for one slot of word_insert_list_kernel;
  C. crafted lists through dist_import_words: duplicates, counts above 32 bits through the merge loop against the
     words-in oracle, removed characters, an empty list, a 20 KB word, and the limit freq x tokens < 2^43;
  D. whole trainings through train_distributed: the model file byte for byte what yttm_api_train_memory writes, the same
     statistics, the reference's or the oracle's model, and the API's error texts;
  E. the corpora of bench.py's configs 3 and 5.

No test here runs dist_connect, dist_import_words, build or run on a context of world > 1: those wait for peer
kernels.  The bodies take the library and `dev`: tests/test_train_dist_emul_cpu.py runs A - D on the SIMT emulator
with dev=False (device memory is host memory there) at small sizes."""
import collections
import ctypes as C
import os
import time

import numpy as np
import pytest

import _cases
import _front_ref as R
import test_train_feed_gpu as F
import test_train_front_gpu as FG
import test_train_loop_gpu as TL
from _bind import read_model, tmp_model_path
from youtokentome_b200 import _lib, synth
from youtokentome_b200 import distributed as D

pytestmark = pytest.mark.gpu
M64 = (1 << 64) - 1
WORLDS = [2, 3, 5, 8]
LIMIT_MSG = "yttm_train_dist_import_words: a word's frequency x tokens must stay below 2^43"


# ---- buffers: device memory through torch on the GPU, host memory on the emulator --------------------------------------
def to_host(ptr, n, dtype, dev):
    """n items of `dtype` from the library's buffer at `ptr`."""
    nbytes = n * np.dtype(dtype).itemsize
    if not nbytes:
        return np.zeros(0, dtype=dtype)
    if dev:
        import torch
        return torch.as_tensor(D._DevView(ptr, nbytes, "|u1"), device="cuda").cpu().numpy().view(dtype).copy()
    return np.frombuffer(C.string_at(ptr, nbytes), dtype=dtype).copy()


def to_device(arr, dev):
    """(pointer, keep-alive) of a copy of `arr`: a torch CUDA tensor on the GPU, a numpy array on the emulator."""
    raw = np.ascontiguousarray(arr).view(np.uint8).ravel()
    raw = raw.copy() if raw.size else np.zeros(1, dtype=np.uint8)
    if dev:
        import torch
        t = torch.from_numpy(raw).cuda()
        torch.cuda.synchronize()
        return t.data_ptr(), t
    return raw.ctypes.data, raw


# ---- the owner of a word, restated --------------------------------------------------------------------------------------
def _mix64(h):
    h ^= h >> 33
    h = (h * 0xff51afd7ed558ccd) & M64
    h ^= h >> 33
    h = (h * 0xc4ceb9fe1a85ec53) & M64
    return h ^ (h >> 33)


def owner(word, world):
    """word_export_kernel's destination: FNV-1a of the bytes plus the length, mixed; its top 32 bits scaled to world."""
    h = 0xcbf29ce484222325
    for b in word:
        h = ((h ^ b) * 0x100000001b3) & M64
    return ((_mix64((h + len(word)) & M64) >> 32) * world) >> 32


# ---- one rank's context ---------------------------------------------------------------------------------------------------
class Rank(TL.Ctx):
    """A context after yttm_train_dist_init(rank, world); connected (to itself) only at world 1."""

    def __init__(self, L, rank=0, world=1):
        super().__init__(L)
        handle = C.create_string_buffer(128)
        assert L.yttm_train_dist_init(self.h, rank, world, handle) == 0, self.err()
        if world == 1:
            assert L.yttm_train_dist_connect(self.h, handle.raw) == 0, self.err()

    def load(self, text, feed_kb=None):
        """load_corpus (feed_kb: fed in blocks of random sizes, pieces of feed_kb KB) + char_hist -> (data_len, hist)"""
        L = self.L
        if feed_kb:
            with FG.env(YTTM_TRAIN_FEED_PIECE_KB=feed_kb):
                F.feed_blocks(L, self.h, text, F._sizes("random"))
        else:
            assert L.yttm_train_load_corpus(self.h, C.cast(C.c_char_p(text), C.c_void_p), len(text), 0) == 0, self.err()
        dl, nd = C.c_uint64(0), C.c_uint64(0)
        assert L.yttm_train_char_hist(self.h, C.byref(dl), C.byref(nd)) == 0, self.err()
        cps = np.zeros(nd.value, dtype=np.uint32)
        cnt = np.zeros(nd.value, dtype=np.uint64)
        L.yttm_train_get_char_hist(self.h, cps.ctypes.data, cnt.ctypes.data)
        return dl.value, dict(zip(cps.tolist(), cnt.tolist()))

    def set_alphabet(self, cp2id):
        kc = np.array(list(cp2id), dtype=np.uint32)
        ki = np.array(list(cp2id.values()), dtype=np.uint32)
        assert self.L.yttm_train_set_alphabet(self.h, kc.ctypes.data, ki.ctypes.data, len(kc), FG.SPACE_ID) == 0

    def export_words(self, world):
        """dist_word_table + dist_export_words -> (bytes per destination, words per destination, (bytes, pos, freq)
        device pointers)"""
        nu = C.c_uint64(0)
        assert self.L.yttm_train_dist_word_table(self.h, C.byref(nu)) == 0, self.err()
        bpd, wpd = (C.c_uint64 * 8)(), (C.c_uint64 * 8)()
        p_b, p_p, p_f = C.c_void_p(), C.c_void_p(), C.c_void_p()
        assert self.L.yttm_train_dist_export_words(self.h, bpd, wpd, C.byref(p_b), C.byref(p_p), C.byref(p_f)) == 0, \
            self.err()
        assert sum(wpd) == nu.value
        return list(bpd)[:world], list(wpd)[:world], (p_b.value, p_p.value, p_f.value)

    def import_words(self, p_b, n_bytes, p_p, p_f, n_words):
        """dist_import_words of one source -> the statistics; ValueError(message) when it fails."""
        st = _lib.TrainStats()
        if self.L.yttm_train_dist_import_words(self.h, p_b, (C.c_uint64 * 8)(n_bytes), p_p, p_f,
                                               (C.c_uint64 * 8)(n_words), C.byref(st)) != 0:
            raise ValueError(self.err())
        return st


def import_list(r, data, pos, freq, dev):
    """The received bytes / positions / counts as caller buffers into dist_import_words -> the statistics."""
    (pb, kb), (pp, kp), (pf, kf) = (to_device(np.frombuffer(data, dtype=np.uint8), dev),
                                    to_device(np.asarray(pos, dtype=np.uint64), dev),
                                    to_device(np.asarray(freq, dtype=np.uint64), dev))
    st = r.import_words(pb, len(data), pp, pf, len(pos))
    del kb, kp, kf
    return st


def word_list(words):
    """[(byte-word, count)] (repeats allowed) -> the export's layout: bytes (each word followed by one space), pos, freq."""
    data, pos, freq = bytearray(), [], []
    for w, f in words:
        pos.append(len(data))
        freq.append(f)
        data += w + b" "
    return bytes(data), pos, freq


# ---- A. the one-rank front ----------------------------------------------------------------------------------------------
def dist_front(L, text, cp2id, feed_kb=None):
    """train_distributed's calls up to the import at one rank -> the fields of _front_ref.expected_front."""
    r = Rank(L)
    try:
        dl, hist = r.load(text, feed_kb)
        r.set_alphabet(cp2id)
        bpd, wpd, (pb, pp, pf) = r.export_words(1)
        st = r.import_words(pb, bpd[0], pp, pf, wpd[0])   # as LocalComm.all_to_all: the export's own buffers
        return dict(F.words_and_pairs(L, r.h, st), data_len=dl, hist=hist)
    finally:
        r.close()


def check_front(L, text, what, feed_kb=None):
    want, cp2id = FG.expected(text)
    FG.assert_same(dist_front(L, text, cp2id, feed_kb), want, "%s (%d bytes)" % (what, len(text)))


def front_pieces(L, small=False):
    for name in ("chunk", "warp", "block", "soup"):
        check_front(L, FG.corpus(name, small), name)


def front_edges(L, small=False):
    for k, text in enumerate(FG.edge_corpora()):
        check_front(L, text, "edge corpus %d" % k)
    for k, text in enumerate(FG.length_corpora()):
        check_front(L, text, "length corpus %d" % k)
    for name, text, *_ in F.edge_corpora(small):
        check_front(L, text, name)


def front_pipelined(L, piece_kb, small=False):
    """dist_word_table takes over the word table built while the text was copied (config 3 at full size)."""
    with FG.env(YTTM_TRAIN_PIPELINE=1, YTTM_TRAIN_PIPELINE_PIECE_KB=piece_kb):
        for name in ("chunk", "soup"):
            check_front(L, FG.corpus(name, small), "%s, pipelined in %s KB pieces" % (name, piece_kb))


def front_overflow(L, pipelined):
    with FG.env(YTTM_TRAIN_PIPELINE=int(pipelined), YTTM_TRAIN_PIPELINE_PIECE_KB=64):
        check_front(L, FG.overflow_corpus(), "word table overflow" + (", pipelined" if pipelined else ""))


def front_fed(L, small=False):
    """A shard loaded by feeding: dist_word_table keeps the words feed_end built, with their counts."""
    for text in (F.abi_text(small)[:12_000 if small else 100_000], _cases.dirty_zipf_text(20_000 if small else 200_000)):
        check_front(L, text, "fed in 1 KB pieces", feed_kb=1)


# ---- B. the export at W ranks, the owners' imports at one ----------------------------------------------------------------
def export_rank(L, shard, rank, world, dev, feed_kb=None):
    """Rank `rank` of `world`: load (or feed) its shard, char_hist, dist_word_table, dist_export_words; the three buffers
    copied to the host; the context destroyed."""
    r = Rank(L, rank, world)
    try:
        dl, hist = r.load(shard, feed_kb)
        bpd, wpd, (pb, pp, pf) = r.export_words(world)
        nb, nw = sum(bpd), sum(wpd)
        return dict(data_len=dl, hist=hist, bpd=bpd, wpd=wpd, bytes=to_host(pb, nb, np.uint8, dev).tobytes(),
                    pos=to_host(pp, nw, np.uint64, dev), freq=to_host(pf, nw, np.uint64, dev))
    finally:
        r.close()


def destinations(ex, world, what):
    """One rank's export cut per destination and checked: its bytes are its words back to back, each non-empty, free of
    space units and followed by exactly one 0x20, at `pos` relative to the destination's first byte; every word goes to
    owner(word).  -> [(segment bytes, pos, freq, {word: count})] per destination."""
    assert len(ex["bytes"]) == sum(ex["bpd"]) and len(ex["pos"]) == len(ex["freq"]) == sum(ex["wpd"]), what
    out, b0, w0 = [], 0, 0
    for d in range(world):
        seg = ex["bytes"][b0:b0 + ex["bpd"][d]]
        pos, freq = ex["pos"][w0:w0 + ex["wpd"][d]], ex["freq"][w0:w0 + ex["wpd"][d]]
        words, at = {}, 0
        for i in np.argsort(pos, kind="stable").tolist():
            p, f = int(pos[i]), int(freq[i])
            assert p == at, "%s, destination %d: a word at byte %d, the bytes before it end at %d" % (what, d, p, at)
            e = seg.find(b" ", p)
            assert e > p, "%s, destination %d: no word, or no space behind it, at byte %d" % (what, d, p)
            w = seg[p:e]
            assert R.byte_words(w) == [w], "%s, destination %d: %r is not one word" % (what, d, w)
            assert owner(w, world) == d, "%s: %r sent to %d, its owner is %d" % (what, w, d, owner(w, world))
            assert w not in words and f > 0, (what, w, f)
            words[w] = f
            at = e + 1
        assert at == len(seg), "%s, destination %d: %d bytes, the words end at %d" % (what, d, len(seg), at)
        out.append((seg, pos, freq, words))
        b0 += ex["bpd"][d]
        w0 += ex["wpd"][d]
    return out


def check_exports(L, text, world, dev, feed_rank=None, balance=False):
    """Every rank's export against the restatement, then each destination's words imported at one rank."""
    cut = D.split_byte_ranges(text, world)
    shards = [text[cut[r]:cut[r + 1]] for r in range(world)]
    exs = [export_rank(L, s, r, world, dev, 1 if r == feed_rank else None) for r, s in enumerate(shards)]
    dl, hist = R.char_hist(text)
    assert sum(e["data_len"] for e in exs) == dl
    assert sum((collections.Counter(e["hist"]) for e in exs), collections.Counter()) == collections.Counter(hist)
    per = [destinations(e, world, "rank %d of %d" % (r, world)) for r, e in enumerate(exs)]
    for r in range(world):
        mine = {w: f for seg in per[r] for w, f in seg[3].items()}
        assert mine == collections.Counter(R.byte_words(shards[r])), "rank %d of %d: words or counts differ" % (r, world)
    where = {}
    for r in range(world):
        for d in range(world):
            for w in per[r][d][3]:
                assert where.setdefault(w, d) == d, "%r goes to %d from one rank and to %d from another" % (w, where[w], d)
    owned = [set().union(*(per[r][d][3] for r in range(world))) for d in range(world)]
    assert sum(map(len, owned)) == len(where) and set(where) == set(R.byte_words(text))
    if balance:
        U = len(where)
        assert U >= 10_000
        assert all(U / (2 * world) <= len(o) <= 2 * U / world for o in owned), (U, [len(o) for o in owned])
    # the owners: W sources back to back, positions rebased by the bytes in front of each segment
    want, cp2id = FG.expected(text)
    total = dict(n_words=0, n_unique=0, n_tokens=0, pairs=collections.Counter())
    for d in range(world):
        segs = [per[r][d] for r in range(world)]
        base = np.cumsum([0] + [len(s[0]) for s in segs])
        data = b"".join(s[0] for s in segs)
        pos = np.concatenate([s[1] + np.uint64(b) for s, b in zip(segs, base)])
        freq = np.concatenate([s[2] for s in segs])
        r = Rank(L)
        try:
            r.set_alphabet(cp2id)
            st = import_list(r, data, pos, freq, dev)
            got = F.words_and_pairs(L, r.h, st)
        finally:
            r.close()
        counts = sum((collections.Counter(s[3]) for s in segs), collections.Counter())
        mine = R.expected_words(counts, cp2id, FG.SPACE_ID)
        for k in ("n_words", "n_unique", "n_tokens", "words", "pairs"):
            assert got[k] == mine[k], "owner %d of %d: %s differs" % (d, world, k)
        for k in ("n_words", "n_unique", "n_tokens"):
            total[k] += got[k]
        total["pairs"].update(got["pairs"])
    for k in ("n_words", "n_unique", "n_tokens", "pairs"):
        assert total[k] == want[k], "%d ranks: %s summed over the owners differs from the whole text's" % (world, k)


def export_corpora(small=False):
    """(name, text, rank fed in 1 KB pieces or None)"""
    half = _cases.zipf().text(6_000 if small else 40_000)
    out = [(os.path.basename(p)[:-5], F.golden(p)[0], None) for p in F.GOLDEN]
    out += [("dirty zipf", _cases.dirty_zipf_text(30_000 if small else 200_000), None),
            ("adversarial pieces", FG.corpus("chunk"), None),
            ("one shard without a word", b"abab abab cd " + b" " * 4000 + b"\t\n" * 2000, None),
            ("the same words in every shard", half + b" " + half, None),
            ("fewer unique words than ranks", b"ab cd ab ab cd " * 40, None),
            ("one shard fed", _cases.dirty_zipf_text(30_000 if small else 200_000), 1)]
    return out


# ---- C. crafted lists -----------------------------------------------------------------------------------------------------
def _alphabet_of(words):
    return FG.alphabet(R.char_hist(b" ".join(w for w, _ in words))[1])


def check_list(L, words, dev, oracle=None, merges=0):
    """[(byte-word, count)] (repeats allowed) imported at one rank: the words and the pair table of the restatement;
    with merges, then yttm_train_run against the words-in oracle (rules, words afterwards, pair table)."""
    counts = collections.Counter()
    for w, f in words:
        counts[w] += f
    cp2id = _alphabet_of(words)
    r = Rank(L)
    try:
        r.set_alphabet(cp2id)
        st = import_list(r, *word_list(words), dev)
        got = F.words_and_pairs(L, r.h, st)
        want = R.expected_words(counts, cp2id, FG.SPACE_ID)
        for k in ("n_words", "n_unique", "n_tokens", "words", "pairs"):
            assert got[k] == want[k], "%s differs" % k
        if merges:
            w = r.export()
            w.check_initial_ids()
            TL.check_run(r, oracle, w, max(cp2id.values()) + 1, merges)
        return got
    finally:
        r.close()


def crafted_duplicates(L, dev):
    """One word listed 1 000 times with count 1, one listed twice with 2^32 - 1: counts sum in one slot."""
    got = check_list(L, [(b"bcb", 1)] * 1000 + [("жжb".encode(), 2 ** 32 - 1)] * 2 + [(b"ce", 7)], dev)
    assert sorted(f for _, f in got["words"]) == [7, 1000, 2 ** 33 - 2]


def crafted_large_counts(L, oracle, dev):
    """Counts near 2^32 and 2^33 reach the pair table and the merge loop."""
    rng = np.random.default_rng(3)
    words = [(b"bcbc", 2 ** 32 - 3), (b"bcbc", 5), (b"cb", 2 ** 33 + 7), (b"bbbcc", 2 ** 32 + 1), (b"efbc", 2 ** 33 - 1),
             ("жbж".encode(), 2 ** 32)]
    words += [(bytes(rng.choice(list(b"bcefhk"), size=int(n)).tolist()), int(f))
              for n, f in zip(rng.integers(1, 12, 300), rng.integers(1, 1 << 20, 300))]
    check_list(L, words, dev, oracle, 40)


def crafted_edges(L, oracle, dev):
    """Words of removed characters only (they vanish), an empty list, and a 20 KB word (longer than a tile)."""
    got = check_list(L, [(b"aad", 9), (b"gda", 3), (b"bca", 2), (b"ad", 1)], dev)   # a, d, g: removed
    assert got["n_unique"] == 1 and got["n_words"] == 15
    got = check_list(L, [], dev)
    assert got["n_unique"] == got["n_tokens"] == got["n_words"] == 0 and got["pairs"] == {}
    rng = np.random.default_rng(8)
    long_word = bytes(rng.choice(list(b"bcef"), size=20_000).tolist())
    check_list(L, [(long_word, 3), (b"bc", 10), (long_word[:5000], 2), (b"efbc", 4)], dev, oracle, 30)


def crafted_limits(L, oracle, dev):
    """freq x tokens < 2^43: a two-token word with 2^42 fails with the message, and so does 2^41 + 2^41 reached only
    through duplicates (each entry alone passes); 2^42 - 1 trains."""
    for words in ([(b"b", 2 ** 42)], [(b"b", 2 ** 41)] * 2, [(b"b", 2 ** 41), (b"ce", 5), (b"b", 2 ** 41)],
                  [(b"bc", 2 ** 43 // 3 + 1)]):
        r = Rank(L)
        try:
            r.set_alphabet(_alphabet_of(words))
            with pytest.raises(ValueError) as e:
                import_list(r, *word_list(words), dev)
            assert str(e.value) == LIMIT_MSG, words
        finally:
            r.close()
    check_list(L, [(b"b", 2 ** 42 - 1), (b"ce", 3)], dev, oracle, 2)
    check_list(L, [(b"bc", 2 ** 43 // 3 - 1)], dev, oracle, 2)


# ---- D. whole trainings ---------------------------------------------------------------------------------------------------
def check_training(L, text, vocab, cov=1.0, special=(0, 1, 2, 3), sharded=True, want=None, oracle=None):
    """train_distributed at one rank: the file yttm_api_train_memory writes, the same n_unique / n_tokens / n_merges,
    the model `want` or the oracle's; or the API's error text."""
    pad, unk, bos, eos = special
    m_api, m = tmp_model_path("api"), tmp_model_path("dist")
    if L.yttm_api_train_memory(text, len(text), m_api.encode(), vocab, cov, pad, unk, bos, eos) != 0:
        msg = L.yttm_api_last_error(None).decode()
        with pytest.raises(ValueError) as e:
            D.train_distributed(text, m, vocab, cov, pad, unk, bos, eos, comm=D.LocalComm(), device=0, lib=L,
                                sharded=sharded)
        assert str(e.value) == msg
        return None
    rep = F.report(L)
    st = {}
    n = D.train_distributed(text, m, vocab, cov, pad, unk, bos, eos, comm=D.LocalComm(), device=0, lib=L,
                            sharded=sharded, stats_out=st)
    assert F.same_file(m, m_api), "train_distributed's model file differs from yttm_api_train_memory's"
    assert (st["n_unique"], st["n_tokens"], st["n_merges"], n) == \
        (rep["n_unique"], rep["n_tokens"], rep["n_merges"], rep["n_merges"]), (st, rep)
    if oracle is not None:
        m_o = tmp_model_path("orc")
        oracle.train(text, m_o, vocab, cov, pad=pad, unk=unk, bos=bos, eos=eos)
        want = read_model(m_o)
    if want is not None:
        assert read_model(m) == want
    return st


def golden_training(L, path, sharded):
    text, vocab, cov, special, want = F.golden(path)
    check_training(L, text, vocab, cov, (special["pad"], special["unk"], special["bos"], special["eos"]), sharded, want)


SPECIAL_LAYOUTS = [((-1, 5, 29, -1), 1.0), ((7, 0, 3, 299), 0.999), ((-1, 1, 2, 3), 1.0), ((-1, 9, -1, -1), 0.9995)]
KNOBS = [dict(YTTM_FORCE_STREAM=1, YTTM_STREAM_Q=64), dict(YTTM_XQ_SEG_CAP=8), dict(YTTM_PAIR_CAP_FLOOR=16),
         dict(YTTM_FRONT_TOP=1), dict(YTTM_NEWP_LIMIT=1), dict(YTTM_TRAIN_PIPELINE=1, YTTM_TRAIN_PIPELINE_PIECE_KB=1)]


def special_layouts(L, oracle, small=False):
    """U+2581 takes the first id that no special token holds: id 0 in the last two layouts."""
    text = synth.readme_corpus(n_lines=100 if small else 300)
    for special, cov in SPECIAL_LAYOUTS:
        check_training(L, text, 300, cov, special, oracle=oracle)


def knob_training(L, oracle, knob, small=False):
    text = _cases.zipf().text(20_000 if small else 200_000)
    with FG.env(**knob):
        check_training(L, text, 500 if small else 2000, 1.0, oracle=oracle)
        check_training(L, _cases.dirty_zipf_text(20_000 if small else 100_000), 400, 0.98, oracle=oracle)


def edge_trainings(L, oracle, small=False):
    rng = np.random.default_rng(9)
    long_word = bytes(rng.choice(list(b"abc"), size=8_000 if small else 60_000).tolist())
    words = [bytes(rng.choice(list(b"abcd"), size=int(n)).tolist()) for n in rng.integers(1, 90, 600 if small else 3000)]
    for text, vocab in [(b"", 10), (b"   \n\t ", 10), (b"a", 10), (b"\xff\xfe", 10), (b"ab ab ab", 1000),
                        (synth.readme_corpus(n_lines=60 if small else 300, seed=3) + long_word + b" ab", 300),
                        (b" ".join(words), 400 if small else 600)]:
        check_training(L, text, vocab, oracle=oracle)


def error_texts(L):
    """Vocabulary too small, coverage out of range, special ids out of range or equal: train_distributed says what
    yttm_api_train says (which checks the configuration where the reference's train_bpe does)."""
    text = b"abcdefgh ijkl mn"
    path = F.corpus_file(text)
    for vocab, cov, special in [(6, 1.0, (0, 1, 2, 3)), (100, 1.5, (0, 1, 2, 3)), (100, 0.0, (0, 1, 2, 3)),
                                (100, 1.0, (0, 1, 1, 3)), (100, 1.0, (2, 1, 2, 3)), (100, 1.0, (0, 100, 2, 3))]:
        with pytest.raises(ValueError) as api:
            F.train_file(L, path, vocab, cov, *special)
        with pytest.raises(ValueError) as dist:
            D.train_distributed(text, tmp_model_path("dist"), vocab, cov, *special, comm=D.LocalComm(), device=0, lib=L)
        assert str(dist.value) == str(api.value), (vocab, cov, special)


# ---- GPU tests --------------------------------------------------------------------------------------------------------------
@pytest.fixture
def lib(product):
    return product


def test_front_adversarial_pieces(lib):
    front_pieces(lib)


def test_front_edges_and_lengths(lib):
    front_edges(lib)


@pytest.mark.parametrize("piece_kb", ["1", "3", "64"])
def test_front_pipelined(lib, piece_kb):
    front_pipelined(lib, piece_kb)


@pytest.mark.parametrize("pipelined", [False, True])
def test_front_word_table_overflow(lib, pipelined):
    front_overflow(lib, pipelined)


def test_front_fed_shard(lib):
    front_fed(lib)


@pytest.mark.parametrize("world", WORLDS)
def test_export_and_owner_imports(lib, world):
    for name, text, fed in export_corpora():
        check_exports(lib, text, world, True, feed_rank=fed if fed is None else world - 1)


@pytest.mark.parametrize("world", WORLDS)
def test_export_balance(lib, world):
    check_exports(lib, FG.overflow_corpus(), world, True, balance=True)


def test_crafted_duplicates(lib):
    crafted_duplicates(lib, True)


def test_crafted_large_counts(lib, oracle):
    crafted_large_counts(lib, oracle, True)


def test_crafted_edges(lib, oracle):
    crafted_edges(lib, oracle, True)


def test_crafted_count_limit(lib, oracle):
    crafted_limits(lib, oracle, True)


@pytest.mark.parametrize("sharded", [True, False])
@pytest.mark.parametrize("path", F.GOLDEN, ids=[os.path.basename(p)[:-5] for p in F.GOLDEN])
def test_training_golden(lib, path, sharded):
    golden_training(lib, path, sharded)


def test_training_stress_seeds(lib, oracle):
    for seed in range(20):
        text, vocab, cov, _ = _cases.stress_case(seed)
        check_training(lib, text, vocab, cov, oracle=oracle)


def test_training_special_layouts(lib, oracle):
    special_layouts(lib, oracle)


@pytest.mark.parametrize("cov", [1.0, 0.98, 0.9, 0.9999])
def test_training_dirty_zipf_coverage(lib, oracle, cov):
    """Python's choose_alphabet against the C++ coverage cut."""
    check_training(lib, _cases.dirty_zipf_text(), 1500, cov, oracle=oracle)


@pytest.mark.parametrize("knob", KNOBS, ids=["_".join(k) for k in KNOBS])
def test_training_knobs(lib, oracle, knob):
    knob_training(lib, oracle, knob)


def test_training_edges(lib, oracle):
    edge_trainings(lib, oracle)


def test_training_error_texts(lib):
    error_texts(lib)


# ---- E. bench shape -------------------------------------------------------------------------------------------------------
BENCH_CHUNK = 125_000_000


def bench_leg(L, shard, vocab, cov):
    """train_distributed as bench.py's train_leg calls it, then yttm_api_train_memory on the same bytes."""
    st, m, m_api = {}, tmp_model_path("leg"), tmp_model_path("api")
    t0 = time.perf_counter()
    n = D.train_distributed(shard, m, vocab, cov, comm=D.LocalComm(), device=0, sharded=True, stats_out=st)
    t_dist = time.perf_counter() - t0
    assert L.yttm_api_train_memory(shard, len(shard), m_api.encode(), vocab, cov, 0, 1, 2, 3) == 0
    rep = F.report(L)
    assert F.same_file(m, m_api)
    assert (st["n_unique"], st["n_tokens"], n) == (rep["n_unique"], rep["n_tokens"], rep["n_merges"]), (st, rep)
    os.remove(m_api)
    return m, n, t_dist


def test_bench_config3_and_config5_shapes(lib, oracle):
    """Config 3: the 1 GB Zipf corpus of eight 125 MB chunks, vocab 32 000; config 5's chunk 0: multilingual, vocab
    64 000, coverage 0.9999.  The first 16 MB of config 3's chunk 0 also against the oracle."""
    for kind, chunks, vocab, cov in (("zipf", range(8), 32_000, 1.0), ("multilingual", [0], 64_000, 0.9999)):
        t0 = time.perf_counter()
        parts = synth.corpus_chunks(kind, chunks, BENCH_CHUNK)
        t_gen = time.perf_counter() - t0
        if kind == "zipf":
            head = parts[0][:16 << 20]
            head = head[:head.rfind(b" ") + 1]
        shard = b"".join(parts)
        del parts
        m, n, t_dist = bench_leg(lib, shard, vocab, cov)
        print("%s, %d MB: generated in %.1f s, train_distributed %.1f s, %d merges" %
              (kind, len(shard) >> 20, t_gen, t_dist, n))
        del shard
    m, _, _ = bench_leg(lib, head, 32_000, 1.0)
    m_o = tmp_model_path("orc")
    oracle.train(head, m_o, 32_000, 1.0)
    assert read_model(m) == read_model(m_o)

"""The front half of device encode, which decides the ids: the word finder (find_words_vec_kernel), the three merge
kernels (encode_rep_words_kernel, encode_long_words_kernel, encode_words_kernel), the rule table of yttm_enc_create
with rule_rank, and the chunk cutter of enc_run_host (youtokentome_b200/csrc/encode.cu).

Every case compares ids and offsets with the plain restatement of tests/_encode_ref.py for every keyword set of
test_encode_gpu.KW, and with the oracle under BPE-dropout where stated.  The restatement takes (char ids, rules,
special ids) directly, so the cases build the model they need (`runs`, `wrap`, `big`, a duplicated pair) instead of
hoping that a trained one has the property.  The bodies are check_*(oracle, ...); tests/test_encode_words_emul_cpu.py
runs them at smaller sizes (small=True) under the SIMT emulator, where blocks run one after the other: group
reservations in any order, blocks that take one group each, and concurrent warps in the block-per-word kernel only
happen here."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

import _cases
import _encode_ref as ER
import test_encode_gpu as EG
from _bind import _pack, read_model, tmp_model_path
from _gpu import GpuEncoder
from youtokentome_b200 import _lib, synth

pytestmark = pytest.mark.gpu

# constexpr values of youtokentome_b200/csrc/encode.cu (test_encode_words_emul_cpu.py compares them with the source)
LOCAL_W = 40       # slots of the thread-private arrays of encode_rep_words_kernel / encode_words_kernel
LONG_W = 512       # a word that owns more slots gets a block of encode_long_words_kernel
LONG_T = 512       # threads of that block = tokens per chunk of its passes
FIND_TILE = 16384  # bytes of a staged piece of the word finder
FIND_GMAX = 256    # sentences per group at most

SP = b"\xe2\x96\x81"
KW = EG.KW
_cache = {}


# ---- plumbing ------------------------------------------------------------------------------------------------------
class Case:
    """One model file with the three things that encode with it: the library, the restatement, the oracle."""

    def __init__(self, oracle, path):
        self.path, self.model, self.memo = path, read_model(path), {}
        self.g, self.o = GpuEncoder(path), oracle.encoder(path)
        self.kws = [kw for kw in KW if not (kw.get("bos") and self.model[2][2] == -1 or kw.get("eos") and self.model[2][3] == -1)]

    def want(self, sents, **kw):
        return ER.encode(self.model, sents, memo=self.memo, **kw)


def _case(oracle, name, make):
    if name not in _cache:
        _cache[name] = Case(oracle, make())
    return _cache[name]


def zipf_case(oracle):
    return _case(oracle, "zipf", lambda: EG._model(oracle, _cases.dirty_zipf_text(), 1500))


def abcd_case(oracle):
    """Few rules: a word of many KB is merged in few passes."""
    return _case(oracle, "abcd", lambda: EG._model(oracle, b"abcd abca bcd " * 200 + b"ab" * 300, 40))


def _hand(cp2id, rules, special=(1, 0, 2, 3)):
    return ER.write_model(tmp_model_path("hand"), cp2id, rules, special)


RUNS_IDS = dict(sp=4, a=5, b=6, c=7, A=8, B=9, C=10, D=11)


def runs_case(oracle):
    """`runs`: alphabet a b c with (a,a)->A, (A,A)->B, (B,B)->C, (C,C)->D, then (U+2581,a) and (b,b): the rule about
    runs x x x ... (every second occurrence from the run's start) is certain to fire at four levels."""
    r = RUNS_IDS
    cp2id = {0x2581: 4, ord("a"): 5, ord("b"): 6, ord("c"): 7}
    rules = [(r["a"], r["a"], 8), (8, 8, 9), (9, 9, 10), (10, 10, 11), (4, 5, 12), (6, 6, 13)]
    return _case(oracle, "runs", lambda: _hand(cp2id, rules))


def runs0_case(oracle):
    """`runs` without (U+2581,a) and with U+2581 at id 0 (no pad): the "▁" of a word never merges, so every word ends
    in the shift that drops it (chunk by chunk in the block-per-word kernel)."""
    cp2id = {0x2581: 0, ord("a"): 4, ord("b"): 5, ord("c"): 6}
    rules = [(4, 4, 7), (7, 7, 8), (8, 8, 9), (9, 9, 10), (5, 5, 11)]
    return _case(oracle, "runs0", lambda: _hand(cp2id, rules, (1, -1, 2, 3)))


def runs_closed_form(k, ids=RUNS_IDS):
    """The ids of a^k inside a `runs` word (not at its start): D ... D then C, B, A, a by the binary digits of k."""
    return [ids["D"]] * (k >> 4) + [ids[n] for n, bit in (("C", 8), ("B", 4), ("A", 2), ("a", 1)) if k & bit]


def _host(g, buf, offs, bos=False, eos=False, reverse=False, dropout=0.0, seed=None):
    """yttm_api_encode_ids on a packed batch -> (ids int32, id offsets uint64)."""
    L = _lib.lib()
    if seed is not None:
        L.yttm_api_set_dropout_seed(g.h, seed)
    n = len(offs) - 1
    tot = C.c_uint64(0)
    rc = L.yttm_api_encode_ids(g.h, C.cast(C.c_char_p(buf), C.c_void_p), offs.ctypes.data, n, int(bos), int(eos),
                               int(reverse), dropout, C.byref(tot))
    assert rc == 0, L.yttm_api_last_error(g.h)
    ids, oo = np.zeros(max(tot.value, 1), dtype=np.int32), np.zeros(n + 1, dtype=np.uint64)
    L.yttm_api_result_ids(g.h, ids.ctypes.data, oo.ctypes.data)
    return ids[:tot.value], oo


def _device(g, buf, offs, shift, lead, dev, kw):
    """yttm_enc_run_device on a batch that lies `shift` bytes into its buffer and ends at the buffer's last byte, with
    offsets that start at `lead` instead of 0.  dev: the buffers are CUDA tensors, else host memory (emulator)."""
    L = _lib.lib()
    enc, n = L.yttm_api_device_encoder(g.h), len(offs) - 1
    offs = (offs + np.uint64(lead)).astype(np.uint64)
    if dev:
        import torch
        from youtokentome_b200.distributed import _DevView
        raw = torch.empty(shift + len(buf), dtype=torch.uint8, device="cuda")
        raw[shift:] = torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()
        d_offs = torch.from_numpy(offs.astype(np.int64)).cuda()
        torch.cuda.synchronize()
        base, p_offs = raw.data_ptr() + shift, d_offs.data_ptr()
    else:
        raw = np.zeros(shift + len(buf) + 16, dtype=np.uint8)
        raw = raw[(-raw.ctypes.data) % 16:][:shift + len(buf)]
        raw[shift:] = np.frombuffer(buf, dtype=np.uint8)
        base, p_offs = raw.ctypes.data + shift, offs.ctypes.data
    assert base % 16 == shift % 16
    p_ids, p_off, tot = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
    rc = L.yttm_enc_run_device(enc, base, p_offs, len(buf), n, int(kw.get("bos", False)), int(kw.get("eos", False)),
                               int(kw.get("reverse", False)), 0.0, 0, 0, C.byref(p_ids), C.byref(p_off), C.byref(tot))
    assert rc == 0, L.yttm_last_error(L.yttm_api_device_context(g.h))
    if dev:
        ids = torch.as_tensor(_DevView(p_ids.value, max(tot.value, 1), "<i4"), device="cuda")[:tot.value].cpu().numpy()
        oo = torch.as_tensor(_DevView(p_off.value, n + 1, "<i8"), device="cuda").cpu().numpy().astype(np.uint64)
    else:
        ids = np.ctypeslib.as_array(C.cast(p_ids, C.POINTER(C.c_int32)), shape=(max(tot.value, 1),))[:tot.value].copy()
        oo = np.ctypeslib.as_array(C.cast(p_off, C.POINTER(C.c_uint64)), shape=(n + 1,)).copy()
    del raw
    return ids, oo


def _equal(got, want, sents, tag):
    """(ids, id offsets) of the library against list[list[int]]: the first sentence that differs is shown."""
    ids, oo = got
    lens = np.fromiter(map(len, want), dtype=np.int64, count=len(want))
    woo = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    wids = np.fromiter(itertools.chain.from_iterable(want), dtype=np.int32, count=int(woo[-1]))
    if np.array_equal(oo, woo) and np.array_equal(ids, wids):
        return
    for s in range(len(want)):
        g = ids[int(oo[s]):int(oo[s + 1])].tolist()
        if g != want[s]:
            k = next((i for i, (x, y) in enumerate(zip(g, want[s])) if x != y), min(len(g), len(want[s])))
            raise AssertionError("%s: sentence %d (%d bytes, starts %r): %d ids for %d, first difference at id %d: %r != %r"
                                 % (tag, s, len(sents[s]), sents[s][:24], len(g), len(want[s]), k, g[k:k + 6], want[s][k:k + 6]))
    raise AssertionError("%s: offsets differ" % (tag,))


def same(case, sents, kws=None, drop=(), seed=9):
    """The library's ids == the restatement's for every keyword set; == the oracle's for every dropout of `drop`."""
    buf, offs = _pack(sents)
    for kw in case.kws if kws is None else kws:
        _equal(_host(case.g, buf, offs, **kw), case.want(sents, **kw), sents, kw)
    for p in drop:
        ids, oo = case.o.encode_packed(buf, offs, dropout=p, seed=seed)
        got = _host(case.g, buf, offs, dropout=p, seed=seed)
        assert np.array_equal(got[1], oo) and np.array_equal(got[0], ids), ("dropout", p)


def _zipf_text(n, seed):
    t = b" ".join(_cases.zipf().sentences(n // 30 + 2, 60, seed=seed))[:n]
    assert len(t) == n
    return t


def _word(rng, n, parts=(b"a", b"b", b"c", b"d", "ж".encode(), "☃".encode(), b"\xff")):
    return b"".join(parts[i] for i in rng.integers(0, len(parts), n))[:n]


def _sized(rng, n, parts):
    """A word of exactly n bytes from `parts` (padded with ASCII)."""
    w = b""
    while len(w) < n:
        p = parts[int(rng.integers(0, len(parts)))]
        w += p if len(w) + len(p) <= n else b"a"
    return w


def owned(word):
    """Slots a word owns: one per byte and one for its "▁"."""
    assert not any(c in word for c in b" \t\n\x0b\x0c\r") and SP not in word
    return len(word) + 1


# ---- the restatement is the oracle where the oracle is pinned -----------------------------------------------------
def check_restatement_equals_oracle(oracle):
    """Trained models: the 30 stress cases, the golden texts, the dirty Zipf model at coverage 1.0 and 0.9, both id-0
    layouts, each on its sentences and _cases.EDGE_SENTENCES, for every keyword set."""
    todo = []
    for seed in range(30):
        text, vocab, cov, sents = _cases.stress_case(seed)
        todo.append((text, vocab, cov, {}, sents))
    for name in sorted(synth.GOLDEN_TEXTS):
        train, test, vocab = synth.GOLDEN_TEXTS[name]
        todo.append((train.encode(), vocab, 1.0, {}, [test.encode()] + test.encode().split(b"\n")))
    for cov in (1.0, 0.9):
        todo.append((_cases.dirty_zipf_text(), 1500, cov, {}, _cases.zipf_sentences(600)))
    text0 = _cases.zipf().text(60_000) + b" zab zab ab z zz z q"
    n_chars = len(set(text0.decode().replace("\n", " ").replace(" ", "")))
    long_word = b"".join(_cases.zipf().sentences(12, 60, seed=6)).replace(b" ", b"")
    for special in (dict(pad=-1, unk=1, bos=2, eos=3), dict(pad=-1, unk=5, bos=-1, eos=-1)):
        todo.append((text0, n_chars + 5 + 25, 1.0, special, _cases.zipf_sentences(300) + [b"zab", b"z", b"q z zz", long_word, b"q" + long_word]))
    n = 0
    for text, vocab, cov, special, sents in todo:
        m = tmp_model_path("orc")
        try:
            oracle.train(text, m, vocab, cov, **special)
        except ValueError:
            continue
        model, o, memo = read_model(m), oracle.encoder(m), {}
        sents = sents + _cases.EDGE_SENTENCES
        for kw in KW:
            if (kw.get("bos") and model[2][2] == -1) or (kw.get("eos") and model[2][3] == -1):
                continue
            assert ER.encode(model, sents, memo=memo, **kw) == o.encode(sents, **kw), (vocab, cov, special, kw)
        n += 1
    assert n >= 30


# ---- hand-built models ------------------------------------------------------------------------------------------------
def _mix64(h):
    M = (1 << 64) - 1
    h ^= h >> 33
    h = h * 0xff51afd7ed558ccd & M
    h ^= h >> 33
    h = h * 0xc4ceb9fe1a85ec53 & M
    return h ^ (h >> 33)


def rule_hash(x, y):
    """rule_hash of bpe_core.cuh: the low 32 bits of mix64(x << 32 | y)."""
    return _mix64(x << 32 | y) & 0xffffffff


def check_wrap_model(oracle):
    """`wrap`: 14 first-level rules whose home slots are the last four of the 1 024-slot rule table, so that the probe
    chain wraps to slots 0 ..; pairs absent from the rules whose home lies inside the chain (a miss walks around the
    end to the first free slot); words that use the first, a middle and the last entry of the chain."""
    chars = list(range(0x400, 0x400 + 160))                  # Cyrillic: two bytes each
    cp2id = {0x2581: 4, **{cp: 5 + i for i, cp in enumerate(chars)}}
    ids = list(range(5, 165))
    mask = 1023
    tail = [(x, y) for x in ids for y in ids if x != y and rule_hash(x, y) & mask >= 1020]
    assert len(tail) >= 30
    first = tail[:14]
    z0 = 165
    rules = [(x, y, z0 + k) for k, (x, y) in enumerate(first)]
    rules += [(z0, z0 + 1, z0 + 14), (z0 + 13, z0, z0 + 15), (4, z0, z0 + 16)]           # products merge on: (r0,r1), (r13,r0), (▁,r0)
    assert len(rules) <= 500
    slot, table = {}, {}                                      # the table as yttm_enc_create fills it
    for x, y, _ in rules:
        h = rule_hash(x, y) & mask
        while h in table:
            h = (h + 1) & mask
        table[h] = (x, y)
        slot[(x, y)] = h
    chain = [slot[p] for p in first]
    assert max(chain) == 1023 and sorted(s for s in chain if s < 512) == list(range(len([s for s in chain if s < 512])))
    n_wrapped = len([s for s in chain if s < 512])
    assert n_wrapped >= 8, chain
    in_chain = set(range(1020, 1024)) | set(range(n_wrapped))
    absent = [p for p in tail[14:]] + [(x, y) for x in ids[:40] for y in ids[:40]
                                       if x != y and rule_hash(x, y) & mask in in_chain and (x, y) not in slot]
    assert len(absent) >= 16
    case = Case(oracle, _hand(cp2id, rules))
    ch = {i: chr(cp).encode() for cp, i in cp2id.items()}
    word = lambda pairs: b"".join(ch[x] + ch[y] for x, y in pairs)   # noqa: E731
    sents = [word([p]) for p in first] + [word([p]) for p in absent]
    sents += [word([first[0], first[1]]), word([first[13], first[0]]), word([first[7], absent[0], first[13]]),
              word(first), word(first[::-1]), word(absent[:20]), b" ".join(word([p, q]) for p, q in zip(first, absent))]
    rng = np.random.default_rng(11)
    pool = first + absent[:20]
    sents += [b" ".join(word([pool[i] for i in rng.integers(0, len(pool), int(rng.integers(1, 9)))]) for _ in range(12))
              for _ in range(60)]
    got = case.want(sents)
    assert got[0] == [z0 + 16], got[0]
    assert all(len(got[14 + k]) == 3 for k in range(len(absent)))          # a miss: "▁" and two characters
    same(case, sents, drop=(0.3,))


def check_big_model(oracle, n_rules=200_000, n_words=20_000):
    """`big`: 1 000 characters and 200 000 rules (rule k joins two distinct earlier ids, every pair once, so the
    product of rule k appears in later rules only, as in any trained model): a rule table of 2^19 slots.  Words are
    random tokens expanded to their characters, and random character strings."""
    rng = np.random.default_rng(23)
    n_chars = 1000
    cp2id = {0x2581: 4, **{0x4e00 + i: 5 + i for i in range(n_chars)}}
    first_z = 5 + n_chars
    xs = (rng.random(n_rules) * (np.arange(n_rules) + n_chars)).astype(np.int64) + 5
    ys = (rng.random(n_rules) * (np.arange(n_rules) + n_chars)).astype(np.int64) + 5
    seen, rules, left, right, length = set(), [], {}, {}, {}
    for k in range(n_rules):
        x, y = int(xs[k]), int(ys[k])
        while x == y or (x, y) in seen:
            x, y = int(rng.integers(5, first_z + k)), int(rng.integers(5, first_z + k))
        seen.add((x, y))
        z = first_z + len(rules)
        rules.append((x, y, z))
        left[z], right[z] = x, y
        length[z] = length.get(x, 1) + length.get(y, 1)
    if n_rules >= 200_000:
        assert 1 << 18 < 2 * n_rules + 2 <= 1 << 19
    case = Case(oracle, _hand(cp2id, rules))

    def expand(t):
        out, stack = [], [t]
        while stack:
            v = stack.pop()
            if v < first_z:
                out.append(chr(0x4e00 + v - 5))
            else:
                stack += [right[v], left[v]]
        return "".join(out)
    short = [z for z, n in length.items() if n <= 24]
    words = [expand(short[i]) for i in rng.integers(0, len(short), n_words // 2)]
    words += ["".join(chr(0x4e00 + int(c)) for c in rng.integers(0, n_chars, int(rng.integers(1, 12)))) for _ in range(n_words // 2)]
    words += [expand(short[i]) + expand(short[j]) for i, j in rng.integers(0, len(short), (n_words // 10, 2))]
    order = rng.permutation(len(words))
    sents = [" ".join(words[i] for i in order[k:k + 25]).encode() for k in range(0, len(words), 25)]
    want = case.want(sents)
    assert sum(map(len, want)) < 0.8 * sum(len(s.decode().replace(" ", "")) + len(s.split()) for s in sents)   # rules do fire
    same(case, sents, kws=KW[:2])


def check_duplicate_pair(oracle):
    """A pair that is listed twice with different products: the later entry gives the rule index and the product
    (rule2id of the loader keeps the last index; the restatement's dict does the same by construction)."""
    cp2id = {0x2581: 4, ord("a"): 5, ord("b"): 6}
    rules = [(5, 6, 7), (6, 6, 8), (5, 6, 9), (9, 5, 10), (4, 9, 11), (7, 5, 12)]
    case = Case(oracle, _hand(cp2id, rules))
    # (keeping the first entry instead would give [4, 12], [4, 7] and [4, 7, 6])
    assert case.want([b"aba", b"ab", b"abb"]) == [[4, 10], [11], [4, 5, 8]]
    sents = [b"aba", b"ab", b"abb", b"abab ba bab abbb", b"ab" * 30, b"ba" * 300, b"ab" * 300 + b"a", b"b" + b"ab" * 700]
    assert owned(sents[-1]) > LONG_W
    same(case, sents)
    buf, offs = _pack(sents)
    for p in (0.3,):   # the dropout kernel reads the same table
        got = _host(case.g, buf, offs, dropout=p, seed=4)
        ids, oo = case.o.encode_packed(buf, offs, dropout=p, seed=4)
        assert np.array_equal(got[0], ids) and np.array_equal(got[1], oo)


# ---- word finder ------------------------------------------------------------------------------------------------------
def check_groups_longer_than_a_piece(oracle, seed):
    """Groups streamed piece by piece (count, reserve, write): sentences of 40 KB and 200 KB, a 40 KB one without spaces,
    a group of many 1 - 3 KB sentences."""
    case = zipf_case(oracle)
    same(case, [_zipf_text(40_000, 1)], drop=(0.3,))
    same(case, [b"a", _zipf_text(200_000, 2), b"b c"])
    rng = np.random.default_rng(seed)
    many = [_zipf_text(int(k), 10 + i) for i, k in enumerate(rng.integers(1000, 3000, 40))]
    same(case, _cases.zipf_sentences(400) + many + _cases.zipf_sentences(50, seed=4), drop=(0.3,))
    # without spaces the sentence is one word for the block-per-word merge kernel
    c2 = abcd_case(oracle)
    word = bytes(rng.choice(list(b"abcd"), size=40_000).tolist())
    same(c2, [word])
    same(c2, [b"ab", word[:20_000] + b" " + word[:9] + SP + word[:FIND_TILE + 5]])


def check_piece_edges(oracle, edge, step=1):
    """Sentence bounds, U+2581 and a truncated E2 96 at every offset -18 .. 18 around the `edge`-th piece edge of the
    first group (the group starts at batch byte 0, aligned: its piece edges are the multiples of 16 384)."""
    case = zipf_case(oracle)
    for d in range(-18, 19, step):
        s1 = _zipf_text(edge * FIND_TILE + d - 12, 20 + d) + b"a " + SP + b"cd " + b"q" * 3
        s2 = SP + b"ab cd" + SP
        s3 = b"\x81x y\xe2\x96"
        tail = [b"w%d x" % k for k in range(20)]
        same(case, [s1, s2, s3, b"", b"", b"\x96\x81z"] + tail, drop=(0.3,) if d % 6 == 0 else ())
        # the edge inside a word, inside E2 96 81, and right behind a truncated E2 96 at the sentence end
        s4 = _zipf_text(edge * FIND_TILE + d - 2, 60 + d) + SP + b"xy" + SP[:2]
        same(case, [s4, SP[2:] + b"k", b"z"], kws=KW[:1])
    # groups that end exactly at the end of their last piece: the last thread of that piece records the group's end
    whole = [_zipf_text(edge * FIND_TILE - 1, 90 + k) + b"x" for k in range(3)]
    same(case, whole[:1])
    same(case, whole, kws=KW[:2], drop=(0.3,))


def check_group_sizes_and_empty_sentences(oracle):
    """Batches where the group size G does not divide the number of sentences, runs of empty sentences inside groups,
    at the start and at the end, and a batch of empty sentences only."""
    case = zipf_case(oracle)
    base = _cases.zipf_sentences(600, target=128)
    G = FIND_TILE * 3 // 4 // (sum(map(len, base)) // len(base))
    for n in (G * 3 - 1, G * 3 + 1, G - 1, G + 1, 1):
        same(case, base[:n], drop=(0.3,) if n == G * 3 - 1 else ())
    holes = []
    for i, s in enumerate(base[:300]):
        holes += [b""] * (i % 7 == 3) * (1 + i % 5) + [s]
    same(case, [b""] * 9 + holes + [b""] * 150, drop=(0.3,))
    same(case, [b""] * 500, drop=(0.3,))
    same(case, [b""] * 3 + [b" "] + [b""] * 3, drop=(0.3,))


def check_dedup_vector_compare(oracle, monkeypatch, weak):
    """Words of 1 .. 70 bytes that repeat at every alignment mod 16 relative to their representative, pairs that
    differ only in the byte after a 16- or 32-byte boundary, and prefix pairs that end at the sentence end, before a
    space or before U+2581; with equal tags (every probe ends in the byte compare) too."""
    if weak:
        monkeypatch.setenv("YTTM_ENC_DEDUP_WEAKTAG", "1")
    case = zipf_case(oracle)
    rng = np.random.default_rng(5)
    sents = []
    for n in range(1, 71):
        w = _word(rng, n)
        step = 16 * ((n + 1 + 15) // 16) + 1   # occurrence i sits at i mod 16
        s = bytearray(b" " * (15 * step + n))
        for i in range(16):
            s[i * step:i * step + n] = w
        sents.append(bytes(s))
    for k in (15, 16, 17, 31, 32, 33, 47, 48):
        w = _word(rng, k + 9)
        x, y = w[:k] + b"x" + w[k + 1:], w[:k] + b"y" + w[k + 1:]
        sents += [x + b" " + y, b"z" + y + b" " + x, b"zz " + x + SP + y, y, x]
    for k in (1, 2, 15, 16, 17, 31, 32, 33):
        w = _word(rng, k)
        sents += [w, w + b"z " + w, w + b" " + w + b"z", w + SP + w + b"z" + SP, w + b"z", b"q" + SP + w,
                  w + b"\xe2\x96", w + b"\xe2\x96 " + w, w + b"\xe2 " + w + b"\xe2\x96\x81", b"  " + w + b"z" + SP[:2]]
    same(case, sents, drop=(0.3,))
    same(case, sents[::-1] + sents)


def check_many_groups(oracle, n_sm, small=False):
    """More groups than the 4 x SMs blocks of the launch (so that blocks loop over groups) at each group size: sentences
    of 1 - 3 bytes (G = FIND_GMAX), of about 50 bytes, of 12 - 20 KB (G = 1, every group is two pieces), and short
    sentences around one of 2 MB (a small G while one group streams 128 pieces)."""
    case = zipf_case(oracle)
    rng = np.random.default_rng(31)
    text = _cases.zipf().text(400_000)
    tiny_n, mid_n, big_n, huge = (6000, 6000, 24, 200_000) if small else (200_000, 150_000, 3000, 2 << 20)

    def groups(sents):
        mean = max(sum(map(len, sents)) // len(sents), 1)
        G = min(FIND_GMAX, max(FIND_TILE * 3 // 4 // mean, 1))
        return G, (len(sents) + G - 1) // G
    parts = [b"a", b" ", b"b", SP, b"\xe2", b"c ", b"\xff", "ж".encode(), b"d"]
    tiny = [b"".join(parts[i] for i in rng.integers(0, len(parts), 3))[:int(k)] for k in rng.integers(1, 4, tiny_n)]
    G, n = groups(tiny)
    assert G == FIND_GMAX and n > 4 * n_sm
    same(case, tiny, kws=KW[:2])
    at = rng.integers(0, len(text) - 100, mid_n)
    mid = [text[int(p):int(p) + int(k)] for p, k in zip(at, rng.integers(30, 70, mid_n))]
    G, n = groups(mid)
    assert 100 < G < FIND_GMAX and n > 4 * n_sm
    same(case, mid, kws=KW[:2], drop=() if small else (0.3,))
    at = rng.integers(0, len(text) - 21_000, big_n)
    big = [text[int(p):int(p) + int(k)] for p, k in zip(at, rng.integers(12_000, 20_000, big_n))]
    G, n = groups(big)
    assert G == 1 and n > 4 * n_sm
    same(case, big, kws=KW[:1])
    one = (text * (huge // len(text) + 1))[:huge]
    mix = mid[:mid_n // 3] + [one] + mid[mid_n // 3:2 * mid_n // 3]
    G, n = groups(mix)
    assert G < FIND_GMAX and n > 4 * n_sm and len(one) > 10 * FIND_TILE
    same(case, mix, kws=KW[:1])


def check_misaligned_device_batches(oracle, dev):
    """Device-resident batches whose base address is 1 .. 15 mod 16, whose offsets start above 0 and whose last
    sentence ends at the last byte of the buffer: a truncated E2 96, a lone E2, a 33-byte word, a 513-byte word."""
    case = zipf_case(oracle)
    rng = np.random.default_rng(41)
    ends = [b"ab" + SP[:2], b"ab " + SP[:1], b"x " + _word(rng, 33, (b"a", b"b", b"c")), _word(rng, 513, (b"a", b"b", "ж".encode()))]
    assert owned(ends[3]) > LONG_W
    for shift in range(1, 16):
        end = ends[shift % 4]
        sents = _cases.zipf_sentences(40, seed=shift) + [SP + b"x" * 33 + b" " + SP + b"ab", b"", b"q " + end]
        buf, offs = _pack(sents)
        for kw in (KW[0], KW[shift % 3 + 1]):
            got = _device(case.g, buf, offs, shift, 7 * shift, dev, kw)
            _equal(got, case.want(sents, **kw), sents, (shift, kw))


# ---- merge kernels at the path boundaries ---------------------------------------------------------------------------------
MULTI = (b"a", b"b", b"c", "ж".encode(), "☃".encode(), b"\xf0\x9f\x98\x80", b"\xff", b"d", b"e")


def check_local_boundary(oracle):
    """Words that own 39, 40, 41 and 42 slots (38 .. 41 bytes): the last sizes merged in the thread-private arrays and
    the first ones merged in place.  ASCII, and with 2-, 3-, 4-byte characters and 0xFF inside (slots and tokens
    differ); unique and repeated; dropout 0.3 against the oracle (the dropout kernel splits at the same size)."""
    rng = np.random.default_rng(43)
    for case in (zipf_case(oracle), runs_case(oracle)):
        words = []
        for n in (37, 38, 39, 40, 41, 42):
            words += [_sized(rng, n, (b"a", b"b", b"c")) for _ in range(6)] + [_sized(rng, n, MULTI) for _ in range(10)]
            words += [b"a" * n, b"ab" * (n // 2) + b"b" * (n % 2), b"\xff" * (n - 1) + b"a", b"a" + b"\xff" * (n - 1)]
        assert {owned(w) for w in words} == {38, 39, 40, 41, 42, 43}
        sents = [w for w in words] + [b" ".join(words[i::7]) for i in range(7)] + [SP.join(words[::-1][i::5]) for i in range(5)]
        sents += [b" ".join([w] * 3) for w in words[::4]]
        same(case, sents, drop=(0.3,))


def check_long_boundary(oracle):
    """Words of 510 .. 514 bytes (the last thread-per-word sizes and the first block-per-word ones); the same sizes in
    slots but about 130 tokens (128 / 129 four-byte characters); 600 bytes of 0xFF (no valid unit: no ids); 600
    out-of-alphabet characters (one <UNK>); <UNK> runs inside an otherwise mergeable long word."""
    rng = np.random.default_rng(47)
    emoji = b"\xf0\x9f\x98\x80"
    for case in (zipf_case(oracle), runs_case(oracle)):
        words = []
        for n in (510, 511, 512, 513, 514):
            words += [_sized(rng, n, (b"a", b"b", b"c")), _sized(rng, n, MULTI), b"a" * n, b"ab" * (n // 2) + b"a" * (n % 2)]
        out = "\ue000\ue001".encode()     # private-use characters: in no alphabet here
        assert 0xE000 not in case.model[0] and 0xE001 not in case.model[0]
        words += [emoji * 128, emoji * 129, emoji * 128 + b"a", b"a" + emoji * 128, b"\xff" * 600, b"\xff" * 600 + b"a",
                  out * 300, b"ab" * 150 + out * 40 + b"abab" * 50 + emoji * 3 + b"aaaa" * 20,
                  b"a" * 300 + b"\xc0\xaf" + out[:3] + b"a" * 300]
        assert sum(owned(w) > LONG_W for w in words) >= 20 and sum(owned(w) <= LONG_W for w in words) >= 8
        assert case.want([b"\xff" * 600, out * 300]) == [[], [case.model[0][0x2581], case.model[2][0]]]
        sents = words + [b" ".join(words[:8]), b"x " + words[12] + b" y " + words[3] + SP + words[13]]
        same(case, sents)
        same(case, sents[:6] + sents[20:24], kws=[], drop=(0.3,))


def check_token_counts(oracle):
    """Words of 511, 512, 513, 1 023, 1 024, 1 025, 1 536 and 1 537 tokens after decode: the chunk edges of every pass
    of the block-per-word kernel (min scan, apply, compaction, re-lookup)."""
    rng = np.random.default_rng(53)
    counts = (511, 512, 513, 1023, 1024, 1025, 1536, 1537)
    for case, alpha in ((zipf_case(oracle), (b"a", b"b", b"c", b"d", b"e")), (runs_case(oracle), (b"a", b"b", b"c")),
                        (runs0_case(oracle), (b"a", b"b", b"c"))):
        words = [_sized(rng, n - 1, alpha) for n in counts] + [b"a" * (n - 1) for n in counts]
        words += [b"c" + b"a" * (n - 2) for n in counts] + [b"ab" * ((n - 1) // 2) + b"c" * ((n - 1) % 2) for n in counts]
        assert all(owned(w) > LONG_W or owned(w) in (511, 512) for w in words)
        same(case, words)


def check_run_rule_across_chunks(oracle, small=False):
    """`runs` model: prefix + a^k + suffix with a prefix of b / c letters of every length 505 .. 520 and k in 2 .. 9 and
    1 020 .. 1 030, so that a run starts on either parity, ends exactly at a chunk end or spans two whole chunks; two
    runs of which the first ends at token 511 and the second starts at token 512; a^(2^k) and a^(2^k +- 1)."""
    case, r = runs_case(oracle), RUNS_IDS
    rng = np.random.default_rng(59)
    words, want = [], []
    pre_lens = (510, 511, 512, 513) if small else range(505, 521)
    ks = (2, 3, 8, 1023, 1024, 1025) if small else list(range(2, 10)) + list(range(1020, 1031))
    for n in pre_lens:
        for k in ks:
            pre = bytes(rng.choice(list(b"bc"), size=n - 1).tolist()) + b"c"      # ("c" joins nothing: the run stands alone)
            words.append(pre + b"a" * k + b"cb")
    # token 0 is "▁": the run of a ends at token 511, a run of b ((b,b) is a rule too) or the next run of a starts at 512 / 513
    for k1, k2 in ((2, 2), (3, 3), (7, 600), (509, 513), (510, 1024)):
        words.append(b"c" * (511 - k1) + b"a" * k1)
        words.append(b"c" * (511 - k1) + b"a" * k1 + b"b" * k2 + b"c")
        words.append(b"c" * (511 - k1) + b"a" * k1 + b"c" + b"a" * k2 + b"c")
        words.append(b"c" * (510 - k1) + b"a" * k1 + b"c" + b"a" * k2)
    top = 11 if small else 13
    for k in range(1, top + 1):
        for n in (2 ** k - 1, 2 ** k, 2 ** k + 1):
            words.append(b"c" + b"a" * n)
            want.append([r["sp"], r["c"]] + runs_closed_form(n))
    same(case, words)
    assert case.want(words[-len(want):]) == want          # the closed form of a run, a third opinion
    same(runs0_case(oracle), words[::3], kws=KW[:2])


def check_id0_long_words(oracle, small=False):
    """U+2581 at id 0: long words of 513, 1 025 and 5 000 tokens whose "▁" never merges (the shift that drops it moves
    more than one chunk), next to ones whose "▁" does merge (a model with a (▁, a) rule and "▁" at id 0)."""
    rng = np.random.default_rng(61)
    case = runs0_case(oracle)
    counts = (513, 1025, 2000) if small else (513, 1025, 5000)
    words = [_sized(rng, n - 1, (b"a", b"b", b"c")) for n in counts] + [b"c" * (n - 1) for n in counts] + [b"a" * (n - 1) for n in counts]
    got = case.want(words)
    assert all(g and g[0] != 0 for g in got) and len(got[3]) == counts[0] - 1       # "▁" left the output
    same(case, words + [b" ".join(words[:3])])
    cp2id = {0x2581: 0, ord("a"): 4, ord("b"): 5, ord("c"): 6}
    rules = [(4, 4, 7), (7, 7, 8), (0, 7, 9), (0, 6, 10), (5, 5, 11)]
    merged = Case(oracle, _hand(cp2id, rules, (1, -1, 2, 3)))
    words2 = [b"aa" + w for w in words[:3]] + [b"c" + w for w in words[:3]] + [b"b" + words[0], b"ab" + words[1]]
    got = merged.want(words2)
    assert got[0][0] == 9 and got[3][0] == 10 and got[6][0] != 0 and len(got[6]) < len(words2[6])
    same(merged, words2 + words)


def check_more_long_words_than_blocks(oracle, n_sm, small=False):
    """More long words than the launch has blocks (one per SM), so that every block loops over words: distinct words of
    520 .. 900 bytes, each repeated once far away (the dedup hands out one representative)."""
    rng = np.random.default_rng(67)
    n = 12 if small else 400
    assert n > n_sm * (2 if small else 3)
    case = zipf_case(oracle)
    words = [_sized(rng, int(k), MULTI[:5] + (b"d", b"e")) + b"%d" % i for i, k in enumerate(rng.integers(520, 900, n))]
    assert len(set(words)) == n and all(owned(w) > LONG_W for w in words)
    fill = _cases.zipf_sentences(n)
    sents = [w + b" " + f for w, f in zip(words, fill)] + [f[:40] + b" " + w for w, f in zip(words[::-1], fill)]
    same(case, sents, kws=KW[:2])


def check_giant_words(oracle, sizes):
    """One word of many KB on the small models (few rules, few passes).  The restatement is quadratic, so the
    expectation is the closed form of the `runs` model: "c"-separated runs of a."""
    case, r = runs_case(oracle), RUNS_IDS
    rng = np.random.default_rng(71)
    assert case.want([b"c" + b"a" * 77 + b"c" + b"a" * 1000]) == [[r["sp"], r["c"]] + runs_closed_form(77) + [r["c"]] + runs_closed_form(1000)]
    for size in sizes:
        ks, left = [], size - 1
        while left > 0:
            k = int(min(left, rng.integers(1, 5000)))
            ks.append(k)
            left -= k + 1
        word = b"c" + b"c".join(b"a" * k for k in ks)
        want = [r["sp"], r["c"]]
        for i, k in enumerate(ks):
            want += ([r["c"]] if i else []) + runs_closed_form(k)
        one = b"c" + b"a" * (size - 1)
        got = _host(case.g, *_pack([word, b"ab", one]))
        _equal(got, [want, case.want([b"ab"])[0], [r["sp"], r["c"]] + runs_closed_form(size - 1)], [word, b"ab", one], size)


def check_dropout_long_words(oracle):
    """Dropout 0.1 / 0.5 / 1.0 on words of 41 .. 45, 513 and 3 000 bytes against the oracle: the sequential kernel in
    place, its scratch at 6 x the word's first slot; two such words adjacent in one sentence (their scratch ranges
    touch)."""
    rng = np.random.default_rng(73)
    for case in (zipf_case(oracle), runs_case(oracle)):
        w = [_sized(rng, n, (b"a", b"b", b"c")) for n in (41, 42, 43, 44, 45, 513, 3000)] + [_sized(rng, n, MULTI) for n in (41, 45, 513)]
        sents = w + [w[0] + b" " + w[1], w[5] + b" " + w[6] + SP + w[9], w[4] + SP + w[7], b"ab " + w[6] + b" " + w[5] + b" ab"]
        same(case, sents, kws=[], drop=(0.1, 0.5, 1.0))


# ---- id layouts of models ----------------------------------------------------------------------------------------------
def check_special_id_layouts(oracle, special):
    """Special ids below, between and above the ids of the characters and rules (the product of rule k is the k-th
    free id): with and without dropout."""
    m = tmp_model_path("orc")
    oracle.train(_cases.dirty_zipf_text(), m, 1200, 1.0, **special)
    case = Case(oracle, m)
    sents = _cases.zipf_sentences(300) + _cases.EDGE_SENTENCES
    kws = [dict(), dict(reverse=True)] + ([dict(eos=True)] if special.get("eos", 3) != -1 else [])
    same(case, sents, kws=kws, drop=(0.4,), seed=11)
    for kw in kws:
        assert case.want(sents, **kw) == case.o.encode(sents, **kw)


def check_rule_products_are_read_from_the_model(oracle, tmp_path):
    """A model whose rule products are NOT the k-th free id (two product ids swapped by hand): the encoder takes the
    id a rule produces from the model, never from the rule's rank."""
    m = tmp_model_path("orc")
    oracle.train(synth.readme_corpus(n_lines=200), m, 60, 1.0)
    c2i, rules, special = read_model(m)
    a, b = rules[5][2], rules[9][2]
    swap = {a: b, b: a}
    rules2 = [tuple(swap.get(v, v) for v in r) for r in rules]
    case = Case(oracle, ER.write_model(str(tmp_path / "swapped.yttm"), c2i, rules2, special))
    sents = [synth.readme_corpus(n_lines=3, seed=4), b"abab cdcd abcd", b"dddd aaaa"]
    same(case, sents)
    assert case.want(sents) == case.o.encode(sents) != Case(oracle, m).want(sents)


# ---- the host pipeline ---------------------------------------------------------------------------------------------------
def expected_chunks(offs, chunk):
    """The cuts of enc_run_host: as many whole sentences as end within `chunk` bytes of the chunk's start (one at
    least), and a tail shorter than a quarter chunk joins the chunk before it."""
    offs = [int(v) for v in offs]
    n, cut = len(offs) - 1, [0]
    while cut[-1] < n:
        lo = cut[-1]
        hi = max(max(i for i in range(lo, n + 1) if offs[i] <= offs[lo] + chunk), lo + 1)
        if offs[n] - offs[hi] < chunk // 4:
            hi = n
        cut.append(hi)
    return cut


def _chunks_used(case):
    L = _lib.lib()
    return int(L.yttm_stage_ms(L.yttm_api_device_context(case.g.h), b"enc_chunks"))


def check_chunk_cutter(oracle, monkeypatch, small=False):
    """1 MB chunks: the number of chunks the call used is asserted (enc_chunks); a sentence of 3 MB alone in its chunk;
    a tail just under and just over a quarter chunk; a long word that is the last word of one chunk and, repeated, the
    first word of the next (representatives never cross chunks).  Dropout against the oracle: the stream is keyed by
    the sentence index, so it does not move with the cuts."""
    monkeypatch.setenv("YTTM_ENC_CHUNK_MB", "1")
    MB = 1 << 20
    m = EG._model(oracle, _cases.dirty_zipf_text(), 1500)
    case = Case(oracle, m)           # a fresh encoder: the chunk size is read per call, the buffers are its own
    text = _cases.zipf().text(3 * MB + 4096).replace(b"\n", b" ")
    kb = [text[i:i + 1024] for i in range(0, 3 * MB, 1024)]          # sentences of exactly 1 KB
    rng = np.random.default_rng(79)
    long_word = _sized(rng, 600, (b"a", b"b", b"c", "ж".encode()))
    assert owned(long_word) > LONG_W
    a, b = kb[1023], kb[1024]
    kb[1023] = a[:1024 - 601] + b" " + long_word
    kb[1024] = long_word + b" " + b[601:]
    assert len(kb[1023]) == len(kb[1024]) == 1024
    for n_tail, chunks in ((255, 2), (256, 3)):
        sents = kb[:2048 + n_tail]
        offs = _pack(sents)[1]
        cut = expected_chunks(offs, MB)
        assert cut == [0, 1024, 2048 + n_tail] if chunks == 2 else cut == [0, 1024, 2048, 2048 + n_tail]
        same(case, sents, kws=KW[1:2])
        assert _chunks_used(case) == chunks
        if n_tail == 256 or not small:
            same(case, sents, kws=[], drop=(0.2,), seed=77)
            assert _chunks_used(case) == chunks
    if small:
        return
    sents = kb[:300] + [text[:3 * MB]] + kb[300:700] + _cases.EDGE_SENTENCES
    cut = expected_chunks(_pack(sents)[1], MB)
    assert cut[:3] == [0, 300, 301] and len(cut) == 4          # the 3 MB sentence is a chunk of its own
    same(case, sents, kws=KW[:2], drop=(0.2,), seed=77)
    assert _chunks_used(case) == 3


# ---- GPU tests -------------------------------------------------------------------------------------------------------------
def _n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_wrap_model(product, oracle):
    check_wrap_model(oracle)


def test_big_model(product, oracle):
    check_big_model(oracle)


def test_duplicate_pair(product, oracle):
    check_duplicate_pair(oracle)


def test_groups_longer_than_a_piece(product, oracle):
    check_groups_longer_than_a_piece(oracle, 1)


@pytest.mark.parametrize("edge", [1, 2])
def test_piece_edges(product, oracle, edge):
    check_piece_edges(oracle, edge)


def test_group_sizes_and_empty_sentences(product, oracle):
    check_group_sizes_and_empty_sentences(oracle)


@pytest.mark.parametrize("weak", [False, True])
def test_dedup_vector_compare(product, oracle, monkeypatch, weak):
    check_dedup_vector_compare(oracle, monkeypatch, weak)


def test_many_groups(product, oracle):
    check_many_groups(oracle, _n_sm())


def test_misaligned_device_batches(product, oracle):
    check_misaligned_device_batches(oracle, dev=True)


def test_local_boundary(product, oracle):
    check_local_boundary(oracle)


def test_long_boundary(product, oracle):
    check_long_boundary(oracle)


def test_token_counts(product, oracle):
    check_token_counts(oracle)


def test_run_rule_across_chunks(product, oracle):
    check_run_rule_across_chunks(oracle)


def test_id0_long_words(product, oracle):
    check_id0_long_words(oracle)


def test_more_long_words_than_blocks(product, oracle):
    check_more_long_words_than_blocks(oracle, _n_sm())


def test_giant_words(product, oracle):
    check_giant_words(oracle, [100_000, 1_000_000])


def test_dropout_long_words(product, oracle):
    check_dropout_long_words(oracle)


@pytest.mark.parametrize("special", [dict(), dict(pad=-1, bos=-1, eos=7, unk=0), dict(pad=3, unk=40, bos=41, eos=1000)])
def test_special_id_layouts(product, oracle, special):
    check_special_id_layouts(oracle, special)


def test_rule_products_are_read_from_the_model(product, oracle, tmp_path):
    check_rule_products_are_read_from_the_model(oracle, tmp_path)


def test_chunk_cutter(product, oracle, monkeypatch):
    check_chunk_cutter(oracle, monkeypatch)


def _sanitizer(tool, args, timeout=900):
    import shutil
    import subprocess
    import sys
    from _bind import ROOT
    exe = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(exe):
        pytest.skip("compute-sanitizer is not installed")
    env = {k: v for k, v in os.environ.items() if not k.startswith(("YTTM_", "YT_EMU_"))}
    env["PYTORCH_NO_CUDA_MEMORY_CACHING"] = "1"
    r = subprocess.run([exe, "--tool", tool, sys.executable, os.path.join(ROOT, "tools", "sanitize_encode_front.py")] + args,
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout)
    text = r.stdout.decode(errors="replace")
    if "Error: Device not supported" in text:
        pytest.skip("compute-sanitizer does not support this device here")
    assert "batches identical to the restatement" in text, text[-1500:]
    return text


def test_zzz_sanitizer_memcheck_encode_front(product):
    """compute-sanitizer memcheck over tools/sanitize_encode_front.py (device batches at base shifts 1 .. 15, each at the
    end of its own cudaMalloc): no report; skips where the tool refuses the device."""
    text = _sanitizer("memcheck", [])
    assert "ERROR SUMMARY: 0 errors" in text, text[-1500:]


def test_zzz_sanitizer_racecheck_long_words(product):
    """compute-sanitizer racecheck over the long-word batches of the same tool: no shared-memory hazard between the
    warps of encode_long_words_kernel; skips where the tool refuses the device."""
    text = _sanitizer("racecheck", ["--long-only"])
    assert "RACECHECK SUMMARY: 0 hazards" in text, text[-1500:]

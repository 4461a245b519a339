"""BPE-dropout of device encode (encode_words_kernel and the span, padded and subword outputs with dropout > 0 in
youtokentome_b200/csrc/encode.cu) compared directly with the unmodified reference, which replays the product's Philox
draws with its own DropoutQueue (tests/_dropout_ref.py), not with the oracle.

Covered: packed ids from host buffers and from device memory at base addresses 1..15 mod 16 with offsets[0] > 0, every
bos / eos / reverse combination, p from 2^-40 to 1 and p just above a word's first draw; the draw keys (a seed with a
high half, sentence indices that cross 2^32 inside a batch, word offsets above 2^16, one word repeated 1 000 times);
word shapes (both sides of the switch between local arrays and in-place global memory, multi-byte characters, <UNK>
runs, invalid UTF-8 before and inside words, U+2581 at id 0, runs a^k, words of 0.5 to 2 KB); the chunked host
pipeline; the BPE handle's sentence counter across calls and threads; spans, padded rows and subword pieces.
tests/test_encode_dropout_emul_cpu.py runs the same bodies at small sizes under the SIMT emulator."""
import ctypes as C
import threading

import numpy as np
import pytest

import _cases
import _dropout_ref as DR
import test_dropout_reference_cpu as DC
import test_encode_padded_gpu as PG
import test_encode_spans_gpu as SG
from _bind import StoredReference, _pack, read_model, tmp_model_path
from youtokentome_b200 import _lib

pytestmark = pytest.mark.gpu

KWS = SG.KWS                       # the 8 bos / eos / reverse combinations
P = [2.0**-40, 0.125, 0.1, 0.5, 1.0]
REF = StoredReference()


def _model(oracle, text, vocab, cov=1.0, **special):
    m = tmp_model_path("orc")
    oracle.train(text, m, vocab, cov, **special)
    return m


def _zipf_model(oracle):
    return _model(oracle, _cases.dirty_zipf_text(), 1500, 0.98)


def _on_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except ImportError:
        return False


def expected(m, sents, p, seed, first, kw=None, subwords=False):
    """The reference's ids (and pieces) with the draws of sentence indices first, first + 1, ..."""
    return DR.replayed(REF, m, sents, p, seed, first, subwords=subwords, **(kw or {}))


def flags(words_per_sent, m, kw):
    """Ids of replay_batch's word results with <BOS> / <EOS> / reverse applied."""
    _, _, (_, _, bos_id, eos_id) = read_model(m)
    out = []
    for words in words_per_sent:
        i = [bos_id] * kw.get("bos", False) + [x for w in words for x in w["ids"]] + [eos_id] * kw.get("eos", False)
        out.append(i[::-1] if kw.get("reverse", False) else i)
    return out


def enc_run(bpe, sents, kw, p, seed, first, shift=0, lead=0, device=False):
    """yttm_enc_run (host buffers) or yttm_enc_run_device (device memory; host memory under the emulator) with an
    explicit seed and first sentence index, on a batch that starts `shift` bytes past a 16-byte boundary and whose
    offsets start at `lead`.  Returns ids per sentence."""
    L = _lib.lib()
    enc = L.yttm_api_device_encoder(bpe._h)
    buf, offs = _pack(sents)
    n = len(sents)
    offs = (offs + np.uint64(lead)).astype(np.uint64)
    b, e, r = (int(kw.get(k, False)) for k in ("bos", "eos", "reverse"))
    if not device:
        raw = np.zeros(shift + lead + len(buf) + 32, dtype=np.uint8)
        raw = raw[(-raw.ctypes.data) % 16:][:shift + lead + len(buf)]
        raw[shift + lead:] = np.frombuffer(buf, dtype=np.uint8)
        base = raw.ctypes.data + shift
        assert base % 16 == shift % 16
        cap = len(buf) + 3 * n + 16
        ids, oo, tot = np.zeros(cap, dtype=np.int32), np.zeros(n + 1, dtype=np.uint64), C.c_uint64(0)
        rc = L.yttm_enc_run(enc, base, offs.ctypes.data, n, b, e, r, p, seed, first, ids.ctypes.data, cap,
                            oo.ctypes.data, C.byref(tot))
        assert rc == 0, L.yttm_last_error(L.yttm_api_device_context(bpe._h))
        ids = ids[:tot.value]
    else:
        # sentence i of yttm_enc_run_device is d_bytes[offsets[i] - offsets[0], offsets[i + 1] - offsets[0])
        p_ids, p_off, tot = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
        if _on_gpu():
            import torch
            from youtokentome_b200.distributed import _DevView
            raw = torch.zeros(shift + len(buf), dtype=torch.uint8, device="cuda")
            if buf:
                raw[shift:] = torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()
            d_offs = torch.from_numpy(offs.astype(np.int64)).cuda()
            torch.cuda.synchronize()
            base, p_offs = raw.data_ptr() + shift, d_offs.data_ptr()
        else:
            raw = np.zeros(shift + len(buf) + 32, dtype=np.uint8)
            raw = raw[(-raw.ctypes.data) % 16:][:shift + len(buf)]
            raw[shift:] = np.frombuffer(buf, dtype=np.uint8)
            base, p_offs = raw.ctypes.data + shift, offs.ctypes.data
        assert base % 16 == shift % 16
        rc = L.yttm_enc_run_device(enc, base, p_offs, len(buf), n, b, e, r, p, seed, first, C.byref(p_ids),
                                   C.byref(p_off), C.byref(tot))
        assert rc == 0, L.yttm_last_error(L.yttm_api_device_context(bpe._h))
        if _on_gpu():
            ids = torch.as_tensor(_DevView(p_ids.value, max(tot.value, 1), "<i4"), device="cuda")[:tot.value].cpu().numpy()
            oo = torch.as_tensor(_DevView(p_off.value, n + 1, "<i8"), device="cuda").cpu().numpy().astype(np.uint64)
        else:
            ids = np.ctypeslib.as_array(C.cast(p_ids, C.POINTER(C.c_int32)), shape=(max(tot.value, 1),))[:tot.value].copy()
            oo = np.ctypeslib.as_array(C.cast(p_off, C.POINTER(C.c_uint64)), shape=(n + 1,)).copy()
        del raw
    oo = oo.astype(np.int64)
    return [ids[oo[i]:oo[i + 1]].tolist() for i in range(n)]


def same(got, want, sents, tag):
    if got == want:
        return
    for s, (g, w) in enumerate(zip(got, want)):
        if g != w:
            k = next((i for i, (x, y) in enumerate(zip(g, w)) if x != y), min(len(g), len(w)))
            raise AssertionError("%s: sentence %d (%d bytes, starts %r): %d ids for %d, first difference at id %d: "
                                 "%r != %r" % (tag, s, len(sents[s]), sents[s][:24], len(g), len(w), k, g[k:k + 6],
                                               w[k:k + 6]))
    raise AssertionError("%s: %d sentences for %d" % (tag, len(got), len(want)))


def _word_shapes(rng):
    """Sentences of the shapes where the per-word dropout loop can go wrong (see the module docstring)."""
    zc = _cases.zipf()
    lex = [w for s in zc.sentences(60, 60, seed=31) for w in s.split()]
    ascii_words = [w for w in lex if w.isascii() and len(w) >= 4][:40] or [b"abcd"]
    out = []
    for n in (38, 39, 40, 41):                                     # owned = bytes + 1 against LOCAL_W = 40
        w = (b"".join(ascii_words[int(i)] for i in rng.integers(0, len(ascii_words), 20)))[:n]
        out.append(b"x " + w + b" " + w[::-1] + b" y")
    cyr = "жизнь".encode()
    out += [cyr * 8 + b"ab", "ж".encode() * 19 + b"a", "ж".encode() * 20, "日本語テキスト".encode() * 2 + b"ab",
            b"\xf0\x9f\x98\x80ab\xf0\x9f\x98\x80" * 4, b"ab\xf0\x9f\x98\x80" * 10]
    out += [b"\xff\xfeabcab \xc0\xafabab\xff cd\x80ef \xe2\x96abab\xe2\x96\x81ab", b"\xed\xa0\x80" + ascii_words[0] * 3,
            "a一丁b丂 七丄 ab".encode(), b"\xf4\x90\x80\x80zz " + "\U0001F600\U0001F601".encode()]
    out += [b"a" * k for k in (2, 3, 5, 8, 17, 33, 39, 40, 41, 64)]
    out += [b" ".join(b"ab" * k for k in (3, 9, 20, 21))]
    for size in (500, 1100, 2048):                                  # the sequential path of long words
        out.append(b"q " + (b"".join(ascii_words[int(i)] for i in rng.integers(0, len(ascii_words), 400)))[:size])
    return out


# ---- checks, shared with the emulator tests ------------------------------------------------------------------------

def check_packed(oracle, small=False):
    """Packed ids from host buffers and from device memory: every flag combination, p from 2^-40 to 1, bases 1..15
    mod 16 and offsets[0] > 0."""
    m = _zipf_model(oracle)
    bpe = SG._bpe(m)
    rng = np.random.default_rng(3)
    sents = _cases.zipf_sentences(40 if small else 400) + _cases.EDGE_SENTENCES + _word_shapes(rng)
    k = 0
    for p in P:
        seed, first = 1000 + int(p * 64), 17 * k
        words = DR.replay_batch(REF, m, sents, p, seed, first)
        for kw in KWS:
            want = flags(words, m, kw)
            for device in (False, True):
                shift, lead = 1 + k % 15, [0, 5, 4096][k % 3]
                k += 1
                same(enc_run(bpe, sents, kw, p, seed, first, shift, lead, device), want, sents, (p, kw, device, shift))


def check_boundary(oracle):
    """p = (r + 0.5) / 2^32 for a word's first draw r, small, middling and close to 2^32: the reference skips that
    event, a threshold of floor(p * 2^32) would not; at p = r / 2^32 exactly it does not skip."""
    m = DC.boundary_model(oracle)
    bpe = SG._bpe(m)
    for w, idx, seed, r, skip, keep in DC.boundary_cases(REF, m, DC.BOUNDARY_WORDS, ["low", "mid", "high"]):
        sents = [b"  " + w, w + b" " + w, w]
        for p, want in (((r + 0.5) / 2**32, skip), (r / 2**32, keep)):
            exp = expected(m, sents, p, seed, idx - 2)
            assert [exp[2]] == want
            for device in (False, True):
                same(enc_run(bpe, sents, {}, p, seed, idx - 2, 3, 0, device), exp, sents, (w, idx, p, device))


def check_keys(oracle, small=False):
    """A seed with a high half; sentence indices 2^32 - 3 ... across the high-half carry; words at byte offsets above
    2^16 of a 100 KB sentence; one word 1 000 times in one sentence, every occurrence with its own draws."""
    m = _zipf_model(oracle)
    bpe = SG._bpe(m)
    zc = _cases.zipf()
    seed = 0xDEADBEEF_00000007
    sents = zc.sentences(8, 80, seed=41)
    for p in (0.1, 0.5):
        want = expected(m, sents, p, seed, 2**32 - 3)
        assert want != expected(m, sents, p, seed & 0xFFFFFFFF, 2**32 - 3)       # the seed's high half matters
        for device in (False, True):
            same(enc_run(bpe, sents, {}, p, seed, 2**32 - 3, device=device), want, sents, ("carry", p, device))
    # words above 2^16: a filler of long words without rules keeps the number of words small
    filler = b" ".join([b"\xe4\xb8\x80" * 300] * (80 if small else 110))                  # 110 words of 900 bytes
    tail = b" ".join(zc.sentences(10 if small else 60, 80, seed=43))
    big = [filler + b" " + tail, tail]
    assert len(big[0]) - len(tail) > 2**16
    want = expected(m, big, 0.3, 5, 9)
    assert want[0][-len(want[1]):] != want[1]                       # the offset is part of the key
    for device in (False, True):
        same(enc_run(bpe, big, {}, 0.3, 5, 9, device=device), want, big, ("offsets", device))
    # one word repeated: every occurrence draws for itself
    word = b"internationalization"
    rep = [b" ".join([word] * (200 if small else 1000))]
    words = DR.replay_batch(REF, m, rep, 0.25, 6, 0)[0]
    assert len({tuple(w["ids"]) for w in words}) > 3
    for device in (False, True):
        same(enc_run(bpe, rep, {}, 0.25, 6, 0, device=device), flags([words], m, {}), rep, ("repeat", device))


def check_space_id_zero(oracle):
    """U+2581 at id 0 (no special token at 0): the word-initial "▁" that is never merged is dropped, with dropout."""
    text = _cases.zipf().text(60_000) + b" zab zab ab z zz z q"
    vocab = len(set(text.decode().replace("\n", " ").replace(" ", ""))) + 5 + 25
    for special in (dict(pad=-1, unk=1, bos=2, eos=3), dict(pad=-1, unk=5, bos=-1, eos=-1)):
        m = _model(oracle, text, vocab, **special)
        assert read_model(m)[0][0x2581] == 0
        bpe = SG._bpe(m)
        sents = _cases.zipf_sentences(30) + list(_cases.EDGE_SENTENCES) + [b"zab", b"z", b"q z zz", "▁▁z".encode()]
        for p in (0.1, 0.5, 1.0):
            kw = dict(bos=True, reverse=True) if special["bos"] != -1 else dict(reverse=True)
            want = expected(m, sents, p, 4, 0, kw)
            for device in (False, True):
                same(enc_run(bpe, sents, kw, p, 4, 0, 7, 3, device), want, sents, (special, p, device))


def check_chunks(oracle, monkeypatch, n_mb=3):
    """YTTM_ENC_CHUNK_MB=1: the host pipeline cuts the batch into chunks, each with its own first sentence index."""
    monkeypatch.setenv("YTTM_ENC_CHUNK_MB", "1")
    m = _zipf_model(oracle)
    bpe = SG._bpe(m)
    zc = _cases.zipf()
    real = zc.sentences(3 * n_mb * 16, 100, seed=47)
    sents = []
    for i, s in enumerate(real):                    # blank fillers carry the batch over the chunk edges, wordless
        sents += [s, b" " * 40000 if i % 3 != 2 else b"\t"]
    assert len(_pack(sents)[0]) > n_mb * (1 << 20)
    bpe.dropout_seed(21)
    want = expected(m, sents, 0.2, 21, 0)
    data, offs = _pack(sents)
    ids, oo = bpe.encode_packed(data, offs, dropout_prob=0.2)
    L = _lib.lib()
    assert L.yttm_stage_ms(L.yttm_api_device_context(bpe._h), b"enc_chunks") >= n_mb
    oo = oo.astype(np.int64)
    same([ids[oo[i]:oo[i + 1]].tolist() for i in range(len(sents))], want, sents, "chunks")


def _lists(ids, oo):
    ids, oo = PG._np(ids), PG._np(oo).astype(np.int64)
    return [ids[oo[i]:oo[i + 1]].tolist() for i in range(len(oo) - 1)]


def _pieces(text, po, so):
    text, po, so = bytes(PG._np(text)), PG._np(po).astype(np.int64), PG._np(so).astype(np.int64)
    pieces = [text[po[k]:po[k + 1]].decode() for k in range(len(po) - 1)]
    return [pieces[so[i]:so[i + 1]] for i in range(len(so) - 1)]


def check_api_counter(oracle, small=False):
    """The BPE handle's sentence counter: encode_packed, encode_padded (both widths) and encode_subwords_packed each
    take the next sentence indices; a call without dropout takes none; dropout_seed starts again at 0.  Spans are the
    restatement's, padded rows the definition over the replayed ids, pieces the reference's own."""
    m = _zipf_model(oracle)
    bpe, model = SG._bpe(m), SG.Model(m)
    _, pad, bos_id, eos_id = read_model(m)[2]
    zc = _cases.zipf()
    A = zc.sentences(20 if small else 200, 80, seed=51) + _cases.EDGE_SENTENCES
    B = zc.sentences(15 if small else 150, 60, seed=52) + _word_shapes(np.random.default_rng(4))[:12]
    Cs = zc.sentences(10 if small else 100, 60, seed=53) + _cases.EDGE_SENTENCES
    seed, p = 0x1234_5678_9ABC, 0.3
    dA, oA = _pack(A)
    dB, oB = _pack(B)
    dC, oC = _pack(Cs)
    bpe.dropout_seed(seed)
    kw = dict(bos=True, eos=True, reverse=True)
    ids, oo, spans = bpe.encode_packed(dA, oA, dropout_prob=p, with_spans=True, **kw)
    want = expected(m, A, p, seed, 0, kw)
    same(_lists(ids, oo), want, A, "packed")
    oo = oo.astype(np.int64)
    for s in range(len(A)):
        got = [tuple(x) for x in spans[oo[s]:oo[s + 1]].tolist()]
        assert got == SG.oracle_spans(model, A[s], want[s], int(oA[s]), True, True, True), s
    bpe.encode_packed(dA, oA)                                                          # no draws: no indices
    c = DR.replay_batch(REF, m, B, p, seed, len(A))
    plain = flags(c, m, {})
    for L in (None, 9):
        rows, lens = PG.call_padded(bpe, dB, oB, L, dict(dropout_prob=p, bos=True, eos=True), False, _on_gpu())
        wr, wl = PG.rows_from_lists(plain, L, bos_id, eos_id, pad, True, True, False)
        first = len(A) + (len(B) if L == 9 else 0)
        if L == 9:
            plain9 = flags(DR.replay_batch(REF, m, B, p, seed, first), m, {})
            wr, wl = PG.rows_from_lists(plain9, L, bos_id, eos_id, pad, True, True, False)
        assert np.array_equal(PG._np(lens), wl) and np.array_equal(PG._np(rows), wr), L
    _, want_pieces = expected(m, Cs, p, seed, len(A) + 2 * len(B), dict(eos=True), subwords=True)
    assert _pieces(*bpe.encode_subwords_packed(dC, oC, eos=True, dropout_prob=p)) == want_pieces
    bpe.dropout_seed(seed + 1)
    same(_lists(*bpe.encode_packed(dC, oC, dropout_prob=p)), expected(m, Cs, p, seed + 1, 0), Cs, "reseeded")


def check_threads(oracle, small=False):
    """Two threads on one handle: the calls take disjoint index ranges, in either order."""
    m = _zipf_model(oracle)
    bpe = SG._bpe(m)
    zc = _cases.zipf()
    n = 30 if small else 300
    batches = [zc.sentences(n, 70, seed=61), zc.sentences(n, 70, seed=62)]
    p, seed = 0.2, 77
    want = [[expected(m, b, p, seed, first) for first in (0, n)] for b in batches]
    bpe.dropout_seed(seed)
    got = [None, None]

    def run(i):
        d, o = _pack(batches[i])
        got[i] = _lists(*bpe.encode_packed(d, o, dropout_prob=p))
    th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert (got[0] == want[0][0] and got[1] == want[1][1]) or (got[0] == want[0][1] and got[1] == want[1][0])


# ---- the GPU tests -------------------------------------------------------------------------------------------------

def test_packed_ids(product, oracle):
    check_packed(oracle)


def test_skip_boundary(product, oracle):
    check_boundary(oracle)


def test_keys(product, oracle):
    check_keys(oracle)


def test_space_id_zero(product, oracle):
    check_space_id_zero(oracle)


def test_chunk_pipeline(product, oracle, monkeypatch):
    check_chunks(oracle, monkeypatch)


def test_api_counter_spans_padded_subwords(product, oracle):
    check_api_counter(oracle)


def test_two_threads_one_handle(product, oracle):
    check_threads(oracle)

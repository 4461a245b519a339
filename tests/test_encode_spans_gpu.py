"""Source spans (`BPE.encode_packed(with_spans=True)`, yttm_enc_run_spans*) and subword pieces
(`BPE.encode_subwords_packed`, yttm_enc_run_subwords*) on the GPU.  Spans are checked against a pure-Python restatement
that derives them from the ids, the model file and the reference's UTF-8 rules (nothing is read from the library's
tables); pieces against the host `encode(output_type=SUBWORD)` (the raw bytes of yttm_api_encode_subwords).  The bodies
take `dev`: True also runs the CUDA-tensor interfaces; tests/test_encode_spans_emul_cpu.py runs them with False under
the SIMT emulator."""
import ctypes as C
import os

import numpy as np
import pytest

import _cases
from _bind import _pack, read_model, tmp_model_path
from youtokentome_b200 import _lib, synth

pytestmark = pytest.mark.gpu

SPACE_CP = 0x2581
KWS = [dict(bos=b, eos=e, reverse=r) for b in (False, True) for e in (False, True) for r in (False, True)]

# invalid UTF-8 at word starts, word ends and inside merged tokens, a literal U+2581, words of invalid bytes only
ADVERSARIAL = [
    b"\xc0\xaf", b"ab\xc0\xafab", b"\xc0\xafabab", b"abab\xc0\xaf", b"a\xed\xa0\x80b ab\xed\xbf\xbfab",
    b"\xf0\x9f\x98 ab\xf0\x9f\x98", b"ab\xe2\x96", b"\x80ab \x80\x80ab\xbf a\x80b\x80", b"\xff\xfe \xfe\xff\xc1\x81",
    b"ab\xe2\x96\x81ab", b"\xe2\x96\x81", b"\xe2\x96\x81\xe2\x96\x81ab\xe2\x96\x81 ", b"\xe0\x80\xaf ab\xf8\x88\x80\x80\x80",
    b"\xf4\x90\x80\x80ab \xf0\x80\x80\x80", b"a\xc3b \xc3\xa9\xc3", "éé ёё 日本\xff語".encode(), b"\xbf\xbf\xbf ab \xc0",
    b"ab" + b"\x80" * 50 + b"ab", "ab☃\x80☃ab ☃☃".encode(),
]


# ---- the restatement ----------------------------------------------------------------------------------------------
def _decode_unit(s, p):
    """(code point or None, length) of the unit at s[p] (utf8.cpp:37-74: overlongs, surrogates and truncated sequences
    are one invalid byte)."""
    b0 = s[p]
    if b0 < 0x80:
        return b0, 1
    n = 2 if b0 & 0xE0 == 0xC0 else 3 if b0 & 0xF0 == 0xE0 else 4 if b0 & 0xF8 == 0xF0 else 0
    if n == 0 or p + n > len(s) or any(c & 0xC0 != 0x80 for c in s[p + 1:p + n]):
        return None, 1
    cp = b0 & (0x7F >> n)
    for c in s[p + 1:p + n]:
        cp = (cp << 6) | (c & 0x3F)
    if cp < (0x80, 0x800, 0x10000)[n - 2] or 0xD800 <= cp <= 0xDFFF or cp >= 0x110000:
        return None, 1
    return cp, n


def _is_space(cp):
    return cp is not None and (cp == 32 or 9 <= cp <= 13 or cp == SPACE_CP)


def _words(s):
    """Words of a sentence: lists of (start, end, code point or None) units between space units."""
    words, cur, p = [], [], 0
    while p < len(s):
        cp, n = _decode_unit(s, p)
        if _is_space(cp):
            if cur:
                words.append(cur)
            cur = []
        else:
            cur.append((p, p + n, cp))
        p += n
    if cur:
        words.append(cur)
    return words


class Model:
    """What the restatement needs from a model file: unit count and piece of every ordinary id, the alphabet, the
    special ids."""

    def __init__(self, path):
        c2i, rules, (self.unk, self.pad, self.bos, self.eos) = read_model(path)
        self.alphabet = set(c2i)
        recipe = {i: [cp] for cp, i in c2i.items()}
        for x, y, z in rules:
            recipe[z] = recipe[x] + recipe[y]
        self.units = {i: len(r) - (r[0] == SPACE_CP) for i, r in recipe.items()}
        self.text = {i: "".join(map(chr, r[1:] if r[0] == SPACE_CP else r)).encode() for i, r in recipe.items()}


def oracle_spans(model, sent, ids, base, bos, eos, reverse):
    """Spans of one sentence's ids (offsets coordinates: the sentence starts at `base`)."""
    ids = list(ids)[::-1] if reverse else list(ids)
    inner = ids[1 if bos else 0:len(ids) - (1 if eos else 0)]
    out, k = [], 0
    for w in _words(sent):
        valid = [u for u in w if u[2] is not None]
        pos = 0
        while pos < len(valid):
            i = inner[k]
            k += 1
            if i == model.unk:
                j = pos
                while j < len(valid) and valid[j][2] not in model.alphabet:
                    j += 1
                assert j > pos, "<UNK> at an in-alphabet unit"
            else:
                j = pos + model.units[i]
            out.append((valid[pos][0], valid[j - 1][1]) if j > pos else (valid[pos][0],) * 2)
            pos = j
    assert k == len(inner), "ids left after the last word"
    out = [(a + base, b + base) for a, b in out]
    if bos:
        out.insert(0, (base, base))
    if eos:
        out.append((base + len(sent),) * 2)
    return out[::-1] if reverse else out


def _valid_bytes(s):
    out, p = b"", 0
    while p < len(s):
        cp, n = _decode_unit(s, p)
        if cp is not None:
            out += s[p:p + n]
        p += n
    return out


def check_properties(model, data, offs, ids, oo, spans, reverse):
    for s in range(len(offs) - 1):
        sp = [tuple(x) for x in spans[oo[s]:oo[s + 1]].tolist()]
        seq = sp[::-1] if reverse else sp
        for (a0, b0), (a1, b1) in zip(seq, seq[1:]):
            assert a0 <= b0 <= a1 <= b1
        for (a, b), i in zip(sp, ids[oo[s]:oo[s + 1]].tolist()):
            assert offs[s] <= a <= b <= offs[s + 1]
            piece = _valid_bytes(data[a:b])
            if i == model.unk:
                assert piece and not set(piece.decode()) & {chr(c) for c in model.alphabet}
            elif i in (model.bos, model.eos):
                assert a == b
            else:
                assert piece == model.text[i]


# ---- library calls -------------------------------------------------------------------------------------------------
def _bpe(m):
    import youtokentome_b200 as yttm
    return yttm.BPE(m)


def host_subwords(bpe, data, offs, kw):
    """encode(output_type=SUBWORD) flattened: (piece bytes, piece offsets, sentence offsets) from the host path."""
    L = _lib.lib()
    n = len(offs) - 1
    need = L.yttm_api_encode_subwords(bpe._h, data, offs.ctypes.data, n, int(kw.get("bos", False)),
                                      int(kw.get("eos", False)), int(kw.get("reverse", False)),
                                      float(kw.get("dropout_prob", 0.0)))
    assert need >= 0, L.yttm_api_last_error(bpe._h)
    n_p, n_s = C.c_uint64(0), C.c_uint64(0)
    L.yttm_api_result_counts(bpe._h, C.byref(n_p), C.byref(n_s))
    buf = C.create_string_buffer(int(need) + 1)
    L.yttm_api_result_text(bpe._h, buf)
    po = np.zeros(n_p.value + 1, dtype=np.uint64)
    so = np.zeros(n_s.value + 1, dtype=np.uint64)
    L.yttm_api_result_offsets(bpe._h, po.ctypes.data, so.ctypes.data)
    return buf.raw[:need], po, so


def _np(x):
    if type(x).__module__.startswith("torch"):
        x = x.cpu().numpy()
        return x if x.dtype == np.uint8 else x.astype(np.uint64)
    return x


def check_batch(bpe, model, data, offs, kw, dev=False, seed=None):
    """ids with spans == encode_packed's; spans == the restatement; the properties; subword pieces == the host path;
    with dev the CUDA interfaces give the same."""
    def fresh():
        if seed is not None:
            bpe.dropout_seed(seed)
    offs = np.asarray(offs, dtype=np.uint64)
    rev = kw.get("reverse", False)
    fresh()
    ids0, oo0 = bpe.encode_packed(data, offs, **kw)
    fresh()
    ids, oo, spans = bpe.encode_packed(data, offs, with_spans=True, **kw)
    assert ids.dtype == np.int32 and oo.dtype == np.uint64 and spans.dtype == np.uint64 and spans.shape == (len(ids), 2)
    assert np.array_equal(ids, ids0) and np.array_equal(oo, oo0)
    raw = bytes(data)
    for s in range(len(offs) - 1):
        a, b = int(offs[s]), int(offs[s + 1])
        want = oracle_spans(model, raw[a:b], ids[oo[s]:oo[s + 1]], a, kw.get("bos", False), kw.get("eos", False), rev)
        got = [tuple(x) for x in spans[oo[s]:oo[s + 1]].tolist()]
        assert got == want, (s, raw[a:b], ids[oo[s]:oo[s + 1]].tolist())
    check_properties(model, raw, offs, ids, oo, spans, rev)
    fresh()
    h_text, h_po, h_so = host_subwords(bpe, raw, offs, kw)
    fresh()
    text, po, so = bpe.encode_subwords_packed(data, offs, **kw)
    assert text.dtype == np.uint8 and po.dtype == np.uint64 and so.dtype == np.uint64
    assert bytes(text) == h_text and np.array_equal(po, h_po) and np.array_equal(so, h_so)
    assert np.array_equal(so, oo)   # one piece per id
    results = [(ids, oo, spans, text, po, so)]
    outs = ["torch"] + (["cuda"] if dev else [])
    for out in outs:
        fresh()
        r = bpe.encode_packed(data, offs, with_spans=True, out=out, **kw)
        fresh()
        r += bpe.encode_subwords_packed(data, offs, out=out, **kw)
        import torch
        assert all(isinstance(t, torch.Tensor) and t.is_cuda == (out == "cuda") for t in r)
        assert r[2].dtype == r[1].dtype == torch.int64 and r[4].dtype == r[5].dtype == torch.int64
        results.append(tuple(_np(t) for t in r))
    if dev:   # CUDA input: the results stay on the device
        import torch
        d_data = torch.tensor(list(raw), dtype=torch.uint8).cuda()
        d_offs = torch.from_numpy(offs.astype(np.int64)).cuda()
        fresh()
        r = bpe.encode_packed(d_data, d_offs, with_spans=True, out="cuda", **kw)
        fresh()
        r += bpe.encode_subwords_packed(d_data, d_offs, out="cuda", **kw)
        assert all(t.is_cuda for t in r)
        results.append(tuple(_np(t) for t in r))
    for other in results[1:]:
        for x, y in zip(results[0], other):
            assert np.array_equal(np.asarray(x), np.asarray(y).reshape(np.asarray(x).shape))


def check_sentences(oracle, model_path, sents, kws=KWS, dev=False, shift=0):
    bpe, model = _bpe(model_path), Model(model_path)
    data, offs = _pack(sents)
    if shift:   # offsets[0] > 0: bytes in front of and behind the batch are not read
        data = b"\xe2\x96" * shift + data + b"\xff" * shift
        offs = offs + np.uint64(2 * shift)
    for kw in kws:
        if (kw.get("bos") and model.bos == -1) or (kw.get("eos") and model.eos == -1):
            continue
        check_batch(bpe, model, data, offs, kw, dev)
    return bpe, model


def _model(oracle, text, vocab, cov=1.0, **special):
    m = tmp_model_path("orc")
    oracle.train(text, m, vocab, cov, **special)
    return m


# ---- bodies shared with the emulator test --------------------------------------------------------------------------
def check_stress(oracle, seed, dev=False):
    text, vocab, cov, sents = _cases.stress_case(seed)
    try:
        m = _model(oracle, text, vocab, cov)
    except ValueError:
        return
    check_sentences(oracle, m, sents + _cases.EDGE_SENTENCES, dev=dev)


def check_golden_texts(oracle, dev=False):
    for name in sorted(synth.GOLDEN_TEXTS):
        train, test, vocab = synth.GOLDEN_TEXTS[name]
        m = _model(oracle, train.encode(), vocab)
        check_sentences(oracle, m, [test.encode()] + test.encode().split(b"\n"), KWS[:2] + KWS[-1:], dev=dev)


def check_dirty_zipf(oracle, cov, n_sents, dev=False):
    m = _model(oracle, _cases.dirty_zipf_text(60_000), 700, cov)
    check_sentences(oracle, m, _cases.zipf_sentences(n_sents) + _cases.EDGE_SENTENCES + ADVERSARIAL, dev=dev)


def check_adversarial(oracle, dev=False):
    text = _cases.dirty_zipf_text(60_000) + b" ab ab abab ba " * 50 + " ☃☃ éé ёё".encode() * 30
    m = _model(oracle, text, 900, 0.97)
    check_sentences(oracle, m, ADVERSARIAL + _cases.EDGE_SENTENCES + [b" ".join(ADVERSARIAL)], dev=dev)


def check_space_id_zero(oracle, special, dev=False):
    """"▁" with id 0: an unmerged word-initial "▁" leaves the output and has no span."""
    text = _cases.zipf().text(60_000) + b" zab zab ab z zz z q"
    n_chars = len(set(text.decode().replace("\n", " ").replace(" ", "")))
    m = _model(oracle, text, n_chars + 5 + 25, 1.0, **special)
    long_word = b"".join(_cases.zipf().sentences(12, 60, seed=6)).replace(b" ", b"")
    sents = _cases.zipf_sentences(100) + list(_cases.EDGE_SENTENCES) + [b"zab", b"z", b"q z zz", long_word,
                                                                          b"q" + long_word] + ADVERSARIAL
    assert Model(m).units[0] == 0
    check_sentences(oracle, m, sents, KWS[:2] + ([KWS[-1]] if special["bos"] != -1 else []), dev=dev)


def check_long_words(oracle, dev=False):
    """Words longer than the thread-local arrays (40 slots), than LONG_W (512 slots, the block kernel) and a 30 KB
    sentence."""
    m = _model(oracle, _cases.dirty_zipf_text(60_000), 900, 0.95)
    zc = _cases.zipf()
    long_sent = b" ".join(zc.sentences(300, 100, seed=5))
    long_word = b"".join(zc.sentences(40, 60, seed=6)).replace(b" ", b"")
    mid_word = long_word[:300]
    sents = [long_sent, long_word, mid_word, b"a" * 3000, long_word + b"\xff" + mid_word + b" " + long_sent,
             b"x" + long_word[:45], b"", long_word]
    check_sentences(oracle, m, sents, KWS[:2], dev=dev)


def check_layouts(oracle, dev=False):
    """Empty and all-space sentences and batches, offsets[0] > 0, several chunks of the host-buffer entry points."""
    m = _model(oracle, _cases.dirty_zipf_text(60_000), 900)
    check_sentences(oracle, m, [b"", b" ", b"\t\n  ", b"\xe2\x96\x81 \xe2\x96\x81"], dev=dev)
    check_sentences(oracle, m, [], KWS[:1], dev=dev)
    check_sentences(oracle, m, [b""] * 5, KWS[:2], dev=dev)
    check_sentences(oracle, m, _cases.zipf_sentences(50) + ADVERSARIAL, KWS[::3], dev=dev, shift=37)


def check_chunks(oracle, monkeypatch, n_bytes, dev=False):
    m = _model(oracle, _cases.dirty_zipf_text(60_000), 900, 0.95)
    monkeypatch.setenv("YTTM_ENC_CHUNK_MB", "1")
    sents = _cases.zipf().sentences(n_bytes // 100, 100, seed=11) + ADVERSARIAL
    bpe, _ = check_sentences(oracle, m, sents, [dict(), dict(bos=True, eos=True, reverse=True)], dev=dev)
    L = _lib.lib()
    assert L.yttm_stage_ms(L.yttm_api_device_context(bpe._h), b"enc_chunks") >= 2


def check_dropout(oracle, p, dev=False):
    m = _model(oracle, _cases.dirty_zipf_text(60_000), 900, 0.95)
    bpe, model = _bpe(m), Model(m)
    sents = _cases.zipf_sentences(150) + _cases.EDGE_SENTENCES + ADVERSARIAL
    data, offs = _pack(sents)
    for kw in (dict(), dict(bos=True, eos=True, reverse=True)):
        check_batch(bpe, model, data, offs, dict(kw, dropout_prob=p), dev, seed=77)
    # the new calls advance the same sentence counter as encode_packed
    bpe.dropout_seed(5)
    a = [bpe.encode_packed(data, offs, dropout_prob=p)[0] for _ in range(2)]
    bpe.dropout_seed(5)
    b = [bpe.encode_packed(data, offs, dropout_prob=p, with_spans=True)[0], bpe.encode_subwords_packed(data, offs,
                                                                                                       dropout_prob=p)]
    assert np.array_equal(a[0], b[0])
    bpe.dropout_seed(5)
    bpe.encode_packed(data, offs, dropout_prob=p)
    h = host_subwords(bpe, data, offs, dict(dropout_prob=p))
    assert bytes(b[1][0]) == h[0] and np.array_equal(b[1][1], h[1])


def check_errors(oracle, dev=False):
    m = tmp_model_path("orc")
    oracle.train(synth.readme_corpus(n_lines=200), m, 100, 1.0, pad=-1, unk=0, bos=-1, eos=-1)
    bpe = _bpe(m)
    data, offs = _pack([b"ab"])
    outs = ["numpy"] + (["cuda"] if dev else [])
    for out in outs:
        for call in (lambda **k: bpe.encode_packed(data, offs, with_spans=True, out=out, **k),
                     lambda **k: bpe.encode_subwords_packed(data, offs, out=out, **k)):
            with pytest.raises(ValueError, match="Can't add <BOS> token. Model was trained without it."):
                call(bos=True)
            with pytest.raises(ValueError, match="Can't add <EOS> token. Model was trained without it."):
                call(eos=True)
            for p in (-0.1, 1.5):
                with pytest.raises(ValueError, match="dropout_prob value must be in the range"):
                    call(dropout_prob=p)
    for call in (lambda: bpe.encode_packed(data, offs, with_spans=True, out="list"),
                 lambda: bpe.encode_subwords_packed(data, offs, out="list")):
        with pytest.raises(ValueError, match="out must be"):
            call()


def check_abi_capacity(oracle, dev=False):
    """The host-buffer C entry points return 2 with the sizes needed, then the same results as the Python surface."""
    m = _model(oracle, _cases.dirty_zipf_text(60_000), 900, 0.95)
    bpe = _bpe(m)
    L = _lib.lib()
    enc = L.yttm_api_device_encoder(bpe._h)
    sents = _cases.zipf_sentences(40) + ADVERSARIAL
    data, offs = _pack(sents)
    n = len(sents)
    ids, oo, spans = bpe.encode_packed(data, offs, with_spans=True, bos=True, eos=True)
    text, po, so = bpe.encode_subwords_packed(data, offs, bos=True, eos=True)
    tot = C.c_uint64(0)
    small_ids, small_oo, small_sp = np.zeros(4, np.int32), np.zeros(n + 1, np.uint64), np.zeros(8, np.uint64)
    assert L.yttm_enc_run_spans(enc, data, offs.ctypes.data, n, 1, 1, 0, 0.0, 0, 0, small_ids.ctypes.data, 4,
                                small_oo.ctypes.data, small_sp.ctypes.data, C.byref(tot)) == 2
    assert tot.value == len(ids)
    k = tot.value
    i2, o2, s2 = np.zeros(k, np.int32), np.zeros(n + 1, np.uint64), np.zeros((k, 2), np.uint64)
    assert L.yttm_enc_run_spans(enc, data, offs.ctypes.data, n, 1, 1, 0, 0.0, 0, 0, i2.ctypes.data, k, o2.ctypes.data,
                                s2.ctypes.data, C.byref(tot)) == 0
    assert np.array_equal(i2, ids) and np.array_equal(o2, oo) and np.array_equal(s2, spans)
    n_p, n_b = C.c_uint64(0), C.c_uint64(0)
    for pcap, bcap in ((len(po) - 1, 3), (2, len(text)), (len(po) - 1, len(text))):
        t3, p3, q3 = np.zeros(max(bcap, 1), np.uint8), np.zeros(pcap + 1, np.uint64), np.zeros(n + 1, np.uint64)
        rc = L.yttm_enc_run_subwords(enc, data, offs.ctypes.data, n, 1, 1, 0, 0.0, 0, 0, t3.ctypes.data, bcap,
                                     p3.ctypes.data, pcap, q3.ctypes.data, C.byref(n_p), C.byref(n_b))
        assert n_p.value == len(po) - 1 and n_b.value == len(text)
        if bcap < len(text) or pcap < len(po) - 1:
            assert rc == 2
        else:
            assert rc == 0 and bytes(t3) == bytes(text) and np.array_equal(p3, po) and np.array_equal(q3, so)
    assert L.yttm_enc_run_spans(None, data, offs.ctypes.data, n, 0, 0, 0, 0.0, 0, 0, None, 0, None, None,
                                C.byref(tot)) == 1
    assert b"null encoder handle" in L.yttm_last_error(None)


# ---- GPU tests -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_spans_stress(product, oracle, seed):
    check_stress(oracle, seed, dev=True)


def test_spans_golden_texts(product, oracle):
    check_golden_texts(oracle, dev=True)


@pytest.mark.parametrize("cov", [1.0, 0.95, 0.9])
def test_spans_dirty_zipf(product, oracle, cov):
    check_dirty_zipf(oracle, cov, 600, dev=True)


def test_spans_adversarial_utf8(product, oracle):
    check_adversarial(oracle, dev=True)


@pytest.mark.parametrize("special", [dict(pad=-1, unk=1, bos=2, eos=3), dict(pad=-1, unk=5, bos=-1, eos=-1)])
def test_spans_space_id_zero(product, oracle, special):
    check_space_id_zero(oracle, special, dev=True)


def test_spans_long_words(product, oracle):
    check_long_words(oracle, dev=True)


def test_spans_layouts(product, oracle):
    check_layouts(oracle, dev=True)


def test_spans_chunks(product, oracle, monkeypatch):
    check_chunks(oracle, monkeypatch, 3_000_000, dev=True)


@pytest.mark.parametrize("p", [0.1, 1.0])
def test_spans_dropout(product, oracle, p):
    check_dropout(oracle, p, dev=True)


def test_spans_errors(product, oracle):
    check_errors(oracle, dev=True)


def test_spans_abi_capacity(product, oracle):
    check_abi_capacity(oracle, dev=True)


def test_zzz_sanitizer_memcheck_spans(product):
    """compute-sanitizer memcheck over tools/sanitize_spans.py: no report; skips where the tool refuses the device."""
    import shutil
    import subprocess
    import sys
    from _bind import ROOT
    exe = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(exe):
        pytest.skip("compute-sanitizer is not installed")
    env = {k: v for k, v in os.environ.items() if not k.startswith(("YTTM_", "YT_EMU_"))}
    r = subprocess.run([exe, "--tool", "memcheck", sys.executable, os.path.join(ROOT, "tools", "sanitize_spans.py")],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    text = r.stdout.decode(errors="replace")
    if "Error: Device not supported" in text:
        pytest.skip("compute-sanitizer does not support this device here")
    assert "spans and subwords identical to the host paths" in text, text[-1500:]
    assert "ERROR SUMMARY: 0 errors" in text, text[-1500:]

"""The front of device encode on the SIMT emulator: the word finder (sentences staged group by group in shared-memory
pieces of 16 KB) and the word dedup (16-byte vector loads and shifts instead of byte-serial gathers).  Every case
compares the ids with the oracle for every keyword set of test_encode_gpu.KW, and with dropout where it applies.

TEST HARNESS ONLY, like tests/test_simt_emul_cpu.py."""
import ctypes as C
import mmap

import numpy as np
import pytest

import _bind
import _cases
import test_encode_gpu as EG
from youtokentome_b200 import _lib

SP = b"\xe2\x96\x81"   # U+2581
PIECE = 16384          # bytes of a staged piece of the word finder
_models = {}


@pytest.fixture
def emu(monkeypatch):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", "2")
    return L


def _model(oracle, name):
    if name not in _models:
        if name == "zipf":
            _models[name] = EG._model(oracle, _cases.dirty_zipf_text(), 1500)
        else:   # few rules: a 40 KB word is merged in few passes
            _models[name] = EG._model(oracle, b"abcd abca bcd " * 200 + b"ab" * 300, 40)
    return _models[name]


def _same(oracle, m, sents, dropout=True):
    g, o = EG.GpuEncoder(m), oracle.encoder(m)
    for kw in EG.KW:
        assert g.encode(sents, **kw) == o.encode(sents, **kw), kw
    if dropout:
        assert g.encode(sents, dropout=0.3, seed=9) == o.encode(sents, dropout=0.3, seed=9)


def _zipf_text(n, seed):
    t = b" ".join(_cases.zipf().sentences(n // 30 + 2, 60, seed=seed))[:n]
    assert len(t) == n
    return t


@pytest.mark.parametrize("sms", ["1", "2", "5"])
def test_groups_longer_than_a_piece(emu, oracle, monkeypatch, sms):
    """Groups streamed piece by piece (count, reserve, write): sentences of 40 KB and 200 KB, a 40 KB one without spaces,
    a group of many 1 - 3 KB sentences, and sentence bounds / U+2581 at every offset mod 16 around a piece edge."""
    monkeypatch.setenv("YT_EMU_SMS", sms)
    m = _model(oracle, "zipf")
    _same(oracle, m, [_zipf_text(40_000, 1)])
    _same(oracle, m, [b"a", _zipf_text(200_000, 2), b"b c"], dropout=False)
    rng = np.random.default_rng(int(sms))
    many = [_zipf_text(int(k), 10 + i) for i, k in enumerate(rng.integers(1000, 3000, 40))]
    _same(oracle, m, _cases.zipf_sentences(400) + many + _cases.zipf_sentences(50, seed=4))
    # without spaces the sentence is one word for the block-per-word merge kernel: 40 KB keeps the emulator in seconds
    m2 = _model(oracle, "abcd")
    word = bytes(rng.choice(list(b"abcd"), size=40_000).tolist())
    _same(oracle, m2, [word], dropout=False)
    _same(oracle, m2, [b"ab", word[:20_000] + b" " + word[:9] + SP + word[:PIECE + 5]], dropout=False)
    # the first group starts at batch byte 0 (aligned): its piece edge is batch byte 16384
    for d in range(-18, 19):
        s1 = _zipf_text(PIECE + d - 12, 20 + d) + b"a " + SP + b"cd " + b"q" * 3
        s2 = SP + b"ab cd" + SP
        s3 = b"\x81x y\xe2\x96"
        tail = [b"w%d x" % k for k in range(20)]
        _same(oracle, m, [s1, s2, s3, b"", b"", b"\x96\x81z"] + tail, dropout=(d % 6 == 0))


def test_group_sizes_and_empty_sentences(emu, oracle):
    """Batches where the group size G does not divide the number of sentences, runs of empty sentences inside groups,
    at the start and at the end, and a batch of empty sentences only."""
    m = _model(oracle, "zipf")
    base = _cases.zipf_sentences(600, target=128)
    G = PIECE * 3 // 4 // (sum(map(len, base)) // len(base))
    for n in (G * 3 - 1, G * 3 + 1, G - 1, G + 1, 1):
        _same(oracle, m, base[:n], dropout=(n == G * 3 - 1))
    holes = []
    for i, s in enumerate(base[:300]):
        holes += [b""] * (i % 7 == 3) * (1 + i % 5) + [s]
    _same(oracle, m, [b""] * 9 + holes + [b""] * 150)
    _same(oracle, m, [b""] * 500)
    _same(oracle, m, [b""] * 3 + [b" "] + [b""] * 3)


def test_misaligned_base_ending_at_the_allocation(emu, oracle):
    """yttm_enc_run_device on a batch at base address shifts 1 .. 15 whose last sentence ends exactly at the last byte
    of the mapping: the page after it is protected, so a load past the batch end faults."""
    m = _model(oracle, "zipf")
    g, o = EG.GpuEncoder(m), oracle.encoder(m)
    ctx, enc = emu.yttm_api_device_context(g.h), emu.yttm_api_device_encoder(g.h)
    libc = C.CDLL(None)
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    page = mmap.PAGESIZE
    for shift in range(1, 16):
        sents = _cases.zipf_sentences(60, seed=shift) + [b"x" * 33 + b" " + SP + b"ab" + SP[:2]]
        pad = (-sum(map(len, sents)) - shift) % 16
        sents[-1] = sents[-1] + b"y" * pad + b" abcdefghijklmno" + b"p" * 16   # (+32 bytes keeps the residue)
        buf, offs = _bind._pack(sents)
        size = len(buf)
        n_pages = (size + page - 1) // page + 1
        mm = mmap.mmap(-1, (n_pages + 1) * page)
        anchor = C.c_char.from_buffer(mm)
        addr = C.addressof(anchor)
        assert libc.mprotect(addr + n_pages * page, page, 0) == 0   # PROT_NONE
        base = addr + n_pages * page - size
        assert base % 16 == shift
        C.memmove(base, bytes(buf), size)
        p_ids, p_off, n = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
        rc = emu.yttm_enc_run_device(enc, base, offs.ctypes.data, size, len(sents), 0, 0, 0, 0.0, 0, 0,
                                     C.byref(p_ids), C.byref(p_off), C.byref(n))
        assert rc == 0, emu.yttm_last_error(ctx)
        ids = np.ctypeslib.as_array(C.cast(p_ids, C.POINTER(C.c_int32)), shape=(n.value,)).copy()
        oo = np.ctypeslib.as_array(C.cast(p_off, C.POINTER(C.c_uint64)), shape=(len(sents) + 1,)).copy()
        assert _bind._unpack(ids, oo) == o.encode(sents), shift
        assert libc.mprotect(addr + n_pages * page, page, 3) == 0   # PROT_READ | PROT_WRITE
        del anchor
        mm.close()


def _word(rng, n):
    parts = [b"a", b"b", b"c", b"d", "ж".encode(), "☃".encode(), b"\xff"]
    w = b"".join(parts[i] for i in rng.integers(0, len(parts), n))
    return w[:n]


@pytest.mark.parametrize("weak", [False, True])
def test_dedup_vector_compare(emu, oracle, monkeypatch, weak):
    """Words of 1 .. 70 bytes that repeat at every alignment mod 16 relative to their representative, pairs that
    differ only in the byte after a 16- or 32-byte boundary, and prefix pairs that end at the sentence end, before a
    space or before U+2581; with equal tags (every probe ends in the byte compare) too."""
    if weak:
        monkeypatch.setenv("YTTM_ENC_DEDUP_WEAKTAG", "1")
    m = _model(oracle, "zipf")
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
    _same(oracle, m, sents)
    _same(oracle, m, sents[::-1] + sents, dropout=False)

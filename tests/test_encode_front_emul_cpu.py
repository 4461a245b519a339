"""The front of device encode on the SIMT emulator: the word finder (sentences staged group by group in shared-memory
pieces of 16 KB) and the word dedup (16-byte vector loads and shifts instead of byte-serial gathers).  The bodies are those of
tests/test_encode_words_gpu.py (ids against the plain restatement for every keyword set of test_encode_gpu.KW, against
the oracle with dropout), so an edge added there runs here too; the protected page behind a misaligned batch exists only
here.

TEST HARNESS ONLY, like tests/test_simt_emul_cpu.py."""
import ctypes as C
import mmap

import numpy as np
import pytest

import _bind
import _cases
import test_encode_words_gpu as WG
from youtokentome_b200 import _lib

SP = b"\xe2\x96\x81"   # U+2581


@pytest.fixture
def emu(monkeypatch):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)
    monkeypatch.setenv("YT_EMU_SMS", "2")
    monkeypatch.setattr(WG, "_cache", {})   # the shared bodies keep encoders: they belong to the library that made them
    return L


@pytest.mark.parametrize("sms", ["1", "2", "5"])
def test_groups_longer_than_a_piece(emu, oracle, monkeypatch, sms):
    """Groups streamed piece by piece (count, reserve, write): sentences of 40 KB and 200 KB, a 40 KB one without spaces,
    a group of many 1 - 3 KB sentences, and sentence bounds / U+2581 at every offset mod 16 around a piece edge."""
    monkeypatch.setenv("YT_EMU_SMS", sms)
    WG.check_groups_longer_than_a_piece(oracle, int(sms))
    WG.check_piece_edges(oracle, 1)


def test_group_sizes_and_empty_sentences(emu, oracle):
    """Batches where the group size G does not divide the number of sentences, runs of empty sentences inside groups,
    at the start and at the end, and a batch of empty sentences only."""
    WG.check_group_sizes_and_empty_sentences(oracle)


def test_misaligned_base_ending_at_the_allocation(emu, oracle):
    """yttm_enc_run_device on a batch at base address shifts 1 .. 15 whose last sentence ends exactly at the last byte
    of the mapping: the page after it is protected, so a load past the batch end faults."""
    case = WG.zipf_case(oracle)
    g, o = case.g, case.o
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


@pytest.mark.parametrize("weak", [False, True])
def test_dedup_vector_compare(emu, oracle, monkeypatch, weak):
    """Words of 1 .. 70 bytes that repeat at every alignment mod 16 relative to their representative, pairs that
    differ only in the byte after a 16- or 32-byte boundary, and prefix pairs that end at the sentence end, before a
    space or before U+2581; with equal tags (every probe ends in the byte compare) too."""
    WG.check_dedup_vector_compare(oracle, monkeypatch, weak)

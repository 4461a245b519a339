"""The decode kernels (youtokentome_b200/csrc/decode.cu) on the CPU under the SIMT emulator, through the same checks as
tests/test_decode_gpu.py at small sizes and with 1, 2 and 5 emulated SMs (a sentence per warp, several rounds of 32 ids,
grid-stride loops that wrap).  Also, with the real library: without a GPU `decode_packed` fails loudly while the host
`decode` keeps working, and the numpy oracle of the GPU tests agrees with the host decode."""
import numpy as np
import pytest

import _cases
import test_decode_gpu as DG
from _bind import tmp_model_path
from youtokentome_b200 import _lib, synth


@pytest.fixture(params=["1", "2", "5"])
def emu(monkeypatch, request):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)  # what _lib.lib() hands to tests/_gpu.py and to the Python BPE class
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


@pytest.mark.parametrize("seed", [0, 3, 7])
def test_decode_parity_stress(emu, oracle, seed):
    DG.check_parity_stress(oracle, seed)


def test_decode_parity_golden_texts(emu, oracle):
    for name in sorted(synth.GOLDEN_TEXTS):
        train, test, vocab = synth.GOLDEN_TEXTS[name]
        DG.check_parity_corpus(oracle, train.encode(), vocab, 1.0, [test.encode()] + test.encode().split(b"\n"))


@pytest.mark.parametrize("cov", [1.0, 0.9])
def test_decode_parity_dirty_zipf(emu, oracle, cov):
    DG.check_parity_corpus(oracle, _cases.dirty_zipf_text(60_000), 700, cov, _cases.zipf_sentences(80) + _cases.EDGE_SENTENCES)


@pytest.mark.parametrize("special", [dict(pad=-1, unk=1, bos=2, eos=3), dict(pad=3, unk=40, bos=41, eos=1000)])
def test_decode_parity_special_layouts(emu, oracle, special):
    DG.check_parity_corpus(oracle, _cases.dirty_zipf_text(60_000), 1100, 1.0, _cases.zipf_sentences(60) + _cases.EDGE_SENTENCES,
                           special)


def test_decode_ignore_ids(emu, oracle):
    DG.check_ignore_ids(oracle)


def test_decode_synthetic_id_lists(emu, oracle):
    DG.check_synthetic_lists(oracle)


def test_decode_long_pieces(emu, oracle):
    DG.check_long_pieces(oracle)


def test_decode_errors(emu, oracle):
    DG.check_errors(oracle)


def test_decode_interfaces(emu, oracle):
    DG.check_interfaces(oracle)


def test_decode_abi_device_entry_and_launches(emu, oracle):
    DG.check_abi_device(oracle)


def test_decode_without_gpu_fails_loudly(product, oracle):
    if product.yttm_device_count() != 0:
        pytest.skip("a GPU is present")
    import youtokentome_b200 as yttm
    m = tmp_model_path()
    oracle.train(b"ab ab abc abd", m, 14)
    bpe = yttm.BPE(m)
    ids = [[4, 5, 6], [7]]
    with pytest.raises(ValueError, match="no CUDA device"):
        bpe.decode_packed(*DG._flat(ids))
    assert len(bpe.decode(ids)) == 2   # the host decode needs no device


def test_numpy_oracle_matches_host_decode(product, oracle):
    """The oracle of the full-size GPU checks against the host BPE.decode (no device needed)."""
    import youtokentome_b200 as yttm
    for special in (dict(), dict(pad=-1, unk=1, bos=2, eos=3), dict(pad=3, unk=40, bos=41, eos=1000)):
        m = DG._model(oracle, _cases.dirty_zipf_text(60_000), 1100, 0.95, **special)
        bpe = yttm.BPE(m)
        tab = DG.piece_table(bpe, m)
        enc = oracle.encoder(m)
        sents = _cases.zipf_sentences(150) + _cases.EDGE_SENTENCES
        kw = dict(bos=True, eos=True) if special.get("bos", 2) != -1 else dict()
        ids = enc.encode(sents, **kw) + enc.encode(sents[:30], reverse=True) + [[], [1]]
        V = bpe.vocab_size()
        sp = DG.read_model(m)[0][9601]
        rng = np.random.default_rng(3)
        ids += [rng.integers(0, V, size=int(n)).tolist() for n in rng.integers(0, 50, size=30)]
        ids += [[sp, sp] + s for s in ids[:10]]
        flat, offs = DG._flat(ids)
        for ign in ((), (2, 3), (sp,), (sp, 1, -5, V + 3)):
            assert DG._texts(*DG.oracle_decode(tab, flat, offs, ign)) == bpe.decode(ids, ignore_ids=list(ign) or None)

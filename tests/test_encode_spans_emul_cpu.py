"""The span and subword kernels (youtokentome_b200/csrc/encode.cu) on the CPU under the SIMT emulator, through the same
bodies as tests/test_encode_spans_gpu.py at small sizes and with 1, 2 and 5 emulated SMs.  Also, with the real library:
without a GPU the new methods fail loudly while the host paths keep working, and the span restatement of the GPU tests
agrees with the host `encode(output_type=SUBWORD)` on the pieces of <UNK>."""
import numpy as np
import pytest

import _cases
import test_encode_spans_gpu as SG
from _bind import _pack, tmp_model_path
from youtokentome_b200 import _lib


@pytest.fixture(params=["1", "2", "5"])
def emu(monkeypatch, request):
    from _emu import emu_lib
    L = emu_lib()
    monkeypatch.setattr(_lib, "_lib", L)  # what _lib.lib() hands to the Python BPE class
    monkeypatch.setenv("YT_EMU_SMS", request.param)
    return L


@pytest.mark.parametrize("seed", [0, 3])
def test_spans_stress(emu, oracle, seed):
    SG.check_stress(oracle, seed)


def test_spans_golden_texts(emu, oracle):
    SG.check_golden_texts(oracle)


@pytest.mark.parametrize("cov", [1.0, 0.95, 0.9])
def test_spans_dirty_zipf(emu, oracle, cov):
    SG.check_dirty_zipf(oracle, cov, 60)


def test_spans_adversarial_utf8(emu, oracle):
    SG.check_adversarial(oracle)


@pytest.mark.parametrize("special", [dict(pad=-1, unk=1, bos=2, eos=3), dict(pad=-1, unk=5, bos=-1, eos=-1)])
def test_spans_space_id_zero(emu, oracle, special):
    SG.check_space_id_zero(oracle, special)


def test_spans_long_words(emu, oracle):
    SG.check_long_words(oracle)


def test_spans_layouts(emu, oracle):
    SG.check_layouts(oracle)


def test_spans_chunks(emu, oracle, monkeypatch):
    SG.check_chunks(oracle, monkeypatch, 2_200_000)


@pytest.mark.parametrize("p", [0.1, 1.0])
def test_spans_dropout(emu, oracle, p):
    SG.check_dropout(oracle, p)


def test_spans_errors(emu, oracle):
    SG.check_errors(oracle)


def test_spans_abi_capacity(emu, oracle):
    SG.check_abi_capacity(oracle)


def test_spans_without_gpu_fails_loudly(product, oracle):
    if product.yttm_device_count() != 0:
        pytest.skip("a GPU is present")
    import youtokentome_b200 as yttm
    m = tmp_model_path()
    oracle.train(b"ab ab abc abd", m, 14)
    bpe = yttm.BPE(m)
    data, offs = _pack([b"ab abc", b"abd"])
    with pytest.raises(ValueError, match="no CUDA device"):
        bpe.encode_packed(data, offs, with_spans=True)
    with pytest.raises(ValueError, match="no CUDA device"):
        bpe.encode_subwords_packed(data, offs)
    assert bpe.vocab_size() > 4 and bpe.decode([[4, 5]]) and bpe.id_to_subword(4)


def test_unk_runs_of_the_restatement_match_host_pieces(emu, oracle):
    """The <UNK> pieces of the host path are the valid bytes of the restatement's spans."""
    m = SG._model(oracle, _cases.dirty_zipf_text(60_000), 700, 0.9)
    bpe, model = SG._bpe(m), SG.Model(m)
    sents = _cases.zipf_sentences(80) + SG.ADVERSARIAL
    data, offs = _pack(sents)
    ids, oo = bpe.encode_packed(data, offs)
    text, po, so = SG.host_subwords(bpe, data, offs, {})
    n_unk = 0
    for s in range(len(sents)):
        a = int(offs[s])
        sp = SG.oracle_spans(model, sents[s], ids[oo[s]:oo[s + 1]], a, False, False, False)
        for k, (i, (x, y)) in enumerate(zip(ids[oo[s]:oo[s + 1]].tolist(), sp)):
            j = int(so[s]) + k
            if i == model.unk:
                n_unk += 1
                assert text[po[j]:po[j + 1]] == SG._valid_bytes(data[x:y])
    assert n_unk > 20
    assert np.array_equal(so, oo)

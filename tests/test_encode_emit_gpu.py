"""The single-pass output kernel of device encode (emit_ids_kernel in youtokentome_b200/csrc/encode.cu): a block per
tile of EMIT_T = 256 consecutive sentences counts the tile's ids, finds the ids of the tiles in front of it by a
decoupled look-back, then writes the offsets, the ids and the spans.  The check bodies place sentences around the tile
edges; tests/test_encode_emit_emul_cpu.py runs them under the SIMT emulator.  On the GPU the tiles run concurrently,
so the look-back also waits for tiles that are not published yet; the bench-shape test covers thousands of tiles."""
import numpy as np
import pytest

import _cases
import test_encode_gpu as EG
import test_encode_spans_gpu as SG
from _gpu import GpuEncoder
from youtokentome_b200 import synth

pytestmark = pytest.mark.gpu

TILE = 256
_models = {}


def _model(oracle):
    if "zipf" not in _models:
        _models["zipf"] = EG._model(oracle, _cases.dirty_zipf_text(), 1500)
    return _models["zipf"]


def _same(oracle, sents, kws=SG.KWS, dropout=False):
    m = _model(oracle)
    g, o = GpuEncoder(m), oracle.encoder(m)
    for kw in kws:
        assert g.encode(sents, **kw) == o.encode(sents, **kw), kw
    if dropout:
        for p, seed in ((0.1, 3), (0.5, 9)):
            assert g.encode(sents, dropout=p, seed=seed) == o.encode(sents, dropout=p, seed=seed), p


def check_tile_counts(oracle, n):
    """n sentences: one, just under / exactly / just over one tile, two and several tiles."""
    sents = _cases.zipf_sentences(n, seed=n)
    _same(oracle, sents, SG.KWS if n in (1, 257) else SG.KWS[::3])


def check_empty_runs(oracle):
    """Runs of empty and wordless sentences that cross tile edges, a tile with no word at all, a batch of them only."""
    z = _cases.zipf_sentences(900, seed=2)
    blank = [b"", b" ", b"\t\n ", b"\xe2\x96\x81", b"\xe2\x96\x81 \xe2\x96\x81"]
    sents = z[:250] + [blank[i % 5] for i in range(12)] + z[250:500] + [b""] * (TILE + 7) + z[500:700]
    sents += [blank[i % 5] for i in range(TILE)] + z[700:]
    sents = [b""] * 3 + sents + [b" "] * (TILE - 1)
    _same(oracle, sents, SG.KWS[::3] + SG.KWS[5:6])
    _same(oracle, [blank[i % 5] for i in range(2 * TILE + 1)], SG.KWS[-1:])


def check_many_words(oracle):
    """Sentences of more than 32 and more than 256 words (a tile's words take several block-wide rounds), next to
    short ones, and a tile of one long sentence."""
    z = _cases.zipf_sentences(600, seed=7)
    words = b" ".join(z).split()
    long40, long300, long3000 = b" ".join(words[:40]), b" ".join(words[:300]), b" ".join(words[:3000])
    sents = z[:100] + [long40] * 5 + z[100:300] + [long300, b"", long3000] + z[300:] + [long40]
    _same(oracle, sents, SG.KWS[::2], dropout=True)
    _same(oracle, [long3000], SG.KWS[-1:])


def check_spans(oracle, n):
    """ids and spans for every bos / eos / reverse combination, with offsets[0] == 0 and != 0, around tile edges."""
    m = SG._model(oracle, _cases.dirty_zipf_text(60_000), 900)
    z = _cases.zipf_sentences(n, seed=5)
    sents = z[:TILE - 2] + [b"", b" ", b"", b"a" * 40 + b" b"] + z[TILE - 2:] + SG.ADVERSARIAL
    SG.check_sentences(oracle, m, sents)
    SG.check_sentences(oracle, m, sents[TILE - 10:TILE + 30], SG.KWS[::3], shift=5)


def check_dropout(oracle, n):
    """dropout > 0: every occurrence is its own record (no representatives), over several tiles."""
    _same(oracle, _cases.zipf_sentences(n, seed=8) + _cases.EDGE_SENTENCES, SG.KWS[::7], dropout=True)


@pytest.mark.parametrize("n", [1, 257, 4000])
def test_tile_counts(product, oracle, n):
    check_tile_counts(oracle, n)


def test_empty_runs_across_tile_edges(product, oracle):
    check_empty_runs(oracle)


def test_many_words_per_sentence(product, oracle):
    check_many_words(oracle)


def test_spans_all_flags_and_shift(product, oracle):
    check_spans(oracle, 1200)


def test_dropout(product, oracle):
    check_dropout(oracle, 5000)


# sha256 of the benchmark-shape ids (int32) followed by their offsets (uint64), as the build before the single-pass
# output kernel computed them with the model of _model()
BENCH_SHAPE_DIGEST = "ac641edefca2048c9751ea7cb6a77efe4bc733d333cef37ce2f4811767f24231"


def bench_shape_outputs(oracle):
    """(batch bytes, offsets, ids, id offsets, digest) of the benchmark's batch encoded with the model of _model()."""
    import hashlib
    import youtokentome_b200 as yttm
    buf, offs = synth.FastZipf(200_000, 1.07, 1234).packed_sentences(1_000_000, 128, seed=4321)
    ids, oo = yttm.BPE(_model(oracle)).encode_packed(np.frombuffer(bytes(buf), dtype=np.uint8),
                                                     np.asarray(offs, dtype=np.uint64))
    ids, oo = np.ascontiguousarray(ids, dtype=np.int32), np.ascontiguousarray(oo, dtype=np.uint64)
    return bytes(buf), offs, ids, oo.astype(np.int64), hashlib.sha256(ids.tobytes() + oo.tobytes()).hexdigest()


def test_bench_shape_against_oracle(product, oracle):
    """The benchmark's batch (1 M x 128 B Zipf sentences, about 3900 tiles): the ids and offsets of the whole batch
    hash to what the earlier build computed, and the ids of a sample spread over the batch (tile edges included) are
    the oracle's."""
    raw, offs, ids, oo, digest = bench_shape_outputs(oracle)
    n = len(offs) - 1
    assert oo[0] == 0 and len(oo) == n + 1 and oo[-1] == len(ids) and np.all(np.diff(oo) >= 0)
    assert digest == BENCH_SHAPE_DIGEST
    rng = np.random.default_rng(1)
    pick = sorted(set(rng.integers(0, n, 3000).tolist()) | {k * TILE + d for k in range(0, n // TILE, 97)
                                                           for d in (-1, 0, 1) if 0 <= k * TILE + d < n} | {n - 1})
    sents = [raw[int(offs[i]):int(offs[i + 1])] for i in pick]
    assert [ids[oo[i]:oo[i + 1]].tolist() for i in pick] == oracle.encoder(_model(oracle)).encode(sents)

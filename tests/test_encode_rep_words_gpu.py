"""The representative merge of device encode (encode_rep_words_kernel, youtokentome_b200/csrc/encode.cu) at the edges of
its shared-memory path: a word of at most SHARED_W = 17 tokens before merging (its "▁" and one per valid unit) is
merged in the thread's slots of shared memory; a word of more than SHARED_W bytes counts its bytes that are not
continuation bytes for that, up to SHARED_B = 64 bytes; any other word takes thread-private local arrays (up to 40
slots) or its slots in global memory.  Every case compares the ids with the oracle for several keyword sets, and the
spans and subword pieces with the restatement and the host path of tests/test_encode_spans_gpu.py:
  words of 15 .. 18 tokens, in 1- to 4-byte units;
  words of 62 .. 66 bytes of at most 17 tokens (stray continuation bytes add bytes, not tokens);
  unknown runs broken by invalid bytes and by stray continuation bytes (they do not break a run), and by known units;
  equal ranks along a word (runs a a a ..., the x == y rule at four levels);
  U+2581 with id 0, which a word drops when no rule merged it;
  words whose final ids number 3 and 4 (the first three ids sit in the word's record, the rest only in its slots);
  words whose length the finder did not know (they cross a piece edge of the finder): the dedup writes it back;
  a batch shaped like bench.py's (FastZipf sentences of 128 bytes, a 32k model trained on the GPU).
tests/test_encode_rep_words_emul_cpu.py runs the same bodies under the SIMT emulator, without the bench-shaped batch."""
import numpy as np
import pytest

import test_encode_spans_gpu as SG
import test_encode_words_gpu as WG

pytestmark = pytest.mark.gpu

SHARED_W, SHARED_B = 17, 64  # constexpr values of encode.cu (test_encode_rep_words_emul_cpu.py compares them)
SP = b"\xe2\x96\x81"
KWS = [dict(), dict(bos=True, eos=True, reverse=True)]
UNITS = [b"a", b"b", "ж".encode(), "и".encode(), "☃".encode(), "日".encode(), "😀".encode()]


def same(case, sents, spans=True):
    """ids == the oracle's for every keyword set; spans and pieces == the restatement and the host path."""
    for kw in KWS:
        if kw.get("bos") and case.model[2][2] == -1:
            continue
        assert case.g.encode(sents, **kw) == case.o.encode(sents, **kw), kw
    if spans:
        SG.check_sentences(None, case.path, sents, kws=KWS[:1])


def _in_sentences(words):
    """Each word alone, between other words, twice in one sentence and after U+2581."""
    return [w for w in words] + [b"x " + w + b" y" for w in words] + [w + b" " + w for w in words] + \
           [SP + w for w in words]


def check_token_counts(oracle):
    """Words of 14 .. 17 units (15 .. 18 tokens) of 1- to 4-byte units, so their byte lengths straddle 17 and 64."""
    case = WG.zipf_case(oracle)
    rng = np.random.default_rng(21)
    words = []
    for units in (14, 15, 16, 17):
        for parts in (UNITS[:2], UNITS[2:4], UNITS[4:6], UNITS[6:], UNITS):
            for _ in range(3):
                words.append(b"".join(parts[i] for i in rng.integers(0, len(parts), units)))
    same(case, _in_sentences(words))


def check_byte_counts(oracle):
    """Words of 62 .. 66 bytes and 14 .. 16 units: 4-byte units with stray continuation bytes or invalid lead bytes
    (the latter count as units for the path, not as tokens) in front of, between and behind them."""
    case = WG.zipf_case(oracle)
    em = "😀".encode()
    words = []
    for n in range(62, 67):
        for units in (14, 15, 16):
            pad = n - 4 * units
            if pad < 0:
                continue
            words += [em * units + b"\x80" * pad, b"\x80" * pad + em * units, b"\xff" * pad + em * units,
                      em * (units // 2) + b"\xbf" * pad + em * (units - units // 2)]
    for w in words:
        assert 62 <= len(w) <= 66
    same(case, _in_sentences(words))


def check_unknown_runs(oracle):
    """Units the model does not know (U+03A9, U+0416 at coverage 1.0 of a Latin text) in runs broken by an invalid
    lead byte, a stray continuation byte, a truncated sequence (they do not break the run) and a known unit."""
    case = WG.abcd_case(oracle)
    u, v = "Ω".encode(), "Ж".encode()
    words = [u + b"\xff" + v, u + b"\x80" + u, u + b"\xe2\x96" + v, u + b"a" + v, b"a" + u + b"\xff" + u + b"b" + v,
             b"\xff" + u + u, u + b"\x80\x80\x80" + b"ab" + v + b"\xc0\xaf" + v + b"c", b"\xff\xfe" + u, u * 15,
             (u + b"a") * 7, (u + b"\xbf") * 15, b"\x80" * 5 + u + b"a" + b"\x80" * 5 + u]
    same(case, _in_sentences(words))


def check_equal_ranks(oracle):
    """Runs a^k, b^k and mixed runs of up to 17 units under `runs` ((a,a) -> A -> B -> C -> D, (b,b))."""
    case = WG.runs_case(oracle)
    words = [b"a" * k for k in range(1, 18)] + [b"b" * k for k in range(1, 18)] + \
            [b"a" * k + b"b" * (15 - k) for k in range(16)] + [b"ab" * 8, b"aab" * 5, b"c" + b"a" * 14, b"abba" * 4]
    same(case, _in_sentences(words))


def check_space_id_zero(oracle):
    """U+2581 with id 0 and no rule for it: every word drops its "▁", on every path."""
    case = WG.runs0_case(oracle)
    words = [b"a" * k for k in range(1, 18)] + [b"c" * k for k in range(1, 18)] + [b"cab" * 5, b"ca" * 9]
    same(case, _in_sentences(words))


def check_record_boundary(oracle):
    """Final id counts 2 .. 5 under `runs`: c^k keeps its k ids, "▁" and k - 1 of them remain with U+2581 at id 0."""
    for case in (WG.runs_case(oracle), WG.runs0_case(oracle)):
        words = [b"c" * k for k in range(1, 6)] + [b"a" * 16 + b"c" * k for k in range(1, 5)]
        same(case, _in_sentences(words))


def check_unknown_lengths(oracle):
    """Words of 1 .. 70 bytes that cross the first piece edge (16 KB) of a long sentence, so the finder does not know
    their length, each its own representative (it occurs once); and the same words elsewhere in short sentences."""
    case = WG.zipf_case(oracle)
    rng = np.random.default_rng(23)
    for n in (1, 2, 15, 16, 17, 40, 63, 64, 65, 70):
        w = WG._sized(rng, n, UNITS)
        at = WG.FIND_TILE - n // 2
        head = WG._zipf_text(at - 1, 300 + n) + b" "
        same(case, [head + w + b" tail"], spans=n < 20)
        same(case, [head + w + b" tail", w, b"q " + w])


def check_bench_shaped(oracle, n_sent):
    """FastZipf sentences of 128 bytes, as bench.py encodes them, with a 32k model trained on the GPU: ids against
    the oracle, and spans and pieces on a slice."""
    from _gpu import GpuEncoder, gpu_train
    from youtokentome_b200 import synth
    fz = synth.FastZipf(n_words=200_000, s=1.07, seed=1234)
    model = gpu_train(fz.text(8_000_000, seed=5), 32_000, 1.0)
    data, offs = fz.packed_sentences(n_sent, 128, seed=4321)
    data = bytes(data)
    g, o = GpuEncoder(model), oracle.encoder(model)
    sents = [data[offs[i]:offs[i + 1]] for i in range(n_sent)]
    for kw in KWS:
        assert g.encode(sents, **kw) == o.encode(sents, **kw), kw
    SG.check_sentences(oracle, model, sents[:1500], kws=KWS[:1])


def test_token_counts(product, oracle):
    check_token_counts(oracle)


def test_byte_counts(product, oracle):
    check_byte_counts(oracle)


def test_unknown_runs(product, oracle):
    check_unknown_runs(oracle)


def test_equal_ranks(product, oracle):
    check_equal_ranks(oracle)


def test_space_id_zero(product, oracle):
    check_space_id_zero(oracle)


def test_record_boundary(product, oracle):
    check_record_boundary(oracle)


def test_unknown_lengths(product, oracle):
    check_unknown_lengths(oracle)


def test_bench_shaped(product, oracle):
    check_bench_shaped(oracle, 200_000)

"""Encoding files of any size to subword text on the GPU (BPE.encode_file(output_type=SUBWORD), yttm encode_file
--output_type subword, yttm_enc_stream_* with YTTM_STREAM_SUBWORD): every piece of a line followed by one space, then
"\\n", as `yttm encode --output_type subword` prints it.  Two references, both on the lines split in Python the way
std::getline splits them: the host path (encode(output_type=SUBWORD): the reference's own piece rule on device ids) and
the product's encode_subwords_packed, each framed in Python.

  1. line edges across piece sizes (every input of test_encode_file_gpu.edge_cases), the 8 bos / eos / reverse
     combinations, and the summary against the id form's;
  2. <UNK> runs (a model with coverage < 1 fed out-of-alphabet runs with invalid bytes inside and between them), pieces
     of more than 1 KB (a model trained on text without spaces), non-default special ids, ids above 65 535;
  3. dropout: the handle's sentence counter runs through the lines and advances as the id form's does;
  4. inputs and errors: a path, a FIFO, a descriptor, the C ABI fed in blocks, the open stream, the decode stream's
     refusal, failed calls, the CLI against `yttm encode --output_type subword`;
  5. the device memory bound (GPU only).

The bodies take the library: tests/test_encode_file_subword_emul_cpu.py runs 1 - 4 on the SIMT emulator."""
import ctypes as C
import os
import tempfile
import threading

import numpy as np
import pytest

import test_encode_file_gpu as F
import test_train_front_gpu as FG
from _bind import Oracle, tmp_model_path
from test_encode_spans_gpu import host_subwords
from youtokentome_b200 import _lib, synth
from youtokentome_b200.youtokentome import BPE, OutputType

pytestmark = pytest.mark.gpu
SUB = OutputType.SUBWORD
KWS = [dict(bos=b, eos=e, reverse=r) for b in (False, True) for e in (False, True) for r in (False, True)]
_models = {}


def framed(text, po, so):
    """Pieces as the CLI prints them: piece + " " per piece, "\\n" per sentence."""
    text, po, so = bytes(text), np.asarray(po).tolist(), np.asarray(so).tolist()
    out = []
    for s in range(len(so) - 1):
        out += [text[po[k]:po[k + 1]] + b" " for k in range(so[s], so[s + 1])]
        out.append(b"\n")
    return b"".join(out)


def want_text(bpe, data, **kw):
    """The subword text of data's getline lines from the host path; encode_subwords_packed must give the same."""
    lines = F.lines_of(data)
    if not lines:
        return b""
    buf, offs = F.packed(lines)
    host = framed(*host_subwords(bpe, buf, offs, kw))
    assert framed(*bpe.encode_subwords_packed(buf, offs, **kw)) == host
    return host


def run_sub(bpe, data, piece_kb=None, **kw):
    """encode_file(output_type=SUBWORD) of data -> (text bytes, summary); text=True is what F.run_file reads back."""
    return F.run_file(bpe, data, piece_kb, text=True, output_type=SUB, **kw)


def check(bpe, data, piece_kb, **kw):
    """The file's subword text equals both references; its summary equals the id form's."""
    want = want_text(bpe, data, **kw)
    got, r = run_sub(bpe, data, piece_kb, **kw)
    assert got == want, (len(got), len(want))
    _, r_id = F.run_file(bpe, data, piece_kb, text=True, **kw)
    assert r == r_id
    return r


def model(kind):
    """Models trained by the oracle once per process: "unk" (coverage 0.95 on multilingual text), "long" (pieces of
    2 KB, trained on text without spaces), "special" (pad / unk / bos / eos at 7 / 0 / 5 / 9)."""
    if kind not in _models:
        m = tmp_model_path(kind)
        if kind == "unk":
            text = (synth.readme_corpus(n_lines=300) + "привет мир ёжик héllo 日本語 テキスト ☃ ωμέγα\n".encode() * 30 +
                    "ünïcödé ǅ ѣѳ ꙮ 丂丄 ♞♜\n".encode() * 2)
            Oracle().train(text, m, 500, 0.95)
        elif kind == "long":
            Oracle().train((b"ab" * 4096 + b"\n") * 40 + b"c d e\n", m, 20, 1.0)
        else:
            Oracle().train(synth.readme_corpus(n_lines=300), m, 300, 1.0, pad=7, unk=0, bos=5, eos=9)
        _models[kind] = m
    return _models[kind]


# ---- 1. line edges ---------------------------------------------------------------------------------------------------
def edges(L, piece_sizes, small=False):
    bpe = BPE(F.model())
    for name, data in F.edge_cases(small):
        for kb in piece_sizes:
            r = check(bpe, data, kb)
            assert r["lines"] == len(F.lines_of(data)), name


def flags(L, piece_sizes):
    bpe = BPE(F.model())
    data = F.edge_cases(small=True)[3][1] + b"\n\n" + "héllo ▁ 日本語\n".encode()
    for kb in piece_sizes:
        for kw in KWS:
            check(bpe, data, kb, **kw)


# ---- 2. <UNK> runs, long pieces, special ids ---------------------------------------------------------------------------
def unk_lines(n, seed=4):
    """Lines full of out-of-alphabet runs, invalid bytes inside and between them, runs at line starts and ends."""
    rng = np.random.default_rng(seed)
    foreign = "ΔΘΛΞΠΣΦΨ한국어글자🙂🚀🎉𝄞ꜰꜱ"
    words = ["ab", "the", "héllo", "мир", "日本"]
    bad = [b"\x80", b"\xff\xfe", b"\xe2\x96", b"\xc0\xaf", b"\xed\xa0\x80", b"\xf0\x9f\x98"]
    out = []
    for _ in range(n):
        parts = []
        for _ in range(int(rng.integers(1, 12))):
            k = int(rng.integers(0, 4))
            if k == 0:
                parts.append(words[int(rng.integers(len(words)))].encode())
            else:
                run = b""
                for _ in range(int(rng.integers(1, 9))):
                    run += foreign[int(rng.integers(len(foreign)))].encode()
                    if rng.random() < 0.3:
                        run += bad[int(rng.integers(len(bad)))]
                parts.append(run)
            parts.append(b" " if rng.random() < 0.7 else bad[int(rng.integers(len(bad)))])
        out.append(b"".join(parts).rstrip(b" "))
    return b"\n".join(out) + b"\n"


def unk_runs(L, piece_sizes, small=False):
    bpe = BPE(model("unk"))
    data = unk_lines(150 if small else 3000)
    buf, offs = F.packed(F.lines_of(data))
    ids, _ = bpe.encode_packed(buf, offs)
    assert np.count_nonzero(ids == bpe.subword_to_id("<UNK>")) > 100
    for kb in piece_sizes:
        check(bpe, data, kb, eos=True)
        check(bpe, data, kb, bos=True, reverse=True)


def long_pieces(L, piece_sizes, small=False):
    bpe = BPE(model("long"))
    assert max(len(p.encode()) for p in bpe.vocab()) >= 1024
    rng = np.random.default_rng(8)
    lines = [b" ".join(b"ab" * int(rng.integers(1, 3000)) + (b"c" if rng.random() < 0.3 else b"") for _ in range(k))
             for k in rng.integers(1, 12, 10 if small else 60)]
    data = b"\n".join(lines) + b"\nab c " + b"ab" * 2048 + b"\xff" + b"ab" * 1500 + b"\n"
    buf, offs = F.packed(F.lines_of(data))
    _, po, _ = bpe.encode_subwords_packed(buf, offs)
    assert np.diff(po.astype(np.int64)).max() >= 1024
    for kb in piece_sizes:
        check(bpe, data, kb)
        check(bpe, data, kb, bos=True, eos=True, reverse=True)


def special_and_wide(L, piece_kb):
    bpe = BPE(model("special"))
    data = synth.readme_corpus(n_lines=200) + "日本 ☃ héllo\n\n".encode()
    for kw in (KWS[0], KWS[-1], dict(bos=True, eos=True)):
        check(bpe, data, piece_kb, **kw)
    wide = BPE(F.model("wide"))
    assert wide.vocab_size() > 65536
    chars = "".join(chr(0x10000 + k) for k in range(0, 70_000, 997))
    data = ("ab " + chars + " cd ☃\n" + chars[::-1] + "\nz\n").encode() * 20
    buf, offs = F.packed(F.lines_of(data))
    assert bpe_ids_max(wide, buf, offs) > 65535
    check(wide, data, piece_kb)
    check(wide, data, piece_kb, bos=True, eos=True)


def bpe_ids_max(bpe, buf, offs):
    return int(bpe.encode_packed(buf, offs)[0].max())


# ---- 3. dropout ------------------------------------------------------------------------------------------------------
def dropout(L, piece_sizes, small=False):
    bpe = BPE(F.model())
    data = synth.readme_corpus(n_lines=300 if small else 3000) + "héllo wörld\n".encode() * 10
    lines = F.lines_of(data)
    buf, offs = F.packed(lines)
    for p in (0.1, 0.5):
        bpe.dropout_seed(11)
        want = [framed(*bpe.encode_subwords_packed(buf, offs, dropout_prob=p)) for _ in range(2)]
        assert want[0] != want[1]
        for kb in piece_sizes:
            bpe.dropout_seed(11)
            for k in range(2):   # the second call continues the sentence counter
                assert run_sub(bpe, data, kb, dropout_prob=p)[0] == want[k]
        assert abi_run(L, bpe, data, 7, 1, dropout=p, seed=11, first=len(lines))[0] == want[1]
    # the counter advances as the id form's: an id file after an N-line subword file gets the draws it gets after an
    # N-line id file
    other = synth.readme_corpus(n_lines=120)
    after = []
    for first in ("subword", "id"):
        bpe.dropout_seed(5)
        if first == "subword":
            run_sub(bpe, data, dropout_prob=0.5)
        else:
            F.run_file(bpe, data, dropout_prob=0.5)
        after.append(F.run_file(bpe, other, dropout_prob=0.5)[0])
    bpe.dropout_seed(5)
    fresh = F.run_file(bpe, other, dropout_prob=0.5)[0]
    np.testing.assert_array_equal(after[0][0], after[1][0])
    np.testing.assert_array_equal(after[0][1], after[1][1])
    assert not np.array_equal(after[0][0], fresh[0])


# ---- 4. inputs and errors --------------------------------------------------------------------------------------------
def abi_run(L, bpe, data, kind, piece_kb, dropout=0.0, seed=0, first=0, bos=0, eos=0, rev=0):
    """yttm_enc_stream_* with YTTM_STREAM_SUBWORD, fed in blocks from ONE reused buffer -> (text, line ends,
    (lines, ids, bytes))."""
    enc, ctx = L.yttm_api_device_encoder(bpe._h), L.yttm_api_device_context(bpe._h)
    got, ends = [], []

    def sink(user, ptr, n, le, nl):
        got.append(C.string_at(ptr, n) if n else b"")
        ends.extend(le[k] for k in range(nl))
        return 0
    cb = _lib.ENC_SINK(sink)
    with FG.env(YTTM_ENC_STREAM_PIECE_KB=piece_kb):
        assert L.yttm_enc_stream_begin(enc, bos, eos, rev, dropout, seed, first, _lib.STREAM_SUBWORD, cb, None) == 0, \
            L.yttm_last_error(ctx)
    buf = C.create_string_buffer(max(len(data), 1))
    at, blocks = 0, F._blocks(kind)
    while at < len(data):
        k = min(next(blocks), len(data) - at)
        C.memmove(buf, data[at:at + k], k)
        assert L.yttm_enc_stream_feed(enc, buf, k) == 0, L.yttm_last_error(ctx)
        C.memset(buf, 0x0a, k)   # the library copied the block
        at += k
    n = [C.c_uint64(0) for _ in range(3)]
    assert L.yttm_enc_stream_end(enc, *[C.byref(x) for x in n]) == 0, L.yttm_last_error(ctx)
    return b"".join(got), np.array(ends, dtype=np.uint64), tuple(x.value for x in n)


def abi_blocks(L, small=False):
    bpe = BPE(model("unk"))
    data = b"".join(c[1] for c in F.edge_cases(small=True)[2:10]) + unk_lines(40)
    data = data[:12_000] if small else data
    kw = dict(bos=True, reverse=True)
    want = want_text(bpe, data, **kw)
    buf, offs = F.packed(F.lines_of(data))
    want_ids, want_offs = bpe.encode_packed(buf, offs, **kw)
    for kind in (1, 7, "random"):
        got, ends, n = abi_run(L, bpe, data, kind, 1, bos=1, rev=1)
        assert got == want
        np.testing.assert_array_equal(ends, want_offs[1:])
        assert n == (len(want_offs) - 1, len(want_ids), len(data))
        assert L.yttm_stage_ms(L.yttm_api_device_context(bpe._h), b"stream_pieces") > 1


def inputs(L, piece_kb):
    """A path, a FIFO, an open file object and a raw descriptor give the same text."""
    bpe = BPE(F.model())
    data = synth.readme_corpus(n_lines=600) + "日本 ☃\n".encode()
    want = want_text(bpe, data)
    got, r = run_sub(bpe, data, piece_kb)
    assert got == want
    path = os.path.join(tempfile.mkdtemp(dir=F._tmp), "fifo")
    os.mkfifo(path)

    def writer():
        with open(path, "wb") as f:
            for k in range(0, len(data), 999):
                f.write(data[k:k + 999])
    t = threading.Thread(target=writer)
    t.start()
    out = os.path.join(tempfile.mkdtemp(dir=F._tmp), "out")
    try:
        with FG.env(YTTM_ENC_STREAM_PIECE_KB=piece_kb):
            r1 = bpe.encode_file(path, out + "1", output_type=SUB)
    finally:
        t.join()
    src = F.write(data)
    with open(src, "rb") as f:
        r2 = bpe.encode_file(f, out + "2", output_type=SUB)
    fd = os.open(src, os.O_RDONLY)
    try:
        r3 = bpe.encode_file(fd, out + "3", text=True, output_type=SUB)   # text=True changes nothing
    finally:
        os.close(fd)
    assert r1 == r2 == r3 == r
    for k in "123":
        with open(out + k, "rb") as f:
            assert f.read() == want


def abi_misuse(L):
    bpe = BPE(F.model())
    enc, ctx = L.yttm_api_device_encoder(bpe._h), L.yttm_api_device_context(bpe._h)
    err = lambda: L.yttm_last_error(ctx).decode()   # noqa: E731
    n = [C.c_uint64(0) for _ in range(3)]
    refs = [C.byref(x) for x in n]
    ok = _lib.ENC_SINK(lambda *a: 0)
    assert L.yttm_enc_stream_begin(enc, 0, 0, 0, 0.0, 0, 0, 4, ok, None) != 0
    assert "YTTM_STREAM_TEXT or YTTM_STREAM_SUBWORD" in err()
    # the decode stream has no subword input
    assert L.yttm_dec_stream_begin(enc, _lib.STREAM_SUBWORD, None, 0, ok, None) != 0
    assert "yttm_dec_stream_begin: format must be" in err()
    # an open subword stream owns the encoder: begin again, encode and decode calls fail; end closes it
    assert L.yttm_enc_stream_begin(enc, 0, 0, 0, 0.0, 0, 0, _lib.STREAM_SUBWORD, ok, None) == 0, err()
    assert L.yttm_enc_stream_feed(enc, b"ab cd\n" * 10, 60) == 0, err()
    assert L.yttm_enc_stream_begin(enc, 0, 0, 0, 0.0, 0, 0, _lib.STREAM_IDS32, ok, None) != 0
    assert "encode stream is open" in err()
    with pytest.raises(ValueError, match="encode stream is open"):
        bpe.encode_subwords_packed(b"ab", np.array([0, 2], dtype=np.uint64))
    with pytest.raises(ValueError, match="encode stream is open"):
        bpe.decode_packed(np.array([5], dtype=np.int32), np.array([0, 1], dtype=np.uint64))
    assert L.yttm_dec_stream_begin(enc, _lib.STREAM_TEXT, None, 0, ok, None) != 0
    assert L.yttm_enc_stream_end(enc, *refs) == 0, err()
    assert n[0].value == 10 and n[2].value == 60
    data = b"ab cd\n" * 10
    assert abi_run(L, bpe, data, 999, 1)[0] == want_text(bpe, data)


def failed_calls(L):
    """A failed call raises and leaves nothing at the output name; the handle works after the failures."""
    bpe = BPE(F.model())
    d = tempfile.mkdtemp(dir=F._tmp)
    out = os.path.join(d, "out.txt")
    with pytest.raises(ValueError, match="missing.txt"):
        bpe.encode_file(os.path.join(d, "missing.txt"), out, output_type=SUB)
    src = F.write(b"ab cd\n" * 100)
    with pytest.raises(ValueError, match="nodir"):
        bpe.encode_file(src, os.path.join(d, "nodir", "out"), output_type=SUB)
    with pytest.raises(ValueError, match="Can't add <BOS>"):
        BPE(F.model("nobos")).encode_file(src, out, bos=True, output_type=SUB)
    with pytest.raises(TypeError, match="output_type must be youtokentome.OutputType"):
        bpe.encode_file(src, out, output_type="subword")
    fd = os.open(d, os.O_RDONLY)   # reading a directory fails after the output was opened
    try:
        with FG.env(YTTM_ENC_STREAM_PIECE_KB=1):
            with pytest.raises(ValueError, match="cannot read the input"):
                bpe.encode_file(fd, out, output_type=SUB)
    finally:
        os.close(fd)
    assert sorted(os.listdir(d)) == [], os.listdir(d)
    r = bpe.encode_file(src, out, output_type=SUB)
    assert r["lines"] == 100 and sorted(os.listdir(d)) == ["out.txt"]
    with open(out, "rb") as f:
        assert f.read() == want_text(bpe, b"ab cd\n" * 100)


# ---- GPU tests -------------------------------------------------------------------------------------------------------
@pytest.fixture
def lib(product):
    return product


def test_line_edges(lib):
    edges(lib, (1, 7, None))


def test_bos_eos_reverse(lib):
    flags(lib, (1, None))


def test_unk_runs(lib):
    unk_runs(lib, (1, 7, None))


def test_long_pieces(lib):
    long_pieces(lib, (1, 7, None))


def test_special_ids_and_wide_model(lib):
    special_and_wide(lib, 1)


def test_dropout_counter(lib):
    dropout(lib, (1, 7, None))


def test_inputs(lib):
    inputs(lib, 1)


def test_abi_blocks(lib):
    abi_blocks(lib)


def test_abi_misuse(lib):
    abi_misuse(lib)


def test_failed_calls_leave_nothing(lib):
    failed_calls(lib)


def test_cli_matches_yttm_encode_subword(lib):
    """`yttm encode_file --output_type subword` from stdin and from a path gives the stdout of `yttm encode
    --output_type subword`, byte for byte, with and without --bos --eos --reverse; the summary goes to stderr."""
    m = model("unk")
    data = F.edge_cases(small=True)[3][1] + "\n\nhéllo \x0b\n\r\n".encode() + unk_lines(30)
    src = F.write(data)
    for flag in ([], ["--bos", "--eos", "--reverse"]):
        old = F._cli("encode", "--model", m, "--output_type", "subword", *flag, stdin=data).stdout
        new = F._cli("encode_file", "--model", m, "--input", "-", "--output", "-", "--output_type", "subword", *flag,
                     stdin=data)
        assert new.stdout == old
        assert b"encode_file: %d lines" % len(F.lines_of(data)) in new.stderr
        out = os.path.join(tempfile.mkdtemp(dir=F._tmp), "t.txt")
        r = F._cli("encode_file", "--model", m, "--input", src, "--output", out, "--output_type", "subword", "--text",
                   *flag)
        assert r.stdout == b""
        with open(out, "rb") as f:
            assert f.read() == old


def test_device_memory_does_not_grow_with_the_file(lib):
    """configs[1]-shaped files of 64 MB and 512 MB in default (32 MB) pieces: the same device peak."""
    bpe = BPE(F.model())
    fz = synth.FastZipf(n_words=200_000, seed=1234)
    small = fz.text(64 << 20, words_per_line=20)
    peaks = []
    for data in (small, small * 8):
        src = F.write(data)
        out = os.path.join(tempfile.mkdtemp(dir=F._tmp), "o.txt")
        r = bpe.encode_file(src, out, output_type=SUB)
        os.remove(src)
        ctx = lib.yttm_api_device_context(bpe._h)
        peaks.append(lib.yttm_stage_ms(ctx, b"stream_dev_peak_bytes"))
        pieces = lib.yttm_stage_ms(ctx, b"stream_pieces")
        size = os.path.getsize(out)
        os.remove(out)
        print("%d MB: %d lines in %d pieces, %d MB of subword text, device peak %.1f MB" %
              (len(data) >> 20, r["lines"], pieces, size >> 20, peaks[-1] / 2 ** 20))
        assert pieces >= len(data) // (32 << 20)
        assert r["lines"] == data.count(b"\n")
    assert peaks[0] == peaks[1], peaks

"""Encoding files of any size on the GPU (BPE.encode_file, yttm encode_file, yttm_enc_stream_* of yttm_b200.h): the
text is fed in pieces that end behind a '\\n', the lines are found on the device, and the ids leave as .npy files or as
the text of `yttm encode --output_type id`.  The references are the product's own encode_packed and the oracle, on
lines split in Python the way std::getline splits them.

  1. line edges across piece sizes: empty and newline-only files, CRLF, lone \\r, \\v / \\f / space lines, \\0, UTF-8
     and invalid bytes next to the cuts, a line much longer than a piece, a long word without spaces, the golden test
     texts and configs[1]-shaped lines, bos / eos / reverse, a model without <BOS>;
  2. dropout: the sentence counter of the handle runs through the lines, whatever the piece and block sizes;
  3. formats: the .npy pair, uint16 and int32 ids, the text form;
  4. inputs and errors: a path, a FIFO, the C ABI fed in blocks with a ctypes sink, misuse, failed calls;
  5. the device memory bound (GPU only).

The bodies take the library: tests/test_encode_file_emul_cpu.py runs 1 - 4 on the SIMT emulator at small sizes."""
import base64
import ctypes as C
import glob
import json
import os
import subprocess
import sys
import tempfile
import threading

import numpy as np
import pytest

import test_train_front_gpu as FG
from _bind import ROOT, Oracle, tmp_model_path
from youtokentome_b200 import _lib, synth
from youtokentome_b200.youtokentome import BPE

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "*.json")))
_tmp = tempfile.mkdtemp(prefix="yttm_encfile_")
_models = {}


def lines_of(data):
    """std::getline's lines: split at '\\n'; a trailing '\\n' ends the last line instead of starting an empty one."""
    parts = data.split(b"\n")
    if parts[-1] == b"":
        parts.pop()
    return parts


def packed(lines):
    offs = np.zeros(len(lines) + 1, dtype=np.uint64)
    if lines:
        np.cumsum([len(s) for s in lines], out=offs[1:])
    return b"".join(lines), offs


def as_text(ids, offs):
    ids, offs = ids.tolist(), offs.tolist()
    return b"".join(b"".join(b"%d " % i for i in ids[offs[k]:offs[k + 1]]) + b"\n" for k in range(len(offs) - 1))


def model(kind="base"):
    """Models trained by the oracle once per process: "base" (vocab 400), "nobos" (no <BOS>), "wide" (a hand-written
    model of 70 000 characters: ids above 65 535)."""
    if kind not in _models:
        m = tmp_model_path(kind)
        if kind == "wide":
            cps = [9601] + list(range(ord("a"), ord("z") + 1)) + list(range(0x10000, 0x10000 + 70_000))
            with open(m, "w") as f:
                f.write("%d 0\n" % len(cps))
                f.writelines("%d %d\n" % (cp, 4 + i) for i, cp in enumerate(cps))
                f.write("1 0 2 3\n")
        else:
            text = synth.readme_corpus(n_lines=300) + "héllo wörld ▁ 日本語 テキスト\n".encode() * 20
            Oracle().train(text, m, 400, 1.0, **({"bos": -1} if kind == "nobos" else {}))
        _models[kind] = m
    return _models[kind]


def write(data):
    fd, path = tempfile.mkstemp(dir=_tmp, suffix=".txt")
    with os.fdopen(fd, "wb") as f:
        f.write(data)
    return path


def run_file(bpe, data, piece_kb=None, text=False, **kw):
    """encode_file of `data` -> (ids, offsets) read back from the .npy pair, or the text bytes; and the summary."""
    src = write(data)
    out = os.path.join(tempfile.mkdtemp(dir=_tmp), "out")
    with FG.env(**({"YTTM_ENC_STREAM_PIECE_KB": piece_kb} if piece_kb else {})):
        r = bpe.encode_file(src, out, text=text, **kw)
    os.remove(src)
    assert r["bytes"] == len(data)
    if text:
        with open(out, "rb") as f:
            return f.read(), r
    ids = np.load(out + ".ids.npy", mmap_mode="r")
    offs = np.load(out + ".offsets.npy", mmap_mode="r")
    assert offs.dtype == np.uint64 and offs[0] == 0 and int(offs[-1]) == len(ids)
    assert r["lines"] == len(offs) - 1 and r["ids"] == len(ids)
    return (np.array(ids), np.array(offs)), r


def expected(bpe, data, **kw):
    buf, offs = packed(lines_of(data))
    return bpe.encode_packed(buf, offs, **kw)


def check(bpe, data, piece_kb, **kw):
    """encode_file equals encode_packed of the getline lines, in both forms."""
    want_ids, want_offs = expected(bpe, data, **kw)
    (ids, offs), r = run_file(bpe, data, piece_kb, **kw)
    assert ids.dtype == np.uint16
    assert len(offs) == len(want_offs), (len(offs), len(want_offs))
    np.testing.assert_array_equal(offs, want_offs)
    np.testing.assert_array_equal(ids.astype(np.int32), want_ids)
    txt, _ = run_file(bpe, data, piece_kb, text=True, **kw)
    assert txt == as_text(want_ids, want_offs)
    return r


# ---- 1. line edges ---------------------------------------------------------------------------------------------------
def edge_cases(small=False):
    rng = np.random.default_rng(3)
    base = synth.readme_corpus(n_lines=400 if small else 2000)
    cjk = "日本語 テキスト▁a ▁▁ 𝄞x héllo\n".encode()
    bad = b"\x80\xbfab \xff\xfeab\xe2\x96 \xc0\xaf\n\xed\xa0\x80 \xf0\x9f\x98\n\x80\x80 "
    long_line = (b"ab cd " * ((30_000 if small else 3_000_000) // 6))
    word = bytes(rng.choice(np.frombuffer(b"abcd", dtype=np.uint8), 30_000 if small else 300_000))
    golden = []
    for path in GOLDEN:
        with open(path) as f:
            golden += [base64.b64decode(s) for s in json.load(f)["sentences_b64"]]
    golden = b"\n".join(golden) + b"\n"
    cfg1 = synth.FastZipf(n_words=20_000, seed=5).packed_sentences(200 if small else 3000, 128, seed=9)
    cfg1_text = b"\n".join(cfg1[0][int(a):int(b)] for a, b in zip(cfg1[1][:-1], cfg1[1][1:])) + b"\n"
    return [
        ("empty", b""),
        ("newline only", b"\n"),
        ("three newlines", b"\n\n\n"),
        ("no final newline", base[:3000] + b"last line"),
        ("crlf", base[:4000].replace(b"\n", b"\r\n")),
        ("lone cr", base[:4000].replace(b"\n", b"\r") + b"\n" + base[:2000]),
        ("blank lines", b"   \n\x0b\x0b\n\x0c\n \x0c \x0b\n\t\n" * 100),
        ("nul bytes", base[:3000].replace(b"a", b"\0") + b"\n\0\n"),
        ("utf-8 at the cuts", b"".join(cjk[:k] + base[k * 13:k * 13 + 211] for k in range(len(cjk))) * 4),
        ("invalid bytes at the cuts", b"".join(bad[k:] + base[k * 11:k * 11 + 97] for k in range(len(bad))) * 6),
        ("line longer than pieces", base[:1500] + long_line + b"\n" + base[:1500]),
        ("long word", b"x " + word + b" y\n" + base[:2000]),
        ("golden test texts", golden),
        ("configs[1] lines", cfg1_text),
    ]


def edges(L, piece_sizes, small=False):
    bpe = BPE(model())
    for name, data in edge_cases(small):
        for kb in piece_sizes:
            r = check(bpe, data, kb)
            assert r["lines"] == len(lines_of(data)), name


def flags(L, piece_kb):
    bpe = BPE(model())
    data = edge_cases(small=True)[3][1] + b"\n\n"
    for bos in (False, True):
        for eos in (False, True):
            for rev in (False, True):
                check(bpe, data, piece_kb, bos=bos, eos=eos, reverse=rev)
    nobos = BPE(model("nobos"))
    with pytest.raises(ValueError) as e_packed:
        nobos.encode_packed(b"ab", np.array([0, 2], dtype=np.uint64), bos=True)
    with pytest.raises(ValueError) as e_file:
        run_file(nobos, b"ab\n", piece_kb, bos=True)
    assert str(e_file.value) == str(e_packed.value) == "Can't add <BOS> token. Model was trained without it."


# ---- 2. dropout ------------------------------------------------------------------------------------------------------
def dropout(L, piece_sizes, small=False):
    m = model()
    bpe = BPE(m)
    data = synth.readme_corpus(n_lines=300 if small else 3000) + "héllo wörld\n".encode() * 10
    lines = lines_of(data)
    buf, offs = packed(lines)
    for p in (0.1, 0.5):
        bpe.dropout_seed(11)
        want = [bpe.encode_packed(buf, offs, dropout_prob=p) for _ in range(2)]
        for kb in piece_sizes:
            bpe.dropout_seed(11)
            for k in range(2):   # the second call continues the sentence counter
                (ids, oo), _ = run_file(bpe, data, kb, dropout_prob=p)
                np.testing.assert_array_equal(ids.astype(np.int32), want[k][0])
                np.testing.assert_array_equal(oo, want[k][1])
        for kind in (7, "random"):   # feed block sizes of the C ABI
            got = abi_run(L, bpe, data, kind, 1, dropout=p, seed=11, first=len(lines))
            np.testing.assert_array_equal(got[0], want[1][0])
        # the oracle on a sample of lines: same Philox key (seed, sentence index, word offset)
        enc = Oracle().encoder(m)
        pick = list(range(0, len(lines), max(1, len(lines) // 40)))
        for i in pick[:40]:
            b1, o1 = packed([lines[i]])
            oi, _ = enc.encode_packed(b1, o1, dropout=p, seed=11, first_index=len(lines) + i)
            np.testing.assert_array_equal(np.asarray(oi, dtype=np.int32),
                                          want[1][0][int(want[1][1][i]):int(want[1][1][i + 1])])


# ---- 3. formats ------------------------------------------------------------------------------------------------------
def wide_ids(L, piece_kb):
    """A model of more than 65 536 ids writes int32, and ids above 65 535 survive."""
    bpe = BPE(model("wide"))
    assert bpe.vocab_size() > 65536
    chars = "".join(chr(0x10000 + k) for k in range(0, 70_000, 997))
    data = ("ab " + chars + " cd\n" + chars[::-1] + "\nz\n").encode() * 20
    want_ids, want_offs = expected(bpe, data)
    assert want_ids.max() > 65535
    (ids, offs), _ = run_file(bpe, data, piece_kb)
    assert ids.dtype == np.int32
    np.testing.assert_array_equal(ids, want_ids)
    np.testing.assert_array_equal(offs, want_offs)
    txt, _ = run_file(bpe, data, piece_kb, text=True)
    assert txt == as_text(want_ids, want_offs)


# ---- 4. inputs and errors --------------------------------------------------------------------------------------------
def fifo(L, piece_kb):
    bpe = BPE(model())
    data = synth.readme_corpus(n_lines=600)
    path = os.path.join(tempfile.mkdtemp(dir=_tmp), "fifo")
    os.mkfifo(path)

    def writer():
        with open(path, "wb") as f:
            for k in range(0, len(data), 999):
                f.write(data[k:k + 999])
    t = threading.Thread(target=writer)
    t.start()
    out = os.path.join(tempfile.mkdtemp(dir=_tmp), "out")
    try:
        with FG.env(YTTM_ENC_STREAM_PIECE_KB=piece_kb):
            r = bpe.encode_file(path, out)
    finally:
        t.join()
    want_ids, want_offs = expected(bpe, data)
    np.testing.assert_array_equal(np.load(out + ".ids.npy").astype(np.int32), want_ids)
    np.testing.assert_array_equal(np.load(out + ".offsets.npy"), want_offs)
    assert r == {"lines": len(want_offs) - 1, "ids": len(want_ids), "bytes": len(data)}
    # an open file object and a raw descriptor
    src = write(data)
    with open(src, "rb") as f:
        r2 = bpe.encode_file(f, out + "2", text=True)
    fd = os.open(src, os.O_RDONLY)
    try:
        r3 = bpe.encode_file(fd, out + "3", text=True)
    finally:
        os.close(fd)
    assert r2 == r3 == r
    with open(out + "2", "rb") as f, open(out + "3", "rb") as g:
        assert f.read() == g.read() == as_text(want_ids, want_offs)


def _blocks(kind, seed=5):
    rng = np.random.default_rng(seed)
    while True:
        yield kind if isinstance(kind, int) else int(rng.integers(1, 3000))


def abi_run(L, bpe, data, kind, piece_kb, fmt=_lib.STREAM_IDS32, dropout=0.0, seed=0, first=0, bos=0, eos=0, rev=0):
    """yttm_enc_stream_* on the handle's encoder, fed in blocks from ONE reused buffer, results gathered by a ctypes
    sink -> (data as int32 / uint16 ids or text bytes, line ends, (lines, ids, bytes))."""
    enc = L.yttm_api_device_encoder(bpe._h)
    ctx = L.yttm_api_device_context(bpe._h)
    got, ends = [], []

    def sink(user, ptr, n, le, nl):
        got.append(C.string_at(ptr, n) if n else b"")
        ends.extend(le[k] for k in range(nl))
        return 0
    cb = _lib.ENC_SINK(sink)
    with FG.env(YTTM_ENC_STREAM_PIECE_KB=piece_kb):
        assert L.yttm_enc_stream_begin(enc, bos, eos, rev, dropout, seed, first, fmt, cb, None) == 0, L.yttm_last_error(ctx)
    buf = C.create_string_buffer(max(len(data), 1))
    at, blocks = 0, _blocks(kind)
    while at < len(data):
        k = min(next(blocks), len(data) - at)
        C.memmove(buf, data[at:at + k], k)
        assert L.yttm_enc_stream_feed(enc, buf, k) == 0, L.yttm_last_error(ctx)
        C.memset(buf, 0x0a, k)   # the library copied the block
        at += k
    n = [C.c_uint64(0) for _ in range(3)]
    assert L.yttm_enc_stream_end(enc, *[C.byref(x) for x in n]) == 0, L.yttm_last_error(ctx)
    raw = b"".join(got)
    out = raw if fmt == _lib.STREAM_TEXT else np.frombuffer(raw, dtype=np.uint16 if fmt == _lib.STREAM_IDS16 else np.int32)
    return out, np.array(ends, dtype=np.uint64), tuple(x.value for x in n), L.yttm_stage_ms(ctx, b"stream_pieces")


def abi_blocks(L, small=False):
    bpe = BPE(model())
    data = b"".join(c[1] for c in edge_cases(small=True)[2:10])
    data = data[:12_000] if small else data
    want_ids, want_offs = expected(bpe, data, bos=True, reverse=True)
    for kind in (1, 7, "random"):
        for fmt in (_lib.STREAM_IDS32, _lib.STREAM_IDS16, _lib.STREAM_TEXT):
            if kind == 1 and fmt != _lib.STREAM_IDS32:
                continue
            out, ends, n, pieces = abi_run(L, bpe, data, kind, 1, fmt, bos=1, rev=1)
            assert n == (len(want_offs) - 1, len(want_ids), len(data))
            assert pieces > 1
            np.testing.assert_array_equal(ends, want_offs[1:])
            if fmt == _lib.STREAM_TEXT:
                assert out == as_text(want_ids, want_offs)
            else:
                np.testing.assert_array_equal(out.astype(np.int32), want_ids)


def abi_misuse(L):
    bpe = BPE(model())
    enc, ctx = L.yttm_api_device_encoder(bpe._h), L.yttm_api_device_context(bpe._h)
    err = lambda: L.yttm_last_error(ctx).decode()   # noqa: E731
    n = [C.c_uint64(0) for _ in range(3)]
    refs = [C.byref(x) for x in n]
    ok = _lib.ENC_SINK(lambda *a: 0)
    assert L.yttm_enc_stream_feed(enc, b"ab\n", 3) != 0 and "yttm_enc_stream_begin has not run" in err()
    assert L.yttm_enc_stream_end(enc, *refs) != 0 and "yttm_enc_stream_begin has not run" in err()
    wide = BPE(model("wide"))
    wenc, wctx = L.yttm_api_device_encoder(wide._h), L.yttm_api_device_context(wide._h)
    assert L.yttm_enc_stream_begin(wenc, 0, 0, 0, 0.0, 0, 0, _lib.STREAM_IDS16, ok, None) != 0
    assert "16-bit ids need a vocabulary of at most 65536" in L.yttm_last_error(wctx).decode()
    # an open stream owns the encoder: begin again, encode and decode calls fail; end closes it
    assert L.yttm_enc_stream_begin(enc, 0, 0, 0, 0.0, 0, 0, _lib.STREAM_IDS32, ok, None) == 0, err()
    assert L.yttm_enc_stream_feed(enc, b"ab cd\n" * 10, 60) == 0, err()
    assert L.yttm_enc_stream_begin(enc, 0, 0, 0, 0.0, 0, 0, _lib.STREAM_IDS32, ok, None) != 0
    assert "encode stream is open" in err()
    with pytest.raises(ValueError, match="encode stream is open"):
        bpe.encode_packed(b"ab", np.array([0, 2], dtype=np.uint64))
    with pytest.raises(ValueError, match="encode stream is open"):
        bpe.decode_packed(np.array([5], dtype=np.int32), np.array([0, 1], dtype=np.uint64))
    assert L.yttm_enc_stream_end(enc, *refs) == 0, err()
    assert n[0].value == 10
    # a failing sink fails the stream with a message; the stream is closed and the next begin works
    bad = _lib.ENC_SINK(lambda *a: 7)
    with FG.env(YTTM_ENC_STREAM_PIECE_KB=1):
        assert L.yttm_enc_stream_begin(enc, 0, 0, 0, 0.0, 0, 0, _lib.STREAM_IDS32, bad, None) == 0, err()
    data = synth.readme_corpus(n_lines=200)
    rc = L.yttm_enc_stream_feed(enc, data, len(data))
    if rc == 0:
        rc = L.yttm_enc_stream_end(enc, *refs)
    assert rc != 0 and "the sink failed (it returned 7)" in err()
    assert L.yttm_enc_stream_feed(enc, b"x\n", 2) != 0 and "yttm_enc_stream_begin has not run" in err()
    np.testing.assert_array_equal(abi_run(L, bpe, data, 999, 1)[0], expected(bpe, data)[0])
    # an encoder destroyed with an open stream frees it
    other = BPE(model())
    assert L.yttm_enc_stream_begin(L.yttm_api_device_encoder(other._h), 0, 0, 0, 0.0, 0, 0, _lib.STREAM_TEXT, ok,
                                   None) == 0
    assert L.yttm_enc_stream_feed(L.yttm_api_device_encoder(other._h), data, len(data)) == 0
    del other


def failed_calls(L):
    """A failed call raises ValueError naming the path and leaves nothing at the output names."""
    bpe = BPE(model())
    d = tempfile.mkdtemp(dir=_tmp)
    out = os.path.join(d, "out")
    missing = os.path.join(d, "missing.txt")
    with pytest.raises(ValueError, match="missing.txt"):
        bpe.encode_file(missing, out)
    src = write(b"ab cd\n" * 100)
    with pytest.raises(ValueError, match="nodir"):
        bpe.encode_file(src, os.path.join(d, "nodir", "out"))
    with pytest.raises(ValueError, match="needs an output prefix"):
        bpe.encode_file(src, "-")
    with pytest.raises(ValueError, match="dropout_prob"):
        bpe.encode_file(src, out, dropout_prob=1.5)
    with pytest.raises(ValueError, match="Can't add <BOS>"):
        BPE(model("nobos")).encode_file(src, out, bos=True)
    fd = os.open(d, os.O_RDONLY)   # reading a directory fails after the outputs were opened
    try:
        with FG.env(YTTM_ENC_STREAM_PIECE_KB=1):
            with pytest.raises(ValueError, match="cannot read the input"):
                bpe.encode_file(fd, out)
            with pytest.raises(ValueError, match="cannot read the input"):
                bpe.encode_file(fd, out + ".txt", text=True)
    finally:
        os.close(fd)
    assert sorted(os.listdir(d)) == [], os.listdir(d)
    r = bpe.encode_file(src, out)   # the handle works after the failures
    assert r["lines"] == 100 and sorted(os.listdir(d)) == ["out.ids.npy", "out.offsets.npy"]


# ---- GPU tests -------------------------------------------------------------------------------------------------------
@pytest.fixture
def lib(product):
    return product


def test_line_edges(lib):
    edges(lib, (1, 7, None))


def test_bos_eos_reverse(lib):
    flags(lib, 1)


def test_dropout_counter(lib):
    dropout(lib, (1, 7, None))


def test_wide_model_int32(lib):
    wide_ids(lib, 1)


def test_fifo_file_object_and_fd(lib):
    fifo(lib, 1)


def test_abi_blocks(lib):
    abi_blocks(lib)


def test_abi_misuse(lib):
    abi_misuse(lib)


def test_failed_calls_leave_nothing(lib):
    failed_calls(lib)


def _cli(*args, stdin=None):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, "-m", "youtokentome_b200.yttm_cli"] + list(args), input=stdin, cwd=ROOT,
                          env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True)


def test_cli_text_matches_yttm_encode(lib):
    """`yttm encode_file --text` from stdin and from a path gives the stdout of `yttm encode --output_type id`, byte for
    byte; the .npy form loads; the summary goes to stderr."""
    m = model()
    data = edge_cases(small=True)[3][1] + "\n\nhéllo \x0b\n\r\n".encode()
    src = write(data)
    old = _cli("encode", "--model", m, "--output_type", "id", "--bos", stdin=data).stdout
    new = _cli("encode_file", "--model", m, "--input", "-", "--output", "-", "--text", "--bos", stdin=data)
    assert new.stdout == old
    assert b"encode_file: %d lines" % len(lines_of(data)) in new.stderr
    out = os.path.join(tempfile.mkdtemp(dir=_tmp), "t.txt")
    r = _cli("encode_file", "--model", m, "--input", src, "--output", out, "--text", "--bos")
    assert r.stdout == b""
    with open(out, "rb") as f:
        assert f.read() == old
    pre = os.path.join(tempfile.mkdtemp(dir=_tmp), "p")
    _cli("encode_file", "--model", m, "--input", src, "--output", pre, "--bos")
    ids, offs = np.load(pre + ".ids.npy", mmap_mode="r"), np.load(pre + ".offsets.npy", mmap_mode="r")
    assert as_text(np.array(ids), np.array(offs)) == old


def test_device_memory_does_not_grow_with_the_file(lib):
    """configs[1]-shaped files of 64 MB and 512 MB in default (32 MB) pieces: the same device peak."""
    bpe = BPE(model())
    fz = synth.FastZipf(n_words=200_000, seed=1234)
    small = fz.text(64 << 20, words_per_line=20)
    peaks = []
    for data in (small, small * 8):
        src = write(data)
        out = os.path.join(tempfile.mkdtemp(dir=_tmp), "o")
        r = bpe.encode_file(src, out)
        os.remove(src)
        ctx = lib.yttm_api_device_context(bpe._h)
        peaks.append(lib.yttm_stage_ms(ctx, b"stream_dev_peak_bytes"))
        pieces = lib.yttm_stage_ms(ctx, b"stream_pieces")
        print("%d MB: %d lines in %d pieces, device peak %.1f MB" % (len(data) >> 20, r["lines"], pieces,
                                                                      peaks[-1] / 2 ** 20))
        assert pieces >= len(data) // (32 << 20)
        n = np.load(out + ".offsets.npy", mmap_mode="r")
        assert len(n) == r["lines"] + 1 == data.count(b"\n") + 1
    assert peaks[0] == peaks[1], peaks

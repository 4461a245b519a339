"""Decoding files of any size on the GPU (BPE.decode_file, yttm decode_file, yttm_dec_stream_* of yttm_b200.h): ids from
the .npy pair encode_file writes, or id text, are fed in pieces, the id text is parsed on the device, and every line's
text leaves with its '\\n'.  The references are `yttm decode` (the host decode_cli: libstdc++'s own `>> int`),
decode_packed and the reference's decode.

  1. the id-text parser across piece sizes: the grammar of `std::stringstream >> int` at its edges, long lines and digit
     runs, NUL and invalid bytes, random lines of its alphabet, the text form encode_file writes;
  2. round trips through encode_file in both forms, with bos / eos, uint16 and int32 ids, ignore_ids;
  3. inputs and errors: a path, a descriptor, a FIFO, np.save pairs, rejected .npy files, ids outside the vocabulary,
     a failing sink, C ABI misuse;
  4. the device memory bound and 5. the CLI (GPU only).

The bodies take the library: tests/test_decode_file_emul_cpu.py runs 1 - 3 on the SIMT emulator at small sizes."""
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

import test_encode_file_gpu as EF
import test_train_front_gpu as FG
from _bind import ROOT, Reference, have_reference
from youtokentome_b200 import _lib, synth
from youtokentome_b200.youtokentome import BPE

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "*.json")))
_tmp = tempfile.mkdtemp(prefix="yttm_decfile_")
_host = {}
IGN = [-2, -2147483648, -1]   # the negative ids of the cases below: ignored, so that the parser's edges reach decode


def _cli(*args, stdin=None, check=True):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, "-m", "youtokentome_b200.yttm_cli"] + list(args), input=stdin, cwd=ROOT,
                          env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=check)


def host_decode(m, data, ignore=None):
    """`yttm decode` of `data`: (stdout, None) or (None, the error message)."""
    key = (m, data, tuple(ignore or ()))
    if key not in _host:
        args = ["decode", "--model", m] + (["--ignore_ids", ",".join(map(str, ignore))] if ignore else [])
        r = _cli(*args, stdin=data, check=False)
        _host[key] = (r.stdout, None) if r.returncode == 0 else \
            (None, r.stderr.decode().strip().splitlines()[-1].split("ValueError: ", 1)[1])
    return _host[key]


def write(data):
    fd, path = tempfile.mkstemp(dir=_tmp, suffix=".ids")
    with os.fdopen(fd, "wb") as f:
        f.write(data)
    return path


def run_text(bpe, data, piece_kb=None, ignore=None):
    """decode_file(text=True) of `data` from a path -> (output bytes, summary)."""
    src = write(data)
    out = os.path.join(tempfile.mkdtemp(dir=_tmp), "out.txt")
    try:
        with FG.env(**({"YTTM_DEC_STREAM_PIECE_KB": piece_kb} if piece_kb else {})):
            r = bpe.decode_file(src, out, ignore_ids=ignore, text=True)
    finally:
        os.remove(src)
    with open(out, "rb") as f:
        got = f.read()
    assert r["bytes"] == len(got) and r["lines"] == len(EF.lines_of(data))
    return got, r


def check_text(m, data, piece_sizes, ignore=None):
    """decode_file(text=True) equals `yttm decode`, output or error message; a failure leaves no file."""
    bpe = BPE(m)
    want, err = host_decode(m, data, ignore)
    for kb in piece_sizes:
        if err is None:
            got, _ = run_text(bpe, data, kb, ignore)
            assert got == want, (kb, data[:200], got[:300], want[:300])
        else:
            d = tempfile.mkdtemp(dir=_tmp)
            src = write(data)
            with FG.env(**({"YTTM_DEC_STREAM_PIECE_KB": kb} if kb else {})):
                with pytest.raises(ValueError) as e:
                    bpe.decode_file(src, os.path.join(d, "out.txt"), ignore_ids=ignore, text=True)
            os.remove(src)
            assert str(e.value) == err
            assert os.listdir(d) == []


# ---- 1. the id-text parser -------------------------------------------------------------------------------------------
TABLE = [b"1-2", b"+-3", b"12a 4", b"1+", b"0x10", b"1.5 2", b"2147483648 5", b"-2147483648 5",
         b"00000000002147483648 1", b"0" * 33 + b"7 1", b"\t1\r", b"1\x0b2\x0c3", b"5\x00 6"]


def random_lines(rng, n, long=False):
    """Lines of the parser's alphabet: small ids with signs and leading zeros, ignored negatives, int32 edges and
    overflows, whitespace of every kind, stop bytes."""
    out = []
    for _ in range(n):
        parts = []
        for _ in range(int(rng.integers(0, 40 if long else 12))):
            r = rng.random()
            if r < 0.55:
                tok = b"%d" % rng.integers(0, 400)
                z = int(rng.integers(0, 700)) if rng.random() < 0.05 else int(rng.integers(0, 3)) * (rng.random() < 0.2)
                tok = (b"+" if rng.random() < 0.1 else b"") + b"0" * z + tok
            elif r < 0.62:
                tok = rng.choice([b"-1", b"-2", b"-0", b"-00002", b"-2147483648", b"-0000000000002147483648"])
            elif r < 0.68:
                tok = rng.choice([b"2147483647", b"2147483648", b"-2147483649", b"99999999999", b"4294967296",
                                  b"0" * 300 + b"10000000000", b"1" + b"0" * 600])
            elif r < 0.75:
                tok = bytes(rng.choice(list(b"+-ax.,\x00\xff\xc3"), size=int(rng.integers(1, 3))).tolist())
            else:
                tok = b""
            # a digit run across tokens could leave the vocabulary; "1-2" without a separator is in TABLE
            sep = bytes(rng.choice(list(b" \t\x0b\x0c\r"), size=int(rng.integers(1, 3))).tolist())
            parts.append(tok + sep)
        out.append(b"".join(parts))
    return out


def parser_cases(small=False):
    rng = np.random.default_rng(17)
    bpe_text_src = synth.readme_corpus(n_lines=200) + "héllo wörld ▁ 日本語\n".encode() * 5
    long_line = b" ".join(b"%d" % v for v in rng.integers(0, 400, size=(6_000 if small else 600_000)))
    zeros = b"0" * 5000
    return [
        ("table", b"\n".join(TABLE) + b"\n"),
        ("empty", b""),
        ("newline only", b"\n"),
        ("newlines", b"\n\n\n"),
        ("no final newline", b"1 2 3\n4 5\n6 7"),
        ("crlf", b"1 2 3\r\n4 5\r\n\r\n6\r\n"),
        ("whitespace lines", b" \t\x0b\x0c\r\n\r\n  \n"),
        ("line longer than pieces", b"5 6\n" + long_line + b"\n7 8\n" + long_line),
        ("zero runs", zeros + b"7 1\n-" + zeros + b"2147483648 3\n" + zeros + b"2147483648 4\n+" + zeros +
         b"12 5\n" + zeros[:4990] + b"12345678901 2\n" + b"9" + zeros + b" 6\n" + zeros + b"\n"),
        ("nul and invalid bytes", b"5\x00 6\n\xff 5\n5 \xc3\xa9 6\n\x80\n7 \xe2\x96\x81 8\n\x00\n9"),
        ("random", b"\n".join(random_lines(rng, 300 if small else 3000)) + b"\n"),
        ("random long", b"\n".join(random_lines(rng, 20 if small else 200, long=True))),
        ("encode_file text", bpe_text_src),   # replaced by its encode_file(text=True) output in `parser`
    ]


def parser(L, piece_sizes, small=False):
    m = EF.model()
    bpe = BPE(m)
    for name, data in parser_cases(small):
        if name == "encode_file text":
            src = write(data)
            out = os.path.join(tempfile.mkdtemp(dir=_tmp), "enc.txt")
            bpe.encode_file(src, out, text=True, bos=True, eos=True)
            with open(out, "rb") as f:
                data = f.read()
            assert data.endswith(b" \n")
        check_text(m, data, piece_sizes, IGN)
    # ignore sets and errors: the first id outside the vocabulary in file order, with decode's message
    data = b"5 6\n7 400 8 999\n401\n"
    for ign in (None, [400], [400, 999], [400, 999, 401, 5]):
        check_text(m, data, piece_sizes, ign)
    check_text(m, b"1 2\n-5\n", piece_sizes)


# ---- 2. round trips --------------------------------------------------------------------------------------------------
def _golden_lines():
    out = []
    for path in GOLDEN:
        with open(path) as f:
            out += [base64.b64decode(s) for s in json.load(f)["sentences_b64"]]
    return out


def round_trip(bpe, text, piece_kb, ignore=None, **kw):
    """encode_file of `text` in both forms, then decode_file of each: identical, and equal to decode_packed of the
    ids with a '\\n' per line.  Returns the decoded bytes and the ids."""
    src = write(text)
    d = tempfile.mkdtemp(dir=_tmp)
    pre, txt = os.path.join(d, "ids"), os.path.join(d, "ids.txt")
    bpe.encode_file(src, pre, **kw)
    bpe.encode_file(src, txt, text=True, **kw)
    os.remove(src)
    with FG.env(YTTM_DEC_STREAM_PIECE_KB=piece_kb):
        r1 = bpe.decode_file(pre, os.path.join(d, "a.txt"), ignore_ids=ignore)
        r2 = bpe.decode_file(txt, os.path.join(d, "b.txt"), ignore_ids=ignore, text=True)
    with open(os.path.join(d, "a.txt"), "rb") as f, open(os.path.join(d, "b.txt"), "rb") as g:
        a, b = f.read(), g.read()
    assert a == b and r1 == r2
    ids, offs = np.load(pre + ".ids.npy"), np.load(pre + ".offsets.npy")
    t, o = bpe.decode_packed(ids.astype(np.int32), offs, ignore_ids=ignore)
    o = o.astype(np.int64)
    want = b"".join(bytes(t[o[i]:o[i + 1]]) + b"\n" for i in range(len(o) - 1))
    assert a == want
    assert r1 == {"lines": len(offs) - 1, "ids": len(ids), "bytes": len(a)}
    return a, ids, offs


def round_trips(L, piece_kb, small=False):
    m = EF.model()
    bpe = BPE(m)
    golden = _golden_lines()
    gtext = b"\n".join(golden) + b"\n"
    cfg1 = synth.FastZipf(n_words=20_000, seed=5).packed_sentences(300 if small else 5000, 128, seed=9)
    cfg1_text = b"\n".join(cfg1[0][int(a):int(b)] for a, b in zip(cfg1[1][:-1], cfg1[1][1:])) + b"\n"
    for kw in (dict(), dict(bos=True, eos=True), dict(bos=True)):
        out, ids, offs = round_trip(bpe, gtext, piece_kb, **kw)
        assert ids.dtype == np.uint16
        if not kw and have_reference("det"):   # the reference's own decode of the same ids
            ref = Reference("det").encoder(m)
            lines = out.split(b"\n")[:-1]
            for i in range(0, len(golden), max(1, len(golden) // 60)):
                assert lines[i] == ref.decode(ids[offs[i]:offs[i + 1]].tolist()).encode(), i
        round_trip(bpe, cfg1_text, piece_kb, **kw)
    # ignore_ids: specials and frequent pieces, and ids outside int32
    ids = np.load(_encoded(bpe, cfg1_text) + ".ids.npy")
    common = [int(x) for x in np.bincount(ids.astype(np.int64)).argsort()[-3:]]
    for ign in ([2, 3], [2, 3] + common, [2, 3, 2**40, -2**40]):
        round_trip(bpe, cfg1_text, piece_kb, ignore=ign, bos=True, eos=True)
    # int32 ids above 65 535
    wide = BPE(EF.model("wide"))
    chars = "".join(chr(0x10000 + k) for k in range(0, 70_000, 997))
    data = ("ab " + chars + " cd\n" + chars[::-1] + "\nz\n\n").encode() * (5 if small else 50)
    _, wids, _ = round_trip(wide, data, piece_kb)
    assert wids.dtype == np.int32 and wids.max() > 65535


def _encoded(bpe, text, **kw):
    src = write(text)
    pre = os.path.join(tempfile.mkdtemp(dir=_tmp), "ids")
    bpe.encode_file(src, pre, **kw)
    os.remove(src)
    return pre


# ---- 3. inputs and errors --------------------------------------------------------------------------------------------
def inputs(L, piece_kb):
    m = EF.model()
    bpe = BPE(m)
    txt = os.path.join(tempfile.mkdtemp(dir=_tmp), "ids.txt")
    src = write(synth.readme_corpus(n_lines=400))
    bpe.encode_file(src, txt, text=True)
    with open(txt, "rb") as f:
        data = f.read()
    want, _ = host_decode(m, data)
    d = tempfile.mkdtemp(dir=_tmp)
    with FG.env(YTTM_DEC_STREAM_PIECE_KB=piece_kb):
        fd = os.open(txt, os.O_RDONLY)
        try:
            r1 = bpe.decode_file(fd, os.path.join(d, "fd.txt"), text=True)
        finally:
            os.close(fd)
        with open(txt, "rb") as f:
            r2 = bpe.decode_file(f, os.path.join(d, "obj.txt"), text=True)
        fifo = os.path.join(d, "fifo")
        os.mkfifo(fifo)

        def writer():
            with open(fifo, "wb") as f:
                for k in range(0, len(data), 777):
                    f.write(data[k:k + 777])
        t = threading.Thread(target=writer)
        t.start()
        try:
            r3 = bpe.decode_file(fifo, os.path.join(d, "fifo.txt"), text=True)
        finally:
            t.join()
    assert r1 == r2 == r3
    for name in ("fd.txt", "obj.txt", "fifo.txt"):
        with open(os.path.join(d, name), "rb") as f:
            assert f.read() == want, name
    # pairs a user saved with np.save: uint16 and int32 ids, NPY format 1.0 / 2.0 / 3.0
    sents = [[5, 6, 7], [], [8], list(range(4, 300))]
    flat = [i for s in sents for i in s]
    offs = np.cumsum([0] + [len(s) for s in sents]).astype(np.uint64)
    want = b"".join(t.encode() + b"\n" for t in bpe.decode(sents))
    for dt in (np.uint16, np.int32):
        for ver in ((1, 0), (2, 0), (3, 0), None):
            pre = os.path.join(tempfile.mkdtemp(dir=_tmp), "p")
            if ver is None:
                np.save(pre + ".ids.npy", np.array(flat, dtype=dt))
                np.save(pre + ".offsets.npy", offs)
            else:
                for suffix, arr in ((".ids.npy", np.array(flat, dtype=dt)), (".offsets.npy", offs)):
                    with open(pre + suffix, "wb") as f:
                        np.lib.format.write_array(f, arr, version=ver)
            out = pre + ".txt"
            r = bpe.decode_file(pre, out)
            with open(out, "rb") as f:
                assert f.read() == want
            assert r == {"lines": 4, "ids": len(flat), "bytes": len(want)}


def rejected(L):
    """Every .npy pair decode_file does not take fails with a ValueError that names the problem, and leaves no file."""
    bpe = BPE(EF.model())
    ids = np.array([5, 6, 7, 8], dtype=np.int32)
    offs = np.array([0, 2, 4], dtype=np.uint64)

    def case(ids_arr=None, offs_arr=None, ids_raw=None, offs_raw=None):
        d = tempfile.mkdtemp(dir=_tmp)
        pre = os.path.join(d, "p")
        for suffix, arr, raw in ((".ids.npy", ids_arr, ids_raw), (".offsets.npy", offs_arr, offs_raw)):
            if raw is not None:
                with open(pre + suffix, "wb") as f:
                    f.write(raw)
            else:
                np.save(pre + suffix, arr)
        out = os.path.join(d, "out.txt")
        with pytest.raises(ValueError) as e:
            bpe.decode_file(pre, out)
        assert str(e.value).startswith("decode_file:"), str(e.value)
        assert not os.path.exists(out) and not [f for f in os.listdir(d) if f.startswith("out")]
        return str(e.value)

    assert "astype(np.int32)" in case(ids.astype(np.int64), offs)
    assert "'>i4'" in case(ids.astype(">i4"), offs)
    assert "'<f4'" in case(ids.astype(np.float32), offs)
    assert "'<i2'" in case(ids.astype(np.int16), offs)
    assert "not 1-D" in case(ids.reshape(2, 2), offs)
    assert "Fortran" in case(ids_raw=_npy(ids, fortran=True), offs_arr=offs)
    assert "'<i8'" in case(ids, offs.astype(np.int64))
    assert "not 1-D" in case(ids, offs.reshape(1, 3))
    full = _npy(ids)
    assert "truncated" in case(ids_raw=full[:-3], offs_arr=offs)
    assert "truncated" in case(ids_raw=full[:20], offs_arr=offs)
    assert "not an .npy file" in case(ids_raw=b"hello", offs_arr=offs)
    assert "offsets[0]" in case(ids, np.array([1, 2, 4], dtype=np.uint64))
    assert "decrease" in case(ids, np.array([0, 3, 2, 4], dtype=np.uint64))
    assert "past the 4 ids" in case(ids, np.array([0, 2, 5], dtype=np.uint64))
    assert "is not the number of ids" in case(ids, np.array([0, 2, 3], dtype=np.uint64))
    assert "no offsets" in case(ids, np.zeros(0, dtype=np.uint64))
    with pytest.raises(ValueError, match="decode_file: cannot open"):
        bpe.decode_file(os.path.join(_tmp, "missing"), os.path.join(_tmp, "x.txt"))
    with pytest.raises(TypeError):
        bpe.decode_file(os.path.join(_tmp, "missing"), os.path.join(_tmp, "x.txt"), ignore_ids=5)


def _npy(arr, fortran=False):
    hdr = "{'descr': '%s', 'fortran_order': %s, 'shape': (%d,), }" % (arr.dtype.str, fortran, len(arr))
    hdr = hdr + " " * (63 - (len(hdr) + 10) % 64) + "\n"
    return b"\x93NUMPY\x01\x00" + len(hdr).to_bytes(2, "little") + hdr.encode() + arr.tobytes()


def out_of_range(L, piece_kb):
    """Ids of a 32 k-id vocabulary decoded with a 400-id model: decode's message for the first bad id in file order, in
    both forms, and no file; a bad id in a later piece fails as well."""
    bpe = BPE(EF.model())
    rng = np.random.default_rng(3)
    lines = [rng.integers(0, 400, size=int(rng.integers(0, 30))).tolist() for _ in range(3000)]
    lines[2500] = [5, 31999, 7, 401]
    lines[2700] = [1000]
    flat = np.array([i for s in lines for i in s], dtype=np.int32)
    offs = np.cumsum([0] + [len(s) for s in lines]).astype(np.uint64)
    d = tempfile.mkdtemp(dir=_tmp)
    pre = os.path.join(d, "p")
    np.save(pre + ".ids.npy", flat)
    np.save(pre + ".offsets.npy", offs)
    txt = os.path.join(d, "t.ids")
    with open(txt, "wb") as f:
        f.write(b"".join(b"".join(b"%d " % i for i in s) + b"\n" for s in lines))
    msg = "id must be in the range [0, vocab_size - 1]. Current value: vocab_size = 400; id=31999;"
    with FG.env(YTTM_DEC_STREAM_PIECE_KB=piece_kb):
        for args in ((pre, os.path.join(d, "a.txt")), (txt, os.path.join(d, "b.txt"), None, True)):
            with pytest.raises(ValueError) as e:
                bpe.decode_file(*args)
            assert str(e.value) == msg
    assert sorted(os.listdir(d)) == ["p.ids.npy", "p.offsets.npy", "t.ids"]
    r = bpe.decode_file(pre, os.path.join(d, "ok.txt"), ignore_ids=[31999, 401, 1000])   # the handle still works
    assert r["lines"] == 3000


def abi_run(L, bpe, fmt, feeds, piece_kb, ignore=()):
    """yttm_dec_stream_* with a ctypes sink: feeds are byte blocks (text) or (ids, line_ends) -> (text, ends, stats)."""
    enc, ctx = L.yttm_api_device_encoder(bpe._h), L.yttm_api_device_context(bpe._h)
    got, ends = [], []

    def sink(user, ptr, n, le, nl):
        got.append(C.string_at(ptr, n) if n else b"")
        ends.extend(le[k] for k in range(nl))
        return 0
    cb = _lib.ENC_SINK(sink)
    ign = np.asarray(ignore, dtype=np.int32)
    with FG.env(YTTM_DEC_STREAM_PIECE_KB=piece_kb):
        assert L.yttm_dec_stream_begin(enc, fmt, ign.ctypes.data, len(ign), cb, None) == 0, L.yttm_last_error(ctx)
    for f in feeds:
        if fmt == _lib.STREAM_TEXT:
            buf = C.create_string_buffer(f, max(len(f), 1))
            assert L.yttm_dec_stream_feed(enc, buf, len(f)) == 0, L.yttm_last_error(ctx)
            C.memset(buf, 0x0a, len(f))   # the library copied the block
        else:
            ids, le = f
            le = np.ascontiguousarray(le, dtype=np.uint64)
            assert L.yttm_dec_stream_feed_ids(enc, ids.ctypes.data, len(ids), le.ctypes.data, len(le)) == 0, \
                L.yttm_last_error(ctx)
    n = [C.c_uint64(0) for _ in range(3)]
    assert L.yttm_dec_stream_end(enc, *[C.byref(x) for x in n]) == 0, L.yttm_last_error(ctx)
    return b"".join(got), ends, tuple(x.value for x in n), L.yttm_stage_ms(ctx, b"dec_stream_pieces")


def abi(L, small=False):
    """The C ABI fed in odd blocks: text in blocks of 1 - 3000 bytes, ids in groups of lines of every size, in 1 KB
    pieces; the sink's line ends are global byte counts."""
    bpe = BPE(EF.model())
    rng = np.random.default_rng(9)
    lines = [rng.integers(0, 400, size=int(rng.integers(0, 60 if small else 400))).tolist() for _ in range(400)]
    lines[7] = rng.integers(0, 400, size=3000).tolist()   # longer than a piece
    flat = np.array([i for s in lines for i in s], dtype=np.int32)
    offs = np.cumsum([0] + [len(s) for s in lines]).astype(np.uint64)
    texts = [t.encode() + b"\n" for t in bpe.decode(lines, ignore_ids=[5])]
    want, want_ends = b"".join(texts), np.cumsum([len(t) for t in texts]).tolist()
    text = b"".join(b" ".join(b"%d" % i for i in s) + b"\n" for s in lines)
    cuts = np.unique(np.concatenate([[0, len(text)], rng.integers(0, len(text), size=300)]))
    blocks = [text[a:b] for a, b in zip(cuts[:-1], cuts[1:])]
    for fmt, feeds in ((_lib.STREAM_TEXT, blocks), (_lib.STREAM_IDS32, None), (_lib.STREAM_IDS16, None)):
        if feeds is None:
            dt = np.int32 if fmt == _lib.STREAM_IDS32 else np.uint16
            feeds, k = [], 0
            for g in (1, 0, 3, 50, 1, 200, 145):
                g = min(g, len(lines) - k)
                feeds.append((flat[offs[k]:offs[k + g]].astype(dt), offs[k + 1:k + g + 1]))
                k += g
            assert k == len(lines)
        out, ends, n, pieces = abi_run(L, bpe, fmt, feeds, 1, ignore=[5])
        assert out == want and ends == want_ends
        assert n == (len(lines), len(flat), len(want)) and pieces > 2


def abi_misuse(L):
    bpe = BPE(EF.model())
    enc, ctx = L.yttm_api_device_encoder(bpe._h), L.yttm_api_device_context(bpe._h)
    err = lambda: L.yttm_last_error(ctx).decode()   # noqa: E731
    n = [C.c_uint64(0) for _ in range(3)]
    refs = [C.byref(x) for x in n]
    ok = _lib.ENC_SINK(lambda *a: 0)
    one = np.array([5], dtype=np.int32)
    end1 = np.array([1], dtype=np.uint64)
    assert L.yttm_dec_stream_feed(enc, b"5\n", 2) != 0 and "yttm_dec_stream_begin has not run" in err()
    assert L.yttm_dec_stream_feed_ids(enc, one.ctypes.data, 1, end1.ctypes.data, 1) != 0
    assert "yttm_dec_stream_begin has not run" in err()
    assert L.yttm_dec_stream_end(enc, *refs) != 0 and "yttm_dec_stream_begin has not run" in err()
    assert L.yttm_dec_stream_begin(enc, 7, None, 0, ok, None) != 0 and "format must be" in err()
    # an open decode stream owns the encoder: begin again, encode / decode calls and an encode stream fail
    assert L.yttm_dec_stream_begin(enc, _lib.STREAM_TEXT, None, 0, ok, None) == 0, err()
    assert L.yttm_dec_stream_feed(enc, b"5 6\n7", 5) == 0, err()
    assert L.yttm_dec_stream_begin(enc, _lib.STREAM_TEXT, None, 0, ok, None) != 0 and "decode stream is open" in err()
    assert L.yttm_enc_stream_begin(enc, 0, 0, 0, 0.0, 0, 0, _lib.STREAM_IDS32, ok, None) != 0
    assert "decode stream is open" in err()
    with pytest.raises(ValueError, match="decode stream is open"):
        bpe.encode_packed(b"ab", np.array([0, 2], dtype=np.uint64))
    with pytest.raises(ValueError, match="decode stream is open"):
        bpe.decode_packed(np.array([5], dtype=np.int32), np.array([0, 1], dtype=np.uint64))
    assert L.yttm_dec_stream_end(enc, *refs) == 0, err()
    assert [x.value for x in n] == [2, 3, len(bpe.decode([[5, 6]])[0]) + len(bpe.decode([[7]])[0]) + 2]
    # an open encode stream: a decode stream fails
    assert L.yttm_enc_stream_begin(enc, 0, 0, 0, 0.0, 0, 0, _lib.STREAM_IDS32, ok, None) == 0, err()
    assert L.yttm_dec_stream_begin(enc, _lib.STREAM_TEXT, None, 0, ok, None) != 0 and "encode stream is open" in err()
    assert L.yttm_enc_stream_end(enc, *refs) == 0, err()
    # the wrong feed for the format fails and closes the stream
    assert L.yttm_dec_stream_begin(enc, _lib.STREAM_IDS32, None, 0, ok, None) == 0, err()
    assert L.yttm_dec_stream_feed(enc, b"5\n", 2) != 0 and "takes ids" in err()
    assert L.yttm_dec_stream_end(enc, *refs) != 0 and "begin has not run" in err()
    assert L.yttm_dec_stream_begin(enc, _lib.STREAM_TEXT, None, 0, ok, None) == 0, err()
    assert L.yttm_dec_stream_feed_ids(enc, one.ctypes.data, 1, end1.ctypes.data, 1) != 0 and "takes id text" in err()
    # line ends that do not fit the ids fail and close the stream
    assert L.yttm_dec_stream_begin(enc, _lib.STREAM_IDS32, None, 0, ok, None) == 0, err()
    two = np.array([1, 0], dtype=np.uint64)
    assert L.yttm_dec_stream_feed_ids(enc, one.ctypes.data, 1, two.ctypes.data, 2) != 0 and "must not decrease" in err()
    assert L.yttm_dec_stream_begin(enc, _lib.STREAM_IDS32, None, 0, ok, None) == 0, err()
    assert L.yttm_dec_stream_feed_ids(enc, one.ctypes.data, 1, end1.ctypes.data, 1) == 0, err()
    assert L.yttm_dec_stream_feed_ids(enc, one.ctypes.data, 1, end1.ctypes.data, 1) != 0   # must start at 1
    # a failing sink fails the stream with a message; the stream is closed and the next begin works
    bad = _lib.ENC_SINK(lambda *a: 7)
    data = b"5 6 7\n" * 2000
    with FG.env(YTTM_DEC_STREAM_PIECE_KB=1):
        assert L.yttm_dec_stream_begin(enc, _lib.STREAM_TEXT, None, 0, bad, None) == 0, err()
    rc = L.yttm_dec_stream_feed(enc, data, len(data))
    if rc == 0:
        rc = L.yttm_dec_stream_end(enc, *refs)
    assert rc != 0 and "yttm_dec_stream: the sink failed (it returned 7)" in err()
    assert L.yttm_dec_stream_feed(enc, b"x\n", 2) != 0 and "yttm_dec_stream_begin has not run" in err()
    assert abi_run(L, bpe, _lib.STREAM_TEXT, [data], 1)[0] == (bpe.decode([[5, 6, 7]])[0].encode() + b"\n") * 2000
    # an encoder destroyed with an open decode stream frees it
    other = BPE(EF.model())
    oenc = L.yttm_api_device_encoder(other._h)
    assert L.yttm_dec_stream_begin(oenc, _lib.STREAM_TEXT, None, 0, ok, None) == 0
    assert L.yttm_dec_stream_feed(oenc, data, len(data)) == 0
    del other


# ---- GPU tests -------------------------------------------------------------------------------------------------------
@pytest.fixture
def lib(product):
    return product


def test_parser_edges(lib):
    parser(lib, (1, 7, None))


def test_round_trips(lib):
    round_trips(lib, 1)
    round_trips(lib, 32 << 10)


def test_inputs(lib):
    inputs(lib, 1)


def test_rejected_npy(lib):
    rejected(lib)


def test_out_of_range_ids(lib):
    out_of_range(lib, 1)


def test_abi_blocks(lib):
    abi(lib)


def test_abi_misuse(lib):
    abi_misuse(lib)


def test_cli_text_matches_yttm_decode(lib):
    """`yttm decode_file --text` from stdin to stdout prints what `yttm decode` prints; the summary line counts."""
    m = EF.model()
    data = b"\n".join(TABLE) + b"\n\n5 6 7\n" + b" ".join(b"%d" % i for i in range(4, 400)) + b"\n"
    old = _cli("decode", "--model", m, "--ignore_ids", "-2,-2147483648", stdin=data).stdout
    new = _cli("decode_file", "--model", m, "--input", "-", "--output", "-", "--text", "--ignore_ids",
               "-2,-2147483648", stdin=data)
    assert new.stdout == old
    n_ids = 0
    for ln in EF.lines_of(data):   # what the parser reads: the ids of the table and the lines after it
        n_ids += {b"1-2": 2, b"+-3": 0, b"12a 4": 1, b"1+": 1, b"0x10": 1, b"1.5 2": 1, b"2147483648 5": 0,
                  b"-2147483648 5": 2, b"00000000002147483648 1": 0, b"\t1\r": 1, b"1\x0b2\x0c3": 3,
                  b"5\x00 6": 1}.get(ln, len(ln.split()))
    assert new.stderr.decode().strip() == "decode_file: %d lines, %d ids, %d bytes" % (
        len(EF.lines_of(data)), n_ids, len(old))
    r = _cli("decode_file", "--model", m, "--input", "-", "--output", "-", stdin=data, check=False)
    assert r.returncode != 0 and b"--text" in r.stderr


def test_device_memory_does_not_grow_with_the_file(lib):
    """configs[1]-shaped id files of 64 MB and 512 MB in default (32 MB) pieces, the second the first repeated 8 times,
    so that both start with the same pieces: the same device peak, in both forms (one handle per form: the decode
    buffers of an encoder outlive its calls)."""
    rng = np.random.default_rng(1)
    lens = rng.integers(5, 60, size=70_000)
    flat = rng.integers(0, 400, size=int(lens.sum())).astype(np.uint16)
    ends = np.cumsum(lens)
    text = b"".join(b"".join(b"%d " % i for i in flat[a:b]) + b"\n" for a, b in zip(ends - lens, ends))
    reps, tiles = -(-(64 << 20) // len(text)), -(-(64 << 20) // flat.nbytes)
    d = tempfile.mkdtemp(dir=_tmp)
    inputs = {}
    for k in (1, 8):
        src = os.path.join(d, "t%d.ids" % k)
        with open(src, "wb") as f:
            for _ in range(k * reps):
                f.write(text)
        pre = os.path.join(d, "p%d" % k)
        np.save(pre + ".ids.npy", np.tile(flat, k * tiles))
        np.save(pre + ".offsets.npy", np.concatenate([[0], np.cumsum(np.tile(lens, k * tiles))]).astype(np.uint64))
        inputs[k] = {"text": (src, os.path.join(d, "a.txt"), None, True), "npy": (pre, os.path.join(d, "b.txt"))}
    for form in ("text", "npy"):
        bpe = BPE(EF.model())
        ctx = lib.yttm_api_device_context(bpe._h)
        peaks = []
        for k in (1, 8):
            r = bpe.decode_file(*inputs[k][form])
            peaks.append(lib.yttm_stage_ms(ctx, b"dec_stream_dev_peak_bytes"))
            pieces = lib.yttm_stage_ms(ctx, b"dec_stream_pieces")
            print("%s %d lines in %d pieces, device peak %.1f MB" % (form, r["lines"], pieces, peaks[-1] / 2 ** 20))
            assert pieces >= 2 * k
        assert peaks[0] == peaks[1], (form, peaks)
    for name in os.listdir(d):
        os.remove(os.path.join(d, name))

"""Encoding a 1 GB text file on one GPU: BPE.encode_file to .npy and to text, against what a user does without it and
against the plain read / write floor.  The file holds bench.py's configs[1] sentences (seeded synth.FastZipf, 128-byte
sentences, one per line); the vocab 32 000 model is trained the way bench.py trains it (100 MB of the same Zipf text,
on the GPU).  In one run, alternating --reps times, it times
  npy        BPE.encode_file(path, prefix): <prefix>.ids.npy (uint16) + <prefix>.offsets.npy
  text       BPE.encode_file(path, out, text=True): the text of `yttm encode --output_type id`
  today      read the file, find the lines with numpy, encode_packed per 32 MB batch of lines, np.save ids + offsets
  read       the input read in 16 MB blocks and dropped
  write_npy / write_text   plain writes of outputs of the sizes npy / text wrote
and checks that npy, text and today hold the same ids.  The input stays in the page cache after the first pass, and so
does most of what is written, so every row measures the same cached file system.  Prints one JSON line per timing.
    python tools/bench_encode_file.py [--size-gb 1] [--reps 3] [--dir /tmp] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from youtokentome_b200 import synth  # noqa: E402
from youtokentome_b200.youtokentome import BPE  # noqa: E402

BLOCK = 16 << 20
BATCH = 32 << 20


def gpu_name():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT)
    return r.stdout.decode().strip().splitlines()[0]


def write_input(path, n_bytes):
    """configs[1] sentences, one per line, 64 MB of them at a time -> bytes written."""
    fz = synth.FastZipf(n_words=200_000, s=1.07, seed=1234)
    written, k = 0, 0
    with open(path, "wb") as f:
        while written < n_bytes:
            n = max(1, min(n_bytes - written, 64 << 20) // 128)
            buf, offs = fz.packed_sentences(n, 128, seed=4321 + k)
            a = np.frombuffer(buf, dtype=np.uint8).copy()
            a[offs[1:].astype(np.int64) - 1] = 10   # each sentence's trailing space becomes its '\n'
            f.write(a.tobytes())
            written += len(a)
            k += 1
    return written


def today(bpe, path, prefix):
    """What a user does without encode_file: the whole file in memory, lines found with numpy, encode_packed per batch
    of about 32 MB of lines (a line keeps its '\\n', a space byte to the encoder), np.save of ids and offsets."""
    with open(path, "rb") as f:
        a = np.frombuffer(f.read(), dtype=np.uint8)
    bounds = np.concatenate([[0], np.flatnonzero(a == 10) + 1]).astype(np.uint64)   # every line ends with '\\n' here
    n = len(bounds) - 1
    ids, offs, base, lo = [], [np.zeros(1, dtype=np.uint64)], 0, 0
    while lo < n:
        hi = min(max(int(np.searchsorted(bounds, bounds[lo] + BATCH, side="right")) - 1, lo + 1), n)
        i, oo = bpe.encode_packed(a, bounds[lo:hi + 1])
        ids.append(i)
        offs.append(oo[1:] + np.uint64(base))
        base += len(i)
        lo = hi
    np.save(prefix + ".ids.npy", np.concatenate(ids))
    np.save(prefix + ".offsets.npy", np.concatenate(offs))


def plain_read(path):
    with open(path, "rb", buffering=0) as f:
        buf = bytearray(BLOCK)
        while f.readinto(buf):
            pass


def plain_write(path, n):
    blk = bytes(BLOCK)
    with open(path, "wb") as f:
        while n > 0:
            f.write(blk[:min(n, BLOCK)])
            n -= BLOCK


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-gb", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dir", default=tempfile.gettempdir())
    ap.add_argument("--out")
    args = ap.parse_args()
    gpu = gpu_name()
    d = tempfile.mkdtemp(dir=args.dir, prefix="yttm_bench_encfile_")
    src = os.path.join(d, "input.txt")
    size = write_input(src, int(args.size_gb * 2 ** 30))
    from _gpu import gpu_train
    model = gpu_train(synth.FastZipf(n_words=200_000, s=1.07, seed=1234).text(100_000_000), 32_000, 1.0)
    bpe = BPE(model)
    bpe.encode_packed(b"warm up", np.array([0, 7], dtype=np.uint64))
    rows, sizes = [], {}

    def out_path(kind):
        return os.path.join(d, kind)

    def clean():
        for f in os.listdir(d):
            if f != "input.txt":
                os.remove(os.path.join(d, f))

    def timed(kind, rep, fn):
        t = time.perf_counter()
        r = fn()
        wall = time.perf_counter() - t
        row = {"gpu": gpu, "kind": kind, "rep": rep, "bytes": size, "wall_s": round(wall, 3),
               "gb_per_s": round(size / wall / 1e9, 3)}
        if isinstance(r, dict):
            row.update(lines=r["lines"], ids=r["ids"])
        print(json.dumps(row), flush=True)
        rows.append(row)

    for rep in range(args.reps):
        clean()
        timed("npy", rep, lambda: bpe.encode_file(src, out_path("npy")))
        timed("text", rep, lambda: bpe.encode_file(src, out_path("text.txt"), text=True))
        timed("today", rep, lambda: today(bpe, src, out_path("today")))
        timed("read", rep, lambda: plain_read(src))
        if rep == 0:
            ids = np.load(out_path("npy") + ".ids.npy", mmap_mode="r")
            offs = np.load(out_path("npy") + ".offsets.npy", mmap_mode="r")
            assert np.array_equal(np.load(out_path("today") + ".ids.npy", mmap_mode="r"), ids), "npy ids differ"
            assert np.array_equal(np.load(out_path("today") + ".offsets.npy", mmap_mode="r"), offs), "npy offsets differ"
            with open(out_path("text.txt"), "rb") as f:   # spot check of the text form: its first 1000 lines
                head = [f.readline() for _ in range(1000)]
            o = offs[:1001].astype(np.int64)
            assert head == [b"".join(b"%d " % v for v in ids[o[k]:o[k + 1]].tolist()) + b"\n" for k in range(1000)]
            sizes = {"npy": sum(os.path.getsize(out_path("npy") + s) for s in (".ids.npy", ".offsets.npy")),
                     "text": os.path.getsize(out_path("text.txt"))}
        timed("write_npy", rep, lambda: plain_write(out_path("plain_npy"), sizes["npy"]))
        timed("write_text", rep, lambda: plain_write(out_path("plain_text"), sizes["text"]))
    summary = {"gpu": gpu, "bytes": size, "output_bytes": sizes}
    for kind in ("npy", "text", "today", "read", "write_npy", "write_text"):
        w = sorted(r["wall_s"] for r in rows if r["kind"] == kind)
        summary[kind + "_median_s"] = w[len(w) // 2]
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in rows + [summary]))
    clean()
    os.remove(src)
    os.rmdir(d)
    print("bench_encode_file: npy, text and the numpy path hold the same ids")


if __name__ == "__main__":
    main()

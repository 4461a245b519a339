"""Decoding the ids of a 1 GB text file on one GPU: BPE.decode_file from the .npy pair and from the id text, against
what a user does without it and against the plain read / write floor.  The input is bench.py's configs[1] sentences
(seeded synth.FastZipf, 128-byte sentences, one per line, as tools/bench_encode_file.py writes them), encoded by
encode_file into both forms with the vocab 32 000 model trained the way bench.py trains it.  In one run, alternating
--reps times, it times
  npy        BPE.decode_file(prefix, out): <prefix>.ids.npy (uint16) + <prefix>.offsets.npy to text
  text       BPE.decode_file(path, out, text=True): the id text of `yttm encode --output_type id` to text
  today      np.load(mmap) of the pair, decode_packed per 32 MB of ids, a '\\n' after every line, written
  read_npy / read_text   plain reads of the inputs of npy / text, in 16 MB blocks
  write      a plain write of the output's size
and, once, `yttm decode` (the host decode_cli) on a seeded 100 000-line sample of the id text.  It checks that npy, text
and today wrote the same bytes and that `yttm decode` printed the sample's lines of them.  Prints one JSON line per
timing.
    python tools/bench_decode_file.py [--size-gb 1] [--reps 3] [--dir /tmp] [--out FILE]"""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_encode_file import gpu_name, plain_read, plain_write, write_input  # noqa: E402
from youtokentome_b200 import synth  # noqa: E402
from youtokentome_b200.youtokentome import BPE  # noqa: E402

BATCH_IDS = (32 << 20) // 4
SAMPLE = 100_000


def today(bpe, prefix, out):
    """What a user does without decode_file: the pair memory-mapped, decode_packed per 32 MB of int32 ids, a '\\n'
    inserted after every line's text, written."""
    ids = np.load(prefix + ".ids.npy", mmap_mode="r")
    offs = np.load(prefix + ".offsets.npy", mmap_mode="r")
    n = len(offs) - 1
    with open(out, "wb") as f:
        lo = 0
        while lo < n:
            hi = min(max(int(np.searchsorted(offs, offs[lo] + np.uint64(BATCH_IDS), side="right")) - 1, lo + 1), n)
            a, b = int(offs[lo]), int(offs[hi])
            t, o = bpe.decode_packed(np.asarray(ids[a:b], dtype=np.int32), np.asarray(offs[lo:hi + 1]) - np.uint64(a))
            f.write(np.insert(t, o[1:].astype(np.int64), 10).tobytes())
            lo = hi


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-gb", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dir", default=tempfile.gettempdir())
    ap.add_argument("--out")
    args = ap.parse_args()
    gpu = gpu_name()
    d = tempfile.mkdtemp(dir=args.dir, prefix="yttm_bench_decfile_")
    src = os.path.join(d, "input.txt")
    size = write_input(src, int(args.size_gb * 2 ** 30))
    from _gpu import gpu_train
    model = gpu_train(synth.FastZipf(n_words=200_000, s=1.07, seed=1234).text(100_000_000), 32_000, 1.0)
    bpe = BPE(model)
    pre, ids_txt = os.path.join(d, "ids"), os.path.join(d, "ids.txt")
    bpe.encode_file(src, pre)
    bpe.encode_file(src, ids_txt, text=True)
    os.remove(src)
    in_bytes = {"npy": sum(os.path.getsize(pre + s) for s in (".ids.npy", ".offsets.npy")),
                "text": os.path.getsize(ids_txt)}
    bpe.decode_packed(np.array([5], dtype=np.int32), np.array([0, 1], dtype=np.uint64))   # the piece table
    rows, out_size = [], 0

    def out_path(kind):
        return os.path.join(d, "out_" + kind)

    def timed(kind, rep, fn, n_bytes):
        t = time.perf_counter()
        r = fn()
        wall = time.perf_counter() - t
        row = {"gpu": gpu, "kind": kind, "rep": rep, "bytes": n_bytes, "wall_s": round(wall, 3),
               "gb_per_s": round(n_bytes / wall / 1e9, 3)}
        if isinstance(r, dict):
            row.update(lines=r["lines"], ids=r["ids"], out_bytes=r["bytes"])
        print(json.dumps(row), flush=True)
        rows.append(row)

    for rep in range(args.reps):
        for k in ("npy", "text", "today", "write"):
            if os.path.exists(out_path(k)):
                os.remove(out_path(k))
        timed("npy", rep, lambda: bpe.decode_file(pre, out_path("npy")), in_bytes["npy"])
        timed("text", rep, lambda: bpe.decode_file(ids_txt, out_path("text"), text=True), in_bytes["text"])
        timed("today", rep, lambda: today(bpe, pre, out_path("today")), in_bytes["npy"])
        timed("read_npy", rep, lambda: [plain_read(pre + s) for s in (".ids.npy", ".offsets.npy")], in_bytes["npy"])
        timed("read_text", rep, lambda: plain_read(ids_txt), in_bytes["text"])
        if rep == 0:
            out_size = os.path.getsize(out_path("npy"))
            for k in ("text", "today"):
                assert subprocess.run(["cmp", "-s", out_path("npy"), out_path(k)]).returncode == 0, k + " differs"
        timed("write", rep, lambda: plain_write(out_path("write"), out_size), out_size)
    # `yttm decode` on a seeded sample of the id text
    offs = np.load(pre + ".offsets.npy", mmap_mode="r")
    n_lines = len(offs) - 1
    with open(ids_txt, "rb") as f:
        id_lines = f.read().split(b"\n")[:-1]
    with open(out_path("npy"), "rb") as f:
        text_lines = f.read().split(b"\n")[:-1]
    pick = np.sort(np.random.default_rng(7).choice(n_lines, size=min(SAMPLE, n_lines), replace=False))
    sample = b"".join(id_lines[i] + b"\n" for i in pick)
    del id_lines
    env = dict(os.environ, PYTHONPATH=ROOT)
    t = time.perf_counter()
    r = subprocess.run([sys.executable, "-m", "youtokentome_b200.yttm_cli", "decode", "--model", model], input=sample,
                       stdout=subprocess.PIPE, check=True, env=env, cwd=ROOT)
    wall = time.perf_counter() - t
    assert r.stdout == b"".join(text_lines[i] + b"\n" for i in pick), "yttm decode differs"
    row = {"gpu": gpu, "kind": "yttm_decode_sample", "lines": len(pick), "wall_s": round(wall, 3),
           "msent_per_s": round(len(pick) / wall / 1e6, 4), "extrapolated_s": round(wall * n_lines / len(pick), 1)}
    print(json.dumps(row), flush=True)
    rows.append(row)
    summary = {"gpu": gpu, "text_bytes": size, "lines": n_lines, "input_bytes": in_bytes, "output_bytes": out_size}
    for kind in ("npy", "text", "today", "read_npy", "read_text", "write"):
        w = sorted(x["wall_s"] for x in rows if x["kind"] == kind)
        summary[kind + "_median_s"] = w[len(w) // 2]
    summary["yttm_decode_extrapolated_s"] = row["extrapolated_s"]
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in rows + [summary]))
    for fn in os.listdir(d):
        os.remove(os.path.join(d, fn))
    os.rmdir(d)
    print("bench_decode_file: npy, text, the numpy path and yttm decode wrote the same text")


if __name__ == "__main__":
    main()

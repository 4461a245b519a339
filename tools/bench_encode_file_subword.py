"""Encoding a 1 GB text file to subword text on one GPU: BPE.encode_file(output_type=SUBWORD), against the id text form,
the plain read / write floor and `yttm encode --output_type subword`.  The file holds bench.py's configs[1] sentences
(seeded synth.FastZipf, 128-byte sentences, one per line, as tools/bench_encode_file.py writes them); the vocab 32 000
model is trained the way bench.py trains it (100 MB of the same Zipf text, on the GPU).  In one run, alternating --reps
times, it times
  subword     BPE.encode_file(path, out, output_type=SUBWORD): the text of `yttm encode --output_type subword`
  text        BPE.encode_file(path, out, text=True): the text of `yttm encode --output_type id`, for context
  read        the input read in 16 MB blocks and dropped
  write_subword / write_text   plain writes of outputs of the sizes subword / text wrote
  yttm_encode_sample   `yttm encode --output_type subword` (the host piece conversion) on the first 10 000 lines, then
              on the first 100 000 when the first run took at most 30 s; each extrapolated to the whole file (an
              extrapolation, not a measurement of the whole file)
It checks that the subword text of the first 2 000 lines equals the host path (the call behind
encode(output_type=SUBWORD), on the raw bytes) and that `yttm encode` printed the sample's lines of it, and reports the
device peak of both forms.  Prints one JSON line per timing.
    python tools/bench_encode_file_subword.py [--size-gb 1] [--reps 3] [--dir /tmp] [--out FILE]"""
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
from test_encode_file_subword_gpu import framed  # noqa: E402
from test_encode_spans_gpu import host_subwords  # noqa: E402
from youtokentome_b200 import _lib, synth  # noqa: E402
from youtokentome_b200.youtokentome import BPE, OutputType  # noqa: E402

SAMPLE = 100_000
SMALL = 10_000
CLI_LIMIT_S = 300
CHECK = 2_000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-gb", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dir", default=tempfile.gettempdir())
    ap.add_argument("--out")
    args = ap.parse_args()
    gpu = gpu_name()
    d = tempfile.mkdtemp(dir=args.dir, prefix="yttm_bench_encsub_")
    src = os.path.join(d, "input.txt")
    size = write_input(src, int(args.size_gb * 2 ** 30))
    from _gpu import gpu_train
    model = gpu_train(synth.FastZipf(n_words=200_000, s=1.07, seed=1234).text(100_000_000), 32_000, 1.0)
    bpe, bpe_text = BPE(model), BPE(model)   # one handle per form: each reports its own device peak
    bpe.encode_subwords_packed(b"warm up", np.array([0, 7], dtype=np.uint64))   # the piece table
    bpe_text.encode_packed(b"warm up", np.array([0, 7], dtype=np.uint64))
    L = _lib.lib()
    rows, sizes, peaks = [], {}, {}

    def out_path(kind):
        return os.path.join(d, kind)

    def timed(kind, rep, fn, handle=None):
        t = time.perf_counter()
        r = fn()
        wall = time.perf_counter() - t
        row = {"gpu": gpu, "kind": kind, "rep": rep, "bytes": size, "wall_s": round(wall, 3),
               "gb_per_s": round(size / wall / 1e9, 3)}
        if isinstance(r, dict):
            row.update(lines=r["lines"], ids=r["ids"], dev_peak_mb=round(
                L.yttm_stage_ms(L.yttm_api_device_context(handle._h), b"stream_dev_peak_bytes") / 2 ** 20, 1))
            peaks[kind] = row["dev_peak_mb"]
        print(json.dumps(row), flush=True)
        rows.append(row)
        return r

    for rep in range(args.reps):
        for f in os.listdir(d):
            if f != "input.txt":
                os.remove(os.path.join(d, f))
        r = timed("subword", rep, lambda: bpe.encode_file(src, out_path("sub.txt"), output_type=OutputType.SUBWORD), bpe)
        timed("text", rep, lambda: bpe_text.encode_file(src, out_path("text.txt"), text=True), bpe_text)
        timed("read", rep, lambda: plain_read(src))
        if rep == 0:
            n_lines = r["lines"]
            sizes = {"subword": os.path.getsize(out_path("sub.txt")), "text": os.path.getsize(out_path("text.txt"))}
            with open(src, "rb") as f:
                head = [f.readline()[:-1] for _ in range(SAMPLE)]
            with open(out_path("sub.txt"), "rb") as f:
                sub_head = [f.readline() for _ in range(SAMPLE)]
            offs = np.zeros(CHECK + 1, dtype=np.uint64)
            offs[1:] = np.cumsum([len(x) for x in head[:CHECK]])
            want = framed(*host_subwords(bpe, b"".join(head[:CHECK]), offs, {}))
            assert b"".join(sub_head[:CHECK]) == want, "subword text differs from the host path"
        timed("write_subword", rep, lambda: plain_write(out_path("plain_sub"), sizes["subword"]))
        timed("write_text", rep, lambda: plain_write(out_path("plain_text"), sizes["text"]))
    # `yttm encode --output_type subword` on the first SMALL lines, and on the first SAMPLE lines when that is quick
    env = dict(os.environ, PYTHONPATH=ROOT)
    for n in (SMALL, SAMPLE):
        t = time.perf_counter()
        try:
            cli = subprocess.run([sys.executable, "-m", "youtokentome_b200.yttm_cli", "encode", "--model", model,
                                  "--output_type", "subword"], input=b"".join(x + b"\n" for x in head[:n]),
                                 stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True, env=env, cwd=ROOT,
                                 timeout=CLI_LIMIT_S)
        except subprocess.TimeoutExpired:
            row = {"gpu": gpu, "kind": "yttm_encode_sample", "lines": n, "wall_s": None,
                   "note": "did not finish within %d s" % CLI_LIMIT_S}
            print(json.dumps(row), flush=True)
            rows.append(row)
            break
        wall = time.perf_counter() - t
        assert cli.stdout == b"".join(sub_head[:n]), "yttm encode --output_type subword differs"
        row = {"gpu": gpu, "kind": "yttm_encode_sample", "lines": n, "wall_s": round(wall, 3),
               "msent_per_s": round(n / wall / 1e6, 4), "extrapolated_s": round(wall * n_lines / n, 1)}
        print(json.dumps(row), flush=True)
        rows.append(row)
        if wall > 30:
            break
    summary = {"gpu": gpu, "bytes": size, "lines": n_lines, "output_bytes": sizes, "dev_peak_mb": peaks}
    for kind in ("subword", "text", "read", "write_subword", "write_text"):
        w = sorted(x["wall_s"] for x in rows if x["kind"] == kind)
        summary[kind + "_median_s"] = w[len(w) // 2]
    summary["yttm_encode_subword_extrapolated_s"] = row.get("extrapolated_s")
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in rows + [summary]))
    for fn in os.listdir(d):
        os.remove(os.path.join(d, fn))
    os.rmdir(d)
    print("bench_encode_file_subword: encode_file's subword text equals the host path and yttm encode on the samples")


if __name__ == "__main__":
    main()

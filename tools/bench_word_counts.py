"""Word-count tables on one GPU: a synthetic corpus (bench.py's config-3 Zipf generator, --gb GB written to a temporary
file) is counted once with BPE.count_words, then trained from the table (BPE.train_from_counts) and from the text
(BPE.train, fed: YTTM_TRAIN_FEED_ABOVE=0), alternating the two --reps times at vocab 32 000 and once at each of
--vocabs.  Every pair of models must be identical.  Prints one JSON line per measurement.
    python tools/bench_word_counts.py [--gb 1] [--reps 2] [--vocabs 8000,32000,64000] [--out FILE]
load_s = total_s - (tokenise + pair_hist + merge loop): the host time of feed_begin .. feed_end and the alphabet, not
read from a device timer; load GB/s = the input's bytes over load_s (the corpus for the text, word bytes plus 16 bytes
per entry for the table)."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from youtokentome_b200 import synth  # noqa: E402
from youtokentome_b200.youtokentome import BPE, train_report  # noqa: E402


def gpu_name():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT)
    return r.stdout.decode().strip().splitlines()[0]


def write_corpus(path, n_bytes):
    gen = synth.FastZipf(n_words=200_000, s=1.07, seed=1234)
    written, k = 0, 0
    with open(path, "wb") as f:
        while written < n_bytes:
            ask = min(n_bytes - written, 256 << 20)
            t = gen.text(ask, seed=k)
            f.write(t)
            written += len(t)
            k += 1
            if len(t) < ask and ask < 256 << 20:   # a chunk ends with a whole line: the last one comes back short
                break
    return written


def timed_train(kind, src, model, vocab):
    t0 = time.perf_counter()
    if kind == "table":
        BPE.train_from_counts(src, model, vocab)
    else:
        BPE.train(src, model, vocab)
    wall = time.perf_counter() - t0
    r = train_report()
    load_s = r["total_s"] - (r["tokenise_ms"] + r["pair_hist_ms"] + r["merge_loop_ms"]) / 1000
    return wall, load_s, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--vocabs", default="8000,32000,64000")
    ap.add_argument("--out")
    a = ap.parse_args()
    gpu = gpu_name()
    os.environ["YTTM_TRAIN_FEED_ABOVE"] = "0"   # the text is fed as well: both trainings run the same front
    tmp = tempfile.mkdtemp(prefix="yttm_bench_counts_")
    out = open(a.out, "w") if a.out else None

    def emit(d):
        d["gpu"] = gpu
        line = json.dumps(d)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()
    try:
        path = os.path.join(tmp, "corpus.txt")
        n = write_corpus(path, int(a.gb * (1 << 30)))
        BPE.count_words(synth.readme_corpus(n_lines=100))   # warm-up: module load, first allocations
        t0 = time.perf_counter()
        table = BPE.count_words(path)
        count_s = time.perf_counter() - t0
        table_bytes = len(table.word_bytes) + 16 * len(table.counts)
        emit(dict(what="count_words", corpus_bytes=n, count_s=round(count_s, 3), unique=len(table.counts),
                  table_bytes=table_bytes, table_over_corpus=round(table_bytes / n, 5),
                  count_gb_s=round(n / count_s / 1e9, 2)))
        vocabs = [32000] * a.reps + [int(v) for v in a.vocabs.split(",")]
        for i, vocab in enumerate(vocabs):
            models = {}
            for kind, src in (("table", table), ("text", path)):
                models[kind] = os.path.join(tmp, "%s.%d.model" % (kind, i))
                wall, load_s, r = timed_train(kind, src, models[kind], vocab)
                in_bytes = table_bytes if kind == "table" else n
                emit(dict(what="train", kind=kind, vocab=vocab, rep=i, wall_s=round(wall, 3), load_s=round(load_s, 3),
                          load_gb_s=round(in_bytes / load_s / 1e9, 2), merge_loop_ms=round(r["merge_loop_ms"], 1),
                          feed_pieces=int(r["feed_pieces"]), device_peak_mb=round(r["device_peak_bytes"] / 2 ** 20, 1)))
            with open(models["table"], "rb") as f, open(models["text"], "rb") as g:
                assert f.read() == g.read(), "vocab %d: the table's model differs from the text's" % vocab
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        if out:
            out.close()


if __name__ == "__main__":
    main()

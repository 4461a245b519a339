"""Training from a file, in memory and fed, on one GPU: the config-3 Zipf and the config-5 multilingual corpora of
bench.py written to files of 1.25 GB (and of --big-gb GB), each trained by train_bpe in memory (the file read whole,
then loaded) and fed (read in blocks, YTTM_TRAIN_FEED_ABOVE=0, pieces of YTTM_TRAIN_FEED_PIECE_KB), alternating the
two --reps times.  Prints one JSON line per training and asserts that the models are identical.
    python tools/bench_train_feed.py [--big-gb 8] [--reps 2] [--piece-kb 32768] [--out FILE]
ingest_s = total_s - read_s - (tokenise + pair_hist + merge loop): the host time of the byte passes (load + char_hist +
word_count in memory; feed_begin .. feed_end fed), not read from a device timer."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from youtokentome_b200 import _lib, synth  # noqa: E402

REPORT = ["n_bytes", "data_len", "n_words", "n_unique", "n_tokens", "n_pairs", "n_merges", "read_s", "h2d_ms",
          "char_hist_ms", "word_count_ms", "tokenise_ms", "pair_hist_ms", "merge_loop_ms", "total_s", "launches",
          "loop_launches", "feed_pieces", "device_peak_bytes"]
CORPORA = {   # bench.py: config 3 (vocab 32 000) and config 5 (vocab 64 000, coverage 0.9999)
    "config3_zipf": (dict(n_words=200_000, s=1.07, seed=1234), 32_000, 1.0),
    "config5_multilingual": (dict(n_words=300_000, s=1.05, seed=777, mix=synth.CONFIG5_MIX), 64_000, 0.9999),
}


def gpu_name():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT)
    return r.stdout.decode().strip().splitlines()[0]


def write_corpus(path, gen, n_bytes):
    """About n_bytes of text, 256 MB at a time (the generator's arrays stay small) -> the bytes written.  A chunk ends
    with a whole line, a little short of what was asked: the file is complete once a chunk comes back short."""
    written, k = 0, 0
    with open(path, "wb") as f:
        while written < n_bytes:
            ask = min(n_bytes - written, 256 << 20)
            t = gen.text(ask, seed=k)
            f.write(t)
            written += len(t)
            k += 1
            if len(t) < ask and ask < 256 << 20:
                break
    return written


def train(L, path, vocab, cov, fed, piece_kb):
    model = path + (".fed" if fed else ".mem") + ".model"
    for k in ("YTTM_TRAIN_FEED_ABOVE", "YTTM_TRAIN_FEED_PIECE_KB"):
        os.environ.pop(k, None)
    if fed:
        os.environ["YTTM_TRAIN_FEED_ABOVE"] = "0"
        os.environ["YTTM_TRAIN_FEED_PIECE_KB"] = str(piece_kb)
    assert L.yttm_api_train(path.encode(), model.encode(), vocab, cov, 1, 0, 1, 2, 3) == 0, L.yttm_api_last_error(None)
    out = (C.c_double * len(REPORT))()
    n = L.yttm_api_train_report(out, len(REPORT))
    r = dict(zip(REPORT[:n], list(out)[:n]))
    with open(model, "rb") as f:
        return f.read(), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-gb", type=float, default=1.25)
    ap.add_argument("--big-gb", type=float, default=0.0)
    ap.add_argument("--emulate", action="store_true", help="dry run on the CPU SIMT emulator (tiny --size-gb only)")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--piece-kb", type=int, default=32 << 10)
    ap.add_argument("--out")
    ap.add_argument("--dir", default=tempfile.gettempdir())
    args = ap.parse_args()
    if args.emulate:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from _emu import emu_lib
        _lib._lib = emu_lib()
    L = _lib.lib()
    gpu = "emulator" if args.emulate else gpu_name()
    sizes = [int(args.size_gb * 2 ** 30)] + ([int(args.big_gb * 2 ** 30)] if args.big_gb else [])
    lines = []
    for name, (kw, vocab, cov) in CORPORA.items():
        gen = synth.FastZipf(**kw)
        for size in sizes:
            path = os.path.join(args.dir, "yttm_feed_%s_%d.txt" % (name, size))
            size = write_corpus(path, gen, size)
            models = {}
            try:
                for rep in range(args.reps):
                    for fed in (False, True):
                        model, r = train(L, path, vocab, cov, fed, args.piece_kb)
                        models.setdefault(fed, model)
                        assert model == models[fed] and model == models[False], "%s: models differ" % name
                        line = {"gpu": gpu, "corpus": name, "bytes": size, "path": "fed" if fed else "in_memory",
                                "rep": rep, "wall_s": round(r["total_s"], 3), "gb_per_s": round(size / r["total_s"] / 1e9, 3),
                                "read_s": round(r["read_s"], 3),
                                "ingest_s": round(r["total_s"] - r["read_s"] - (r["tokenise_ms"] + r["pair_hist_ms"] +
                                                                                r["merge_loop_ms"]) / 1e3, 3),
                                "tokenise_ms": round(r["tokenise_ms"], 1), "pair_hist_ms": round(r["pair_hist_ms"], 1),
                                "merge_loop_ms": round(r["merge_loop_ms"], 1), "feed_pieces": int(r["feed_pieces"]),
                                "device_peak_mb": round(r["device_peak_bytes"] / 2 ** 20, 1),
                                "piece_kb": args.piece_kb if fed else None, "n_unique": int(r["n_unique"]),
                                "n_merges": int(r["n_merges"])}
                        print(json.dumps(line), flush=True)
                        lines.append(line)
            finally:
                os.remove(path)
    if args.out:
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(x) + "\n" for x in lines))
    print("bench_train_feed: models identical in memory and fed on every corpus")


if __name__ == "__main__":
    main()

"""Padded rows (BPE.encode_padded, yttm_enc_run_padded*) on the configs[1] shape: 1 M synthetic 128-byte sentences
(synth.FastZipf, the seeds of bench.py's workload) and a vocab 32 000 model trained on the GPU, as tools/bench_spans.py
builds it.

    python tools/bench_padded.py [--steps 20] [--warmup 3] [--out DIR]

Prints one JSON line (and writes it to DIR/bench_padded.json) with ms per call (host clock around calls that end in a
synchronise, median over --steps after --warmup calls) of
  device_ids           yttm_enc_run_device (the packed ids), for comparison
  device_padded_64     yttm_enc_run_padded_device at L = 64, ids / ids + spans
  device_padded_32     the same at L = 32, ids (at vocab 32 k no row of this batch reaches 64 ids; rows do reach 32)
  device_padded_auto   the same with L = the longest row (width 0)
  packed_torch_pad_64  yttm_enc_run_device, then the fastest plain-torch padding of the packed ids to the same
                       [N, 64] rows and lengths (a row index per id, one masked scatter); timed alternating with
                       device_padded_64, call by call
  host_padded_64       yttm_enc_run_padded from pinned host buffers into pinned host rows
  gpu                  name and power limit (nvidia-smi, read in the same run)
Before any number is printed, the outputs of the last timed call of each kind are checked against the definition of
tests/test_encode_padded_gpu.py over the packed ids and spans."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

N_SENT, SENT_LEN, VOCAB, TRAIN_BYTES, WIDTH = 1_000_000, 128, 32_000, 100_000_000, 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import youtokentome_b200 as yttm
    import test_encode_padded_gpu as PG
    from _bind import read_model, tmp_model_path
    from _gpu import gpu_train
    from bench_decode import gpu_info
    from youtokentome_b200 import _lib, synth
    from youtokentome_b200.distributed import _DevView
    if not torch.cuda.is_available():
        sys.exit("bench_padded: no CUDA device")
    L = _lib.lib()
    fz = synth.FastZipf(n_words=200_000, s=1.07, seed=1234)
    model = gpu_train(fz.text(TRAIN_BYTES), VOCAB, 1.0, model=tmp_model_path("bench_padded"))
    L.yttm_api_release_training_cache()
    _, pad_id, bos_id, eos_id = read_model(model)[2]
    buf, offs = fz.packed_sentences(N_SENT, SENT_LEN, seed=4321)
    offs = np.asarray(offs).astype(np.uint64)
    bpe = yttm.BPE(model)
    ctx, enc = L.yttm_api_device_context(bpe._h), L.yttm_api_device_encoder(bpe._h)
    dev = torch.device("cuda")
    d_bytes = torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()
    d_offs = torch.from_numpy(offs.astype(np.int64)).cuda()
    pin_bytes = torch.frombuffer(bytearray(buf), dtype=torch.uint8).pin_memory()
    pin_offs = torch.from_numpy(offs.astype(np.int64)).pin_memory()
    pin_rows = torch.empty((N_SENT, WIDTH), dtype=torch.int32).pin_memory()
    pin_len = torch.empty(N_SENT, dtype=torch.int64).pin_memory()
    torch.cuda.synchronize()
    p = [C.c_void_p() for _ in range(3)]
    n1, w = C.c_uint64(0), C.c_uint32(0)
    dev_args = (enc, d_bytes.data_ptr(), d_offs.data_ptr(), len(buf), N_SENT, 0, 0, 0, 0.0, 0, 0)

    def ok(rc):
        assert rc == 0, L.yttm_last_error(ctx)

    def view(ptr, n, ts, shape):
        return torch.as_tensor(_DevView(ptr.value, max(n, 1), ts), device=dev)[:n].view(shape)

    def padded(width, spans):
        ok(L.yttm_enc_run_padded_device(*dev_args, width, pad_id, int(spans), C.byref(p[0]), C.byref(p[1]), C.byref(p[2]),
                                        C.byref(w)))

    def packed():
        ok(L.yttm_enc_run_device(*dev_args, C.byref(p[0]), C.byref(p[1]), C.byref(n1)))

    row_cols = torch.arange(WIDTH, device=dev)

    def packed_torch_pad():
        # the ids stay valid until the next encode call: pad them before anything else runs on the handle
        packed()
        ids = view(p[0], n1.value, "<i4", (n1.value,))
        oo = view(p[1], N_SENT + 1, "<i8", (N_SENT + 1,))
        cnt = oo[1:] - oo[:-1]
        lens = torch.clamp(cnt, max=WIDTH)
        row = torch.repeat_interleave(torch.arange(N_SENT, device=dev), cnt, output_size=n1.value)
        col = torch.arange(n1.value, device=dev) - oo[:-1][row]
        keep = col < WIDTH
        out = torch.full((N_SENT, WIDTH), pad_id, dtype=torch.int32, device=dev)
        out[row[keep], col[keep]] = ids[keep]
        return out, lens

    def host_padded():
        ok(L.yttm_enc_run_padded(enc, pin_bytes.data_ptr(), pin_offs.data_ptr(), N_SENT, 0, 0, 0, 0.0, 0, 0, WIDTH, pad_id,
                                 pin_rows.data_ptr(), pin_len.data_ptr(), None))

    calls = {
        "device_ids": packed,
        "device_padded_64": lambda: padded(WIDTH, False),
        "device_padded_64_spans": lambda: padded(WIDTH, True),
        "device_padded_32": lambda: padded(32, False),
        "device_padded_auto": lambda: padded(0, False),
        "device_padded_auto_spans": lambda: padded(0, True),
        "host_padded_64": host_padded,
    }

    def timed(call):
        t0 = time.perf_counter()
        r = call()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    ms, got = {}, {}
    for name, call in calls.items():
        for _ in range(args.warmup):
            call()
            torch.cuda.synchronize()
        l0 = L.yttm_launch_count(ctx)
        wall = [timed(call)[0] for _ in range(args.steps)]
        ms[name] = {"ms_per_call": round(statistics.median(wall) * 1e3, 3),
                    "launches_per_call": (L.yttm_launch_count(ctx) - l0) / args.steps}
        if name.startswith("device_padded"):
            W = w.value
            r = [view(p[0], N_SENT * W, "<i4", (N_SENT, W)).clone(), view(p[1], N_SENT, "<i8", (N_SENT,)).clone()]
            if name.endswith("spans"):
                r.append(view(p[2], 2 * N_SENT * W, "<i8", (N_SENT, W, 2)).clone())
            got[name] = r
        elif name == "device_ids":
            got[name] = (view(p[0], n1.value, "<i4", (n1.value,)).clone(), view(p[1], N_SENT + 1, "<i8", (N_SENT + 1,)).clone())
        else:
            got[name] = (pin_rows.clone(), pin_len.clone())
    # ---- the new call against packed ids + torch padding, alternated call by call
    for _ in range(args.warmup):
        packed_torch_pad()
        padded(WIDTH, False)
        torch.cuda.synchronize()
    t_new, t_torch = [], []
    for _ in range(args.steps):
        t_torch.append(timed(packed_torch_pad)[0])
        t_new.append(timed(lambda: padded(WIDTH, False))[0])
    torch_rows = packed_torch_pad()
    torch.cuda.synchronize()
    ms["alternated"] = {"device_padded_64_ms": round(statistics.median(t_new) * 1e3, 3),
                        "packed_torch_pad_64_ms": round(statistics.median(t_torch) * 1e3, 3)}

    # ---- the timed outputs against the definition
    ids, oo = got["device_ids"]
    ok(L.yttm_enc_run_spans_device(*dev_args, C.byref(p[0]), C.byref(p[1]), C.byref(p[2]), C.byref(n1)))
    spans = view(p[2], 2 * n1.value, "<i8", (n1.value, 2)).clone()
    d_offs64 = d_offs.clone()
    want = PG.padded_ref(ids, oo, 32, bos_id, eos_id, pad_id)
    assert torch.equal(got["device_padded_32"][0], want[0]) and torch.equal(got["device_padded_32"][1], want[1])
    for name, width in (("device_padded_64", WIDTH), ("device_padded_auto", None)):
        want = PG.padded_ref(ids, oo, width, bos_id, eos_id, pad_id, spans=spans, offs=d_offs64)
        for r in (got[name], got[name + "_spans"]):
            assert torch.equal(r[0], want[0]) and torch.equal(r[1], want[1]), name
        assert torch.equal(got[name + "_spans"][2], want[2]), name
        if width == WIDTH:
            assert torch.equal(torch_rows[0], want[0]) and torch.equal(torch_rows[1], want[1])
            assert torch.equal(got["host_padded_64"][0], want[0].cpu()) and torch.equal(got["host_padded_64"][1],
                                                                                          want[1].cpu())
        else:
            auto_width = int(want[0].shape[1])
        del want
    res = {
        "workload": "encode 1M x 128 B synthetic sentences (FastZipf seed 1234 / 4321), vocab 32k, padded rows",
        "n_sent": N_SENT, "n_ids": int(ids.numel()), "width": WIDTH, "auto_width": auto_width,
        "rows_cut_at_64": int((got["device_padded_64"][1] == WIDTH).sum()),
        "rows_cut_at_32": int((got["device_padded_32"][1] == 32).sum()), "steps": args.steps, "warmup": args.warmup,
        "calls": ms, "gpu": gpu_info(),
        "verified": "every timed output == the padded definition over the packed ids and spans; torch padding and "
                    "host-buffer rows equal too",
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_padded.json"), "w") as f:
            f.write(line + "\n")
    os.remove(model)


if __name__ == "__main__":
    main()

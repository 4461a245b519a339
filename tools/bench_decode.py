"""Decode throughput on the configs[1] shape: 1 M synthetic 128-byte sentences (synth.FastZipf, the seeds of bench.py's
workload), vocab 32 000 model trained on the GPU, ids encoded on the device, then yttm_dec_run_device timed.

    python tools/bench_decode.py [--steps 20] [--warmup 3] [--out DIR]

Prints one JSON line (and writes it to DIR/bench_decode.json):
  device            Msent/s and output GB/s of yttm_dec_run_device (ids and offsets resident in HBM); ms per call from
                    the library's CUDA-event timer "decode" and from a host clock around calls that end in a synchronise;
                    per-stage ms (dec_count / dec_scan / dec_emit) and kernel launches per call
  algo_bytes        4 n_ids + 16 (S + 1) + output bytes, and their rate as a share of an HBM figure that is NOT reached
                    by this code: the H100 SXM data sheet's 3.35 TB/s, or MEASURED_PEAKS.json's hbm_gbs when present
  e2e               yttm_dec_run from pinned host buffers (H2D of ids and offsets, kernels, D2H of text and offsets)
  host_decode       BPE.decode (the host path) on a seeded sample of 50 000 of the sentences: the CPU baseline
  gpu               name and power limit (nvidia-smi, read in the same run)
Before any number is printed the timed output is compared with the numpy oracle of tests/test_decode_gpu.py."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

N_SENT, SENT_LEN, VOCAB, TRAIN_BYTES = 1_000_000, 128, 32_000, 100_000_000
DATASHEET_HBM_GBS = 3350.0


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = [x.strip() for x in out[0].split(",")]
        return {"name": name, "power_limit": power}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return {"name": None, "power_limit": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=50_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import youtokentome_b200 as yttm
    from _bind import tmp_model_path
    from _gpu import gpu_train
    from test_decode_gpu import oracle_decode, piece_table
    from youtokentome_b200 import _lib, synth
    if not torch.cuda.is_available():
        sys.exit("bench_decode: no CUDA device")
    L = _lib.lib()
    fz = synth.FastZipf(n_words=200_000, s=1.07, seed=1234)
    model = gpu_train(fz.text(TRAIN_BYTES), VOCAB, 1.0, model=tmp_model_path("bench_decode"))
    L.yttm_api_release_training_cache()
    buf, offs = fz.packed_sentences(N_SENT, SENT_LEN, seed=4321)
    bpe = yttm.BPE(model)
    ctx, enc = L.yttm_api_device_context(bpe._h), L.yttm_api_device_encoder(bpe._h)
    d_bytes = torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()
    d_offs = torch.from_numpy(np.asarray(offs).astype(np.int64)).cuda()
    torch.cuda.synchronize()
    p_ids, p_ioff, n_ids = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
    assert L.yttm_enc_run_device(enc, d_bytes.data_ptr(), d_offs.data_ptr(), len(buf), N_SENT, 0, 0, 0, 0.0, 0, 0,
                                 C.byref(p_ids), C.byref(p_ioff), C.byref(n_ids)) == 0, L.yttm_last_error(ctx)
    torch.cuda.synchronize()
    n = n_ids.value

    p_text, p_toff, n_text = C.c_void_p(), C.c_void_p(), C.c_uint64(0)

    def dec():
        rc = L.yttm_dec_run_device(enc, p_ids, n, p_ioff, N_SENT, None, 0, C.byref(p_text), C.byref(p_toff), C.byref(n_text))
        assert rc == 0, L.yttm_last_error(ctx)

    for _ in range(args.warmup):
        dec()
    stages = {k: [] for k in ("decode", "dec_count", "dec_scan", "dec_emit")}
    l0 = L.yttm_launch_count(ctx)
    wall = []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        dec()   # returns after a synchronise of the library's stream
        wall.append(time.perf_counter() - t0)
        for k in stages:
            stages[k].append(L.yttm_stage_ms(ctx, k.encode()))
    launches = (L.yttm_launch_count(ctx) - l0) / args.steps
    from youtokentome_b200.distributed import _DevView
    text = torch.as_tensor(_DevView(p_text.value, n_text.value, "|u1"), device="cuda").cpu().numpy()
    toff = torch.as_tensor(_DevView(p_toff.value, N_SENT + 1, "<i8"), device="cuda").cpu().numpy().astype(np.uint64)
    h_ids = torch.as_tensor(_DevView(p_ids.value, n, "<i4"), device="cuda").cpu().numpy()
    h_ioff = torch.as_tensor(_DevView(p_ioff.value, N_SENT + 1, "<i8"), device="cuda").cpu().numpy()

    # ---- the timed output equals the numpy oracle
    tab = piece_table(bpe, model)
    step = 100_000
    for lo in range(0, N_SENT, step):
        t_o, o_o = oracle_decode(tab, h_ids, h_ioff[lo:lo + step + 1])
        a, b = int(toff[lo]), int(toff[lo + step])
        assert np.array_equal(text[a:b], t_o) and np.array_equal(toff[lo:lo + step + 1] - toff[lo], o_o), lo

    # ---- end to end from pinned host buffers
    pin_ids = torch.from_numpy(h_ids).pin_memory()
    pin_off = torch.from_numpy(h_ioff.view(np.uint64).copy().view(np.int64)).pin_memory()
    pin_out = torch.empty(n_text.value + 16, dtype=torch.uint8).pin_memory()
    pin_oo = torch.empty(N_SENT + 1, dtype=torch.int64).pin_memory()
    tot = C.c_uint64(0)

    def e2e():
        rc = L.yttm_dec_run(enc, pin_ids.data_ptr(), pin_off.data_ptr(), N_SENT, None, 0, pin_out.data_ptr(), pin_out.numel(),
                            pin_oo.data_ptr(), C.byref(tot))
        assert rc == 0, L.yttm_last_error(ctx)

    for _ in range(args.warmup):
        e2e()
    e2e_wall = []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        e2e()
        e2e_wall.append(time.perf_counter() - t0)
    assert np.array_equal(pin_out.numpy()[:tot.value], text) and np.array_equal(pin_oo.numpy().view(np.uint64), toff)

    # ---- host decode on a seeded sample (the CPU baseline)
    sample = np.sort(np.random.default_rng(7).choice(N_SENT, args.sample, replace=False))
    lists = [h_ids[h_ioff[i]:h_ioff[i + 1]].tolist() for i in sample]
    t0 = time.perf_counter()
    host = bpe.decode(lists)
    host_s = time.perf_counter() - t0
    assert host == [bytes(text[toff[i]:toff[i + 1]]).decode() for i in sample]

    ms = statistics.median(stages["decode"])
    wall_ms = statistics.median(wall) * 1e3
    out_bytes = int(n_text.value)
    algo = 4 * n + 16 * (N_SENT + 1) + out_bytes
    peak, peak_src = DATASHEET_HBM_GBS, "H100 SXM data sheet (3.35 TB/s), not a reached figure"
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            peak, peak_src = float(json.load(f)["hbm_gbs"]), "MEASURED_PEAKS.json hbm_gbs"
    except (OSError, KeyError, ValueError, TypeError):
        pass
    dev_msent = N_SENT / (ms * 1e-3) / 1e6
    host_msent = args.sample / host_s / 1e6
    res = {
        "workload": "decode 1M x 128 B synthetic sentences (FastZipf seed 1234 / 4321), vocab 32k",
        "n_sent": N_SENT, "n_ids": n, "out_bytes": out_bytes, "steps": args.steps, "warmup": args.warmup,
        "device": {
            "Msent_s": round(dev_msent, 2), "out_GB_s": round(out_bytes / (ms * 1e-3) / 1e9, 2),
            "ms_per_call_events": round(ms, 4), "ms_per_call_wall": round(wall_ms, 4),
            "stage_ms": {k: round(statistics.median(v), 4) for k, v in stages.items()},
            "launches_per_call": launches,
        },
        "algo_bytes": algo,
        "algo_GB_s": round(algo / (ms * 1e-3) / 1e9, 2),
        "share_of_hbm_figure": round(algo / (ms * 1e-3) / 1e9 / peak, 4), "hbm_figure_GB_s": peak, "hbm_figure_source": peak_src,
        "e2e": {"ms_per_call": round(statistics.median(e2e_wall) * 1e3, 3),
                "Msent_s": round(N_SENT / statistics.median(e2e_wall) / 1e6, 2)},
        "host_decode": {"sentences": args.sample, "seconds": round(host_s, 4), "Msent_s": round(host_msent, 4)},
        "device_over_host": round(dev_msent / host_msent, 1),
        "e2e_over_host": round(N_SENT / statistics.median(e2e_wall) / 1e6 / host_msent, 1),
        "gpu": gpu_info(),
        "verified": "timed output == numpy oracle (all sentences); host decode == device text on the sample",
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_decode.json"), "w") as f:
            f.write(line + "\n")
    os.remove(model)


if __name__ == "__main__":
    main()

"""Spans and subwords throughput on the configs[1] shape: 1 M synthetic 128-byte sentences (synth.FastZipf, the seeds of
bench.py's workload) and a vocab 32 000 model trained on the GPU, as tools/bench_decode.py uses.

    python tools/bench_spans.py [--steps 20] [--warmup 3] [--sample 50000] [--out DIR]

Prints one JSON line (and writes it to DIR/bench_spans.json) with ms per call (host clock around calls that end in a
synchronise, median over --steps after --warmup calls) of
  device   ids (yttm_enc_run_device), ids + spans (yttm_enc_run_spans_device), subwords (yttm_enc_run_subwords_device),
           input resident in HBM
  host     the same three from pinned host buffers (yttm_enc_run, yttm_enc_run_spans, yttm_enc_run_subwords)
  host_subwords  BPE.encode(output_type=SUBWORD) (the host path) on a seeded sample of --sample sentences
  gpu      name and power limit (nvidia-smi, read in the same run)
Before any number is printed the timed outputs are checked: the ids of every call equal yttm_enc_run_device's, the
spans of a seeded sample of 3 000 sentences equal the restatement of tests/test_encode_spans_gpu.py, and the pieces of
the --sample sentences equal the host path's."""
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

N_SENT, SENT_LEN, VOCAB, TRAIN_BYTES = 1_000_000, 128, 32_000, 100_000_000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=50_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import youtokentome_b200 as yttm
    import test_encode_spans_gpu as SG
    from _bind import tmp_model_path
    from _gpu import gpu_train
    from bench_decode import gpu_info
    from youtokentome_b200 import _lib, synth
    from youtokentome_b200.distributed import _DevView
    if not torch.cuda.is_available():
        sys.exit("bench_spans: no CUDA device")
    L = _lib.lib()
    fz = synth.FastZipf(n_words=200_000, s=1.07, seed=1234)
    model = gpu_train(fz.text(TRAIN_BYTES), VOCAB, 1.0, model=tmp_model_path("bench_spans"))
    L.yttm_api_release_training_cache()
    buf, offs = fz.packed_sentences(N_SENT, SENT_LEN, seed=4321)
    offs = np.asarray(offs).astype(np.uint64)
    bpe = yttm.BPE(model)
    ctx, enc = L.yttm_api_device_context(bpe._h), L.yttm_api_device_encoder(bpe._h)
    d_bytes = torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()
    d_offs = torch.from_numpy(offs.astype(np.int64)).cuda()
    pin_bytes = torch.frombuffer(bytearray(buf), dtype=torch.uint8).pin_memory()
    pin_offs = torch.from_numpy(offs.astype(np.int64)).pin_memory()
    torch.cuda.synchronize()
    cap = len(buf) + 3 * N_SENT + 16
    bcap = 4 * len(buf) + 10 * N_SENT + 16
    pin_ids = torch.empty(cap, dtype=torch.int32).pin_memory()
    pin_oo = torch.empty(N_SENT + 1, dtype=torch.int64).pin_memory()
    pin_sp = torch.empty((cap, 2), dtype=torch.int64).pin_memory()
    pin_text = torch.empty(bcap, dtype=torch.uint8).pin_memory()
    pin_po = torch.empty(cap + 1, dtype=torch.int64).pin_memory()
    p = [C.c_void_p() for _ in range(3)]
    n1, n2 = C.c_uint64(0), C.c_uint64(0)
    dev_args = (enc, d_bytes.data_ptr(), d_offs.data_ptr(), len(buf), N_SENT, 0, 0, 0, 0.0, 0, 0)
    host_args = (enc, pin_bytes.data_ptr(), pin_offs.data_ptr(), N_SENT, 0, 0, 0, 0.0, 0, 0)

    def ok(rc):
        assert rc == 0, L.yttm_last_error(ctx)

    calls = {
        "device_ids": lambda: ok(L.yttm_enc_run_device(*dev_args, C.byref(p[0]), C.byref(p[1]), C.byref(n1))),
        "device_spans": lambda: ok(L.yttm_enc_run_spans_device(*dev_args, C.byref(p[0]), C.byref(p[1]), C.byref(p[2]),
                                                               C.byref(n1))),
        "device_subwords": lambda: ok(L.yttm_enc_run_subwords_device(*dev_args, C.byref(p[0]), C.byref(p[1]),
                                                                     C.byref(p[2]), C.byref(n1), C.byref(n2))),
        "host_ids": lambda: ok(L.yttm_enc_run(*host_args, pin_ids.data_ptr(), cap, pin_oo.data_ptr(), C.byref(n1))),
        "host_spans": lambda: ok(L.yttm_enc_run_spans(*host_args, pin_ids.data_ptr(), cap, pin_oo.data_ptr(),
                                                      pin_sp.data_ptr(), C.byref(n1))),
        "host_subwords": lambda: ok(L.yttm_enc_run_subwords(*host_args, pin_text.data_ptr(), bcap, pin_po.data_ptr(), cap,
                                                            pin_oo.data_ptr(), C.byref(n1), C.byref(n2))),
    }

    def dev_copy(ptr, n, ts):
        return torch.as_tensor(_DevView(ptr.value, max(n, 1), ts), device="cuda")[:n].cpu().numpy()

    ms, out = {}, {}
    for name, call in calls.items():
        for _ in range(args.warmup):
            call()
            torch.cuda.synchronize()
        l0 = L.yttm_launch_count(ctx)
        wall = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            call()
            torch.cuda.synchronize()
            wall.append(time.perf_counter() - t0)
        ms[name] = {"ms_per_call": round(statistics.median(wall) * 1e3, 3),
                    "Msent_s": round(N_SENT / statistics.median(wall) / 1e6, 2),
                    "launches_per_call": (L.yttm_launch_count(ctx) - l0) / args.steps}
        # what the last timed call returned
        if name == "device_ids":
            out[name] = (dev_copy(p[0], n1.value, "<i4"), dev_copy(p[1], N_SENT + 1, "<i8"))
        elif name == "device_spans":
            out[name] = (dev_copy(p[0], n1.value, "<i4"), dev_copy(p[1], N_SENT + 1, "<i8"),
                         dev_copy(p[2], 2 * n1.value, "<i8").reshape(-1, 2))
        elif name == "device_subwords":
            out[name] = (dev_copy(p[0], n2.value, "|u1"), dev_copy(p[1], n1.value + 1, "<i8"),
                         dev_copy(p[2], N_SENT + 1, "<i8"))
        elif name == "host_ids":
            out[name] = (pin_ids.numpy()[:n1.value].copy(), pin_oo.numpy().copy())
        elif name == "host_spans":
            out[name] = (pin_ids.numpy()[:n1.value].copy(), pin_oo.numpy().copy(), pin_sp.numpy()[:n1.value].copy())
        else:
            out[name] = (pin_text.numpy()[:n2.value].copy(), pin_po.numpy()[:n1.value + 1].copy(), pin_oo.numpy().copy())

    # ---- the timed outputs
    ids, oo = out["device_ids"]
    for k in ("host_ids", "device_spans", "host_spans"):
        assert np.array_equal(out[k][0], ids) and np.array_equal(out[k][1], oo), k
    assert np.array_equal(out["device_spans"][2], out["host_spans"][2])
    for a, b in zip(out["device_subwords"], out["host_subwords"]):
        assert np.array_equal(a, b)
    assert np.array_equal(out["device_subwords"][2], oo)
    spans = out["device_spans"][2].astype(np.uint64)
    m = SG.Model(model)
    raw = bytes(buf)
    rng = np.random.default_rng(11)
    for s in np.sort(rng.choice(N_SENT, 3000, replace=False)):
        a, b = int(offs[s]), int(offs[s + 1])
        want = SG.oracle_spans(m, raw[a:b], ids[oo[s]:oo[s + 1]], a, False, False, False)
        assert [tuple(x) for x in spans[oo[s]:oo[s + 1]].tolist()] == want, s
    text, po, _ = out["device_subwords"]
    sample = np.sort(np.random.default_rng(7).choice(N_SENT, args.sample, replace=False))
    from _bind import _pack
    s_data, s_offs = _pack([raw[int(offs[i]):int(offs[i + 1])] for i in sample])
    t0 = time.perf_counter()
    h_text, h_po, h_so = SG.host_subwords(bpe, s_data, s_offs, {})   # encode(output_type=SUBWORD)'s host call
    host_s = time.perf_counter() - t0
    sel = np.concatenate([np.arange(oo[i], oo[i + 1]) for i in sample]).astype(np.int64)
    got = b"".join(bytes(text[po[j]:po[j + 1]]) for j in sel)
    assert got == h_text and np.array_equal(np.diff(po.astype(np.int64))[sel], np.diff(h_po.astype(np.int64)))

    res = {
        "workload": "encode 1M x 128 B synthetic sentences (FastZipf seed 1234 / 4321), vocab 32k",
        "n_sent": N_SENT, "n_ids": int(len(ids)), "piece_bytes": int(len(text)), "steps": args.steps,
        "warmup": args.warmup, "calls": ms,
        "spans_over_ids": {k: round(ms[k + "_spans"]["ms_per_call"] / ms[k + "_ids"]["ms_per_call"], 3)
                           for k in ("device", "host")},
        "host_subwords": {"sentences": args.sample, "seconds": round(host_s, 4),
                          "Msent_s": round(args.sample / host_s / 1e6, 4)},
        "device_subwords_over_host": round(ms["device_subwords"]["Msent_s"] / (args.sample / host_s / 1e6), 1),
        "gpu": gpu_info(),
        "verified": "ids of every call == yttm_enc_run_device; spans == restatement on 3000 sentences; pieces == host "
                    "encode(SUBWORD) on the sample; device == host-buffer results",
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_spans.json"), "w") as f:
            f.write(line + "\n")
    os.remove(model)


if __name__ == "__main__":
    main()

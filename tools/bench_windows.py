"""Overlapping windows (BPE.encode_windows, yttm_enc_run_windows_device) against the paths a user has without it, with a
vocab 32 000 model trained on the GPU as tools/bench_padded.py builds it.

    python tools/bench_windows.py [--steps 20] [--warmup 3] [--out DIR]

Two workloads, all inputs and results on the device:
  (a) the configs[1] shape: 1 M synthetic 128-byte sentences (synth.FastZipf, the seeds of bench.py's workload) at
      L = 64, S = 0.  No sentence of this batch reaches 64 ids, so every sentence is one window and the rows equal
      encode_padded's.  Timed alternating call by call: windows, yttm_enc_run_padded_device at L = 64 and
      yttm_enc_run_device (the packed ids).
  (b) long documents: 4 000 sentences of about 32 KB at L = 512, S = 128, ids and ids + spans.  Timed alternating call
      by call: windows, and yttm_enc_run_device / yttm_enc_run_spans_device followed by the fastest plain-torch
      windowing of the packed ids (and spans): a row index per window by repeat_interleave, one gather of [W, L] cells.
Prints one JSON line (and writes it to DIR/bench_windows.json) with ms per call (host clock around calls that end in a
synchronise, median over --steps after --warmup calls of every kind), launches per call, and the GPU's name and power
limit (nvidia-smi, read in the same run).  Before any number is printed, the output of the last timed call of each kind
is checked against the definition of tests/test_encode_windows_gpu.py over the packed ids and spans."""
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

VOCAB, TRAIN_BYTES = 32_000, 100_000_000
A_SENT, A_LEN, A_WIDTH = 1_000_000, 128, 64
B_SENT, B_LEN, B_WIDTH, B_STRIDE = 4_000, 32_768, 512, 128


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import youtokentome_b200 as yttm
    import test_encode_windows_gpu as WG
    from _bind import read_model, tmp_model_path
    from _gpu import gpu_train
    from bench_decode import gpu_info
    from youtokentome_b200 import _lib, synth
    from youtokentome_b200.distributed import _DevView
    if not torch.cuda.is_available():
        sys.exit("bench_windows: no CUDA device")
    L = _lib.lib()
    fz = synth.FastZipf(n_words=200_000, s=1.07, seed=1234)
    model = gpu_train(fz.text(TRAIN_BYTES), VOCAB, 1.0, model=tmp_model_path("bench_windows"))
    L.yttm_api_release_training_cache()
    _, pad_id, bos_id, eos_id = read_model(model)[2]
    bpe = yttm.BPE(model)
    ctx, enc = L.yttm_api_device_context(bpe._h), L.yttm_api_device_encoder(bpe._h)
    dev = torch.device("cuda")
    p = [C.c_void_p() for _ in range(5)]
    n_out, rows, w = C.c_uint64(0), C.c_uint64(0), C.c_uint32(0)

    def ok(rc):
        assert rc == 0, L.yttm_last_error(ctx)

    def view(ptr, n, ts, shape):
        return torch.as_tensor(_DevView(ptr.value, max(n, 1), ts), device=dev)[:n].view(shape)

    def alternate(calls, got):
        """Every call of `calls` (name -> fn) in turn, --steps rounds after --warmup: ms per call and launches per call.
        got[name] = a copy of what the call returned in its last timed run, taken after the clock stopped (the
        library's results live until the next encode call)."""
        for _ in range(args.warmup):
            for call in calls.values():
                call()
                torch.cuda.synchronize()
        t = {k: [] for k in calls}
        launches = {k: 0 for k in calls}
        for _ in range(args.steps):
            for k, call in calls.items():
                l0 = L.yttm_launch_count(ctx)
                t0 = time.perf_counter()
                r = call()
                torch.cuda.synchronize()
                t[k].append(time.perf_counter() - t0)
                launches[k] += L.yttm_launch_count(ctx) - l0
                got[k] = [x.clone() for x in r] if r is not None else None
        return {k: {"ms_per_call": round(statistics.median(v) * 1e3, 3), "launches_per_call": launches[k] / args.steps}
                for k, v in t.items()}

    def batch(n, length, seed):
        buf, offs = fz.packed_sentences(n, length, seed=seed)
        offs = np.asarray(offs).astype(np.uint64)
        d_bytes = torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()
        d_offs = torch.from_numpy(offs.astype(np.int64)).cuda()
        return d_bytes, d_offs, (enc, d_bytes.data_ptr(), d_offs.data_ptr(), len(buf), n, 0, 0, 0, 0.0, 0, 0)

    def windows(dev_args, n, width, stride, spans):
        ok(L.yttm_enc_run_windows_device(*dev_args, width, stride, pad_id, int(spans), *[C.byref(x) for x in p],
                                         C.byref(rows)))
        W = rows.value
        r = [view(p[0], W * width, "<i4", (W, width))] + [view(p[i], W, "<i8", (W,)) for i in (1, 2, 3)]
        return r + ([view(p[4], 2 * W * width, "<i8", (W, width, 2))] if spans else [])

    def packed(dev_args, n, spans):
        if spans:
            ok(L.yttm_enc_run_spans_device(*dev_args, C.byref(p[0]), C.byref(p[1]), C.byref(p[2]), C.byref(n_out)))
        else:
            ok(L.yttm_enc_run_device(*dev_args, C.byref(p[0]), C.byref(p[1]), C.byref(n_out)))
        k = n_out.value
        return ([view(p[0], k, "<i4", (k,)), view(p[1], n + 1, "<i8", (n + 1,))] +
                ([view(p[2], 2 * k, "<i8", (k, 2))] if spans else []))

    def torch_windows(dev_args, d_offs, n, width, stride, spans):
        # the packed results stay valid until the next encode call: window them before anything else runs on the handle
        r = packed(dev_args, n, spans)
        ids, oo = r[0], r[1]
        D = width - stride
        cnt = oo[1:] - oo[:-1]
        nw = torch.where(cnt <= width, 1, 1 + (cnt - width + D - 1).clamp(min=0) // D)
        first = torch.cumsum(nw, 0) - nw
        W = int(first[-1] + nw[-1])
        sent = torch.repeat_interleave(torch.arange(n, device=dev), nw, output_size=W)
        start = (torch.arange(W, device=dev) - first[sent]) * D
        lens = torch.clamp(cnt[sent] - start, max=width)
        src = oo[:-1][sent][:, None] + start[:, None] + torch.arange(width, device=dev)[None, :]
        keep = torch.arange(width, device=dev)[None, :] < lens[:, None]
        src = torch.where(keep, src, 0)
        out = [torch.where(keep, ids[src], pad_id), lens, sent, start]
        if spans:
            hi = d_offs[1:][sent][:, None, None]
            out.append(torch.where(keep[..., None], r[2][src], hi))
        return out

    res = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup}
    # ---- (a) the configs[1] shape
    d_bytes, d_offs, dev_args = batch(A_SENT, A_LEN, 4321)
    got = {}
    res["a"] = alternate({
        "windows_64": lambda: windows(dev_args, A_SENT, A_WIDTH, 0, False),
        "padded_64": lambda: ok(L.yttm_enc_run_padded_device(*dev_args, A_WIDTH, pad_id, 0, C.byref(p[0]), C.byref(p[1]),
                                                             C.byref(p[2]), C.byref(w))),
        "packed_ids": lambda: packed(dev_args, A_SENT, False),
    }, got)
    ok(L.yttm_enc_run_padded_device(*dev_args, A_WIDTH, pad_id, 0, C.byref(p[0]), C.byref(p[1]), C.byref(p[2]),
                                    C.byref(w)))
    pad_rows = [view(p[0], A_SENT * A_WIDTH, "<i4", (A_SENT, A_WIDTH)).clone(), view(p[1], A_SENT, "<i8", (A_SENT,)).clone()]
    want = WG.windows_ref(got["packed_ids"][0], got["packed_ids"][1], A_WIDTH, 0, bos_id, eos_id, pad_id)
    assert all(torch.equal(a, b) for a, b in zip(got["windows_64"], want[:4]))
    assert torch.equal(got["windows_64"][0], pad_rows[0]) and torch.equal(got["windows_64"][1], pad_rows[1])
    assert int(got["windows_64"][0].shape[0]) == A_SENT
    res["a"].update(n_sent=A_SENT, n_ids=int(got["packed_ids"][0].numel()), width=A_WIDTH, stride=0,
                    longest_row=int(pad_rows[1].max()))
    del d_bytes, d_offs, got, want, pad_rows
    torch.cuda.empty_cache()
    # ---- (b) long documents
    d_bytes, d_offs, dev_args = batch(B_SENT, B_LEN, 99)
    got = {}
    res["b"] = alternate({
        "windows": lambda: windows(dev_args, B_SENT, B_WIDTH, B_STRIDE, False),
        "packed_torch": lambda: torch_windows(dev_args, d_offs, B_SENT, B_WIDTH, B_STRIDE, False),
        "windows_spans": lambda: windows(dev_args, B_SENT, B_WIDTH, B_STRIDE, True),
        "packed_torch_spans": lambda: torch_windows(dev_args, d_offs, B_SENT, B_WIDTH, B_STRIDE, True),
    }, got)
    ids, oo, sp = packed(dev_args, B_SENT, True)
    want = WG.windows_ref(ids, oo, B_WIDTH, B_STRIDE, bos_id, eos_id, pad_id, spans=sp, offs=d_offs)
    for name in ("windows", "packed_torch", "windows_spans", "packed_torch_spans"):
        assert all(torch.equal(a, b) for a, b in zip(got[name], want)), name
    res["b"].update(n_sent=B_SENT, n_bytes=int(d_offs[-1]), n_ids=int(ids.numel()), rows=int(want[0].shape[0]),
                    width=B_WIDTH, stride=B_STRIDE)
    res["workload"] = ("(a) 1M x 128 B FastZipf sentences (seed 1234 / 4321), L = 64, S = 0; (b) 4000 x 32 KB "
                       "(seed 99), L = 512, S = 128; vocab 32k")
    res["verified"] = ("every timed output == the windows definition over the packed ids and spans; (a) also == "
                       "encode_padded at L = 64")
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_windows.json"), "w") as f:
            f.write(line + "\n")
    os.remove(model)


if __name__ == "__main__":
    main()

"""A/B of the encode kernels' variants on the bench workload (run on one GPU):
    python tools/ab_encode.py [n_sentences] [reps] [result.json] [model file]
For each of {default, YTTM_ENC_PLAIN (the round-1 kernels), plain + one variant, ...}: median CUDA-event ms of find / words / gather
over `reps` runs of yttm_enc_run_device on inputs resident in HBM, and a check that the ids are identical."""
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402


def main(L=None, n_sent=None, reps=None, train_bytes=20_000_000, vocab=8000):
    import torch
    from youtokentome_b200 import _lib, synth
    from _gpu import gpu_train
    L = L or _lib.lib()
    n_sent = n_sent or (int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000)
    reps = reps or (int(sys.argv[2]) if len(sys.argv) > 2 else 7)
    fz = synth.FastZipf(n_words=200_000, s=1.07, seed=1234)
    if len(sys.argv) > 4:  # an existing model file (bench.py passes its 32 k model: the bench configuration exactly)
        model = sys.argv[4]
    else:
        model = gpu_train(fz.text(train_bytes), vocab, 1.0)
    buf, offs = fz.packed_sentences(n_sent, 128, seed=4321)
    h = L.yttm_api_open(model.encode(), 1)
    assert h, L.yttm_api_last_error(None)
    ctx, enc = L.yttm_api_device_context(h), L.yttm_api_device_encoder(h)
    assert ctx and enc, "no device encoder: " + (L.yttm_last_error(None) or b"").decode()
    on_gpu = torch.cuda.is_available()
    if on_gpu:
        from youtokentome_b200.distributed import _DevView
    d_bytes = torch.frombuffer(bytearray(buf), dtype=torch.uint8)
    d_offs = torch.from_numpy(offs.astype(np.int64))
    if on_gpu:
        d_bytes, d_offs = d_bytes.cuda(), d_offs.cuda()
    base = None
    out = {}
    KNOBS = ("YTTM_ENC_PLAIN", "YTTM_ENC_SLOTS", "YTTM_ENC_FIND_CACHED", "YTTM_ENC_BUCKETED", "YTTM_ENC_ZLIN", "YTTM_ENC_DEDUP", "YTTM_ENC_FIND_VEC", "YTTM_ENC_LONG")
    # default since round 2 = vector word finder + word dedup + block-per-long-word; "plain" = the round-1 kernels
    for name, env in [("default", []), ("slots", ["YTTM_ENC_SLOTS"]), ("plain", ["YTTM_ENC_PLAIN"]), ("plain+find_vec", ["YTTM_ENC_PLAIN", "YTTM_ENC_FIND_VEC"]),
                      ("plain+dedup", ["YTTM_ENC_PLAIN", "YTTM_ENC_DEDUP"]), ("bucketed", ["YTTM_ENC_BUCKETED"]),
                      ("dedup+find_cached", ["YTTM_ENC_FIND_CACHED"])]:
        for k in KNOBS:
            os.environ.pop(k, None)
        for k in env:
            os.environ[k] = "1"
        ms = {"enc_find": [], "enc_words": [], "enc_gather": [], "encode": []}
        if name in ("default", "slots", "plain+dedup", "dedup+find_cached"):  # the launches inside enc_words
            ms.update({"enc_dedup": [], "enc_rep": [], "enc_copy": [], "enc_count": []})
        for _ in range(reps + 2):
            p_ids, p_off, n = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
            rc = L.yttm_enc_run_device(enc, d_bytes.data_ptr(), d_offs.data_ptr(), len(buf), n_sent, 0, 0, 0, 0.0, 0, 0,
                                       C.byref(p_ids), C.byref(p_off), C.byref(n))
            assert rc == 0, L.yttm_last_error(ctx)
            for k in ms:
                ms[k].append(L.yttm_stage_ms(ctx, k.encode()))
        if on_gpu:
            torch.cuda.synchronize()
            from youtokentome_b200.distributed import _DevView
            ids = torch.as_tensor(_DevView(p_ids.value, n.value, "<i4"), device="cuda").cpu().numpy()
        else:  # emulated library: "device" memory is host memory
            ids = np.ctypeslib.as_array(C.cast(p_ids, C.POINTER(C.c_int32)), shape=(n.value,)).copy()
        if base is None:
            base = ids
        same = bool(np.array_equal(base, ids))
        out[name] = {k: statistics.median(v[2:]) for k, v in ms.items()}
        out[name]["ids_equal_default"] = same
        out[name]["n_ids"] = int(n.value)
    # BASELINE config 4 encodes with dropout_prob = 0.1: the default kernels' stage times there (ids are random by design)
    for k in KNOBS:
        os.environ.pop(k, None)
    ms = {"enc_find": [], "enc_words": [], "enc_gather": [], "encode": []}
    for r in range(reps + 2):
        p_ids, p_off, n = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
        rc = L.yttm_enc_run_device(enc, d_bytes.data_ptr(), d_offs.data_ptr(), len(buf), n_sent, 0, 0, 0, 0.1, 1234 + r, 0,
                                   C.byref(p_ids), C.byref(p_off), C.byref(n))
        assert rc == 0, L.yttm_last_error(ctx)
        for k in ms:
            ms[k].append(L.yttm_stage_ms(ctx, k.encode()))
    out["default_dropout_0.1"] = {k: statistics.median(v[2:]) for k, v in ms.items()}
    out["default_dropout_0.1"]["n_ids"] = int(n.value)
    L.yttm_api_close(h)
    # host-only knob: slots per rule of the encoder's rule table (default 2), read when the encoder is created
    for slots in (4, 8, 16):
        os.environ["YTTM_ENC_RULE_SLOTS"] = str(slots)
        h2 = L.yttm_api_open(model.encode(), 1)
        assert h2, L.yttm_api_last_error(None)
        ctx2, enc2 = L.yttm_api_device_context(h2), L.yttm_api_device_encoder(h2)
        ms = {"enc_find": [], "enc_words": [], "enc_gather": [], "encode": []}
        for _ in range(reps + 2):
            p_ids, p_off, n = C.c_void_p(), C.c_void_p(), C.c_uint64(0)
            rc = L.yttm_enc_run_device(enc2, d_bytes.data_ptr(), d_offs.data_ptr(), len(buf), n_sent, 0, 0, 0, 0.0, 0, 0,
                                       C.byref(p_ids), C.byref(p_off), C.byref(n))
            assert rc == 0, L.yttm_last_error(ctx2)
            for k in ms:
                ms[k].append(L.yttm_stage_ms(ctx2, k.encode()))
        if on_gpu:
            torch.cuda.synchronize()
            ids = torch.as_tensor(_DevView(p_ids.value, n.value, "<i4"), device="cuda").cpu().numpy()
        else:
            ids = np.ctypeslib.as_array(C.cast(p_ids, C.POINTER(C.c_int32)), shape=(n.value,)).copy()
        out["rule_slots_%d" % slots] = {k: statistics.median(v[2:]) for k, v in ms.items()}
        out["rule_slots_%d" % slots]["ids_equal_default"] = bool(np.array_equal(base, ids))
        out["rule_slots_%d" % slots]["n_ids"] = int(n.value)
        L.yttm_api_close(h2)
    os.environ.pop("YTTM_ENC_RULE_SLOTS", None)
    print(json.dumps(out, indent=1))
    if len(sys.argv) > 3:  # optional: also write the result to a file
        with open(sys.argv[3], "w") as fh:
            json.dump(out, fh, indent=1)
    return out


if __name__ == "__main__":
    main()

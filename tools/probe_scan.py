"""Probe: per-iteration scan of a synthetic packed token buffer >> L2 (STREAMING tiles via TMA)."""
import ctypes as C, sys, os, json
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from youtokentome_b200 import _lib
L = _lib.lib()
T = int(float(sys.argv[1])) if len(sys.argv) > 1 else 256 * 1024 * 1024
wl = int(sys.argv[2]) if len(sys.argv) > 2 else 8
iters = int(sys.argv[3]) if len(sys.argv) > 3 else 12
alpha = 2000
log2_first = int(sys.argv[4]) if len(sys.argv) > 4 else 0   # 0: every word starts with the same token (heavy merges)
n_first = 1 << log2_first
c2 = C.c_void_p(); assert L.yttm_ctx_create(0, C.byref(c2)) == 0
assert L.yttm_train_synth_words(c2, T // wl, wl, alpha | (log2_first << 24), 7) == 0, L.yttm_last_error(c2)
rules = np.zeros(3 * iters, dtype=np.uint32); fr = np.zeros(iters, dtype=np.uint64); nd = C.c_uint32(0)
assert L.yttm_train_run(c2, 4 + n_first + alpha, iters, rules.ctypes.data, fr.ctypes.data, C.byref(nd)) == 0, L.yttm_last_error(c2)
g = lambda k: L.yttm_stage_ms(c2, k.encode())
it = max(g("loop_iters"), 1.0)
t_scan = (g("loop_apply") + g("loop_partition") + g("loop_drain")) / it
ab = 4 * T + 4 * (T // wl)
print(json.dumps({"log2_first": log2_first, "T": T, "wl": wl, "iters": int(nd.value), "resident": g("loop_resident"), "ms_scan": t_scan,
                  "GBps": ab / (t_scan * 1e-3) / 1e9, "frac_of_3350": ab / (t_scan * 1e-3) / 1e9 / 3350.0,
                  "phase_ms": {k: g(k) / it for k in ["loop_elect", "loop_apply", "loop_partition", "loop_drain"]},
                  "rules_head": rules[:6].tolist(), "freq_head": fr[:2].tolist()}))
L.yttm_ctx_destroy(c2)

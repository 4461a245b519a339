"""bench.py's control flow and the JSON-line contract, checked without a GPU: tools/bench_dryrun_emulated.py runs
bench.main() unchanged on the CPU emulator build of the kernels (torch.cuda stubbed, workload shrunk).  The numbers are
meaningless here; the keys, their types and the internal consistency of the line are what the driver depends on."""
import json
import math
import os
import subprocess
import sys

import pytest

from _bind import ROOT, have_reference


def _half_unit_4g(x):
    """Half a unit in the 4th significant digit of x: the most a value printed as "%.4g" is off."""
    return 0.5 * 10.0 ** (math.floor(math.log10(abs(x))) - 3)


def test_bench_line_contract_on_the_emulator(tmp_path):
    env = dict(os.environ, YTTM_BENCH_CACHE=str(tmp_path / "cache"))
    for k in [k for k in env if k.startswith(("YTTM_ENC_", "YTTM_LOOP_"))]:
        env.pop(k)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_dryrun_emulated.py")], cwd=ROOT, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, r.stderr.decode(errors="replace")[-2000:]
    lines = [ln for ln in r.stdout.decode().splitlines() if ln.strip()]
    assert len(lines) == 1, "stdout must carry exactly ONE line"
    d = json.loads(lines[0])
    for k, t in (("metric", str), ("value", float), ("unit", str), ("n_gpus", int), ("steps", int), ("warmup", int),
                 ("ms_per_step", float), ("higher_is_better", bool), ("scaling", str), ("dtype", str), ("data", str),
                 ("config", dict), ("e2e", dict), ("gpu_launches", int), ("clocks", dict), ("roofline", dict),
                 ("cpu_baseline", dict)):
        assert isinstance(d[k], t), (k, d[k])
    assert d["vs_baseline"] is None and d["n_gpus"] == 1 and d["steps"] == 2 and d["warmup"] >= 3 and d["gpu_launches"] > 0
    assert "workload" in d["config"] and "model" not in d["config"]
    assert set(d["e2e"]) >= {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} and d["e2e"]["h2d_bytes_per_step"] > 0
    rf = d["roofline"]
    assert set(rf) >= {"bound", "achieved", "peak", "unit", "frac", "traffic"} and rf["bound"] == "hbm"
    # frac is achieved / peak: both are printed to 4 significant digits, so some rate must round to `achieved` while
    # that rate / peak rounds to `frac` (a fixed absolute tolerance fails at random once the rate reaches 0.01 GB/s)
    a, f, p = rf["achieved"], rf["frac"], rf["peak"]
    ha, hf = _half_unit_4g(a) * (1 + 1e-12), _half_unit_4g(f) * (1 + 1e-12)
    assert a > 0 and f > 0 and (a - ha) / p <= f + hf and (a + ha) / p >= f - hf, (a, f, p)
    cb = d["cpu_baseline"]
    assert set(cb) >= {"value", "unit", "cores", "kind", "sample"} and cb["kind"] in ("reference", "port") and cb["ids_equal_on_sample"]
    assert abs(d["ms_per_step"] * d["value"] / 1e3 - d["config"]["sentences_per_gpu"] / 1e6) < 1e-6   # value = S / t
    # hot path (a) travels in keys the driver keeps: config.train.* and roofline.train_*
    tr = d["config"]["train"]
    assert set(tr) >= {"config1", "config3", "config5"}
    with_reference = have_reference("det") and have_reference("prod")   # bench.py's parity legs run the reference itself
    for key in ("config3", "config5"):
        leg = tr[key]
        assert leg["gpus"] == 1 and leg["merges"] > 0 and leg["GBps"] > 0 and leg["us_per_merge"] > 0 and len(leg["model_sha1"]) == 12
        if with_reference:
            assert leg["parity_chunk0"]["equals_reference"] is True
    if with_reference:
        assert tr["config1"]["equals_reference"] is True
    assert set(rf["train_scan"]) >= {"heavy", "light", "algorithmic_bytes_per_merge"} and rf["train_scan"]["heavy"]["frac"] > 0
    assert set(rf["train_front"]) >= {"char_hist_GBps", "word_count_GBps"}
    e4 = d["config"]["encode_config4"]
    assert e4["dropout"] == 0.1 and e4["ids_equal_oracle_on_sample"] is True and e4["Msent_s_device"] > 0
    assert d["e2e"]["pageable_value"] > 0 and set(cb) >= {"n_threads_1"} | ({"train_1GB_8thr"} if with_reference else set())
    assert len(lines[0]) < 8000, "the line must stay small enough for the driver's retained tail"


def test_reference_arm_line_contract(tmp_path, checkers):
    """`bench.py --impl reference` (the unmodified reference's CPU encode_as_ids from oracle/_ref, no GPU involved)."""
    if not checkers.have_reference("prod"):
        pytest.skip("oracle/_ref not built: the reference arm times the reference library itself")
    env = dict(os.environ, YTTM_BENCH_CACHE=str(tmp_path / "cache"))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, r.stderr.decode(errors="replace")[-2000:]
    lines = [ln for ln in r.stdout.decode().splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "Msent/s" and d["higher_is_better"] is True and d["value"] > 0
    assert d["metric"] == "encode throughput, 1M x 128 B synthetic sentences, vocab 32k"
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = d["cpu_baseline"]
    assert cb["kind"] == "reference" and cb["cores"] >= 1 and cb["value"] == d["value"] and cb["sample"]
    assert cb["steps_s"]["min"] <= cb["steps_s"]["median"] <= cb["steps_s"]["max"]
    assert d["config"]["workload"] == "configs[1]: encode 1M synthetic 128-byte sentences, vocab 32k"

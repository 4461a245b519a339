"""Every selectable kernel variant on real hardware against the ORACLE (runs last: zzz).  tools/sanitize_small.py in a
subprocess with a hard timeout: tiny trainings (RESIDENT and forced STREAMING, roomy and tiny exchange segments /
table partitions) and encodes with the default kernels (vector word finder + word dedup + block-per-long-word), the
round-1 kernels (YTTM_ENC_PLAIN) and every opt-in variant, each compared with the oracle inside the script.  A
difference, a crash or a hang FAILS (round 1 could only xfail here)."""
import json
import os
import subprocess
import sys

import pytest

from _bind import ROOT

pytestmark = pytest.mark.gpu


def _clean_env():
    return {k: v for k, v in os.environ.items() if not k.startswith(("YTTM_ENC_", "YTTM_LOOP_", "YTTM_FORCE_", "YTTM_STREAM_",
                                                                         "YTTM_STAGES", "YTTM_XQ_", "YTTM_PAIR_"))}


def test_every_variant_matches_the_oracle(product):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sanitize_small.py")], cwd=ROOT, env=_clean_env(),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=420)
    text = r.stdout.decode(errors="replace")
    assert r.returncode == 0 and "checks identical to the oracle" in text, text[-2000:]


def test_encode_variants_return_the_default_ids_on_the_bench_shape(product, tmp_path):
    """tools/ab_encode.py on a 200 k-sentence cut of the bench workload: ids of every variant == the default kernels'."""
    out_json = tmp_path / "ab.json"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ab_encode.py"), "200000", "3", str(out_json)], cwd=ROOT,
                       env=_clean_env(), stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, timeout=420)
    assert r.returncode == 0 and out_json.exists(), r.stderr.decode(errors="replace")[-1500:]
    res = json.loads(out_json.read_text())
    assert res["default"]["n_ids"] > 0 and set(res) >= {"default", "slots", "plain", "plain+find_vec", "plain+dedup", "bucketed"}
    bad = [k for k, v in res.items() if not v.get("ids_equal_default", True)]
    assert not bad, "variants differ from the default ids on hardware: %s" % bad

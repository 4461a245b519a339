"""compute-sanitizer over tools/sanitize_small.py on the GPU box (SURVEY 8f-4, second half; the reference's own
sanitizer job: tests/unit_tests/test_stress.py:19-30).  memcheck and synccheck must report 0 errors; racecheck must
report no ERROR-severity hazard (its WARNING-severity reports are the two documented benign ones of process_tile —
merge_loop.cuh: a warp re-reads a word that another warp may be rewriting and then competes for the word's claim bit;
a stale read only costs a no-op rewrite).  Every result of the workload is also compared with the oracle inside the
script.  A report, a crash or a timeout FAILS; a sanitizer that refuses the device (where the driver does not let it
attach) skips.  Runs last (zzz)."""
import os
import re
import shutil
import subprocess
import sys

import pytest

from _bind import ROOT

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tool", ["memcheck", "synccheck", "racecheck"])
def test_sanitizer(product, tool):
    exe = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(exe):
        pytest.skip("compute-sanitizer is not installed")
    env = {k: v for k, v in os.environ.items() if not k.startswith(("YTTM_", "YT_EMU_"))}
    env["YTTM_SANITIZE_QUICK"] = "1"   # the tools slow kernels down 10 - 100 x: the short form of the workload
    r = subprocess.run([exe, "--tool", tool, sys.executable, os.path.join(ROOT, "tools", "sanitize_small.py")], cwd=ROOT,
                       env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
    text = r.stdout.decode(errors="replace")
    if "Error: Device not supported" in text:
        pytest.skip("compute-sanitizer does not support this device here")
    assert "checks identical to the oracle" in text, text[-1500:]
    if tool == "racecheck":
        m = re.search(r"RACECHECK SUMMARY: (\d+) hazards? displayed \((\d+) errors?, (\d+) warnings?\)", text)
        assert m and int(m.group(2)) == 0, text[-1500:]
        bad = [ln for ln in text.splitlines() if "Race reported" in ln and "process_tile" not in ln and "warp_apply_word" not in ln]
        assert not bad, bad[:3]
    else:
        assert "ERROR SUMMARY: 0 errors" in text, text[-1500:]

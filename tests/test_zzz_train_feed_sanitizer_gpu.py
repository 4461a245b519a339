"""compute-sanitizer memcheck and racecheck over tools/sanitize_train_feed.py (fed trainings: small pieces, misaligned
blocks, table and arena growth).  Any report fails, and so does a result that differs from the restatement; a
sanitizer that refuses the device (where the driver does not let it attach) skips.  Runs last (zzz)."""
import os
import re
import shutil
import subprocess
import sys

import pytest

from _bind import ROOT

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_sanitizer_fed_training(product, tool):
    exe = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(exe):
        pytest.skip("compute-sanitizer is not installed")
    env = {k: v for k, v in os.environ.items() if not k.startswith(("YTTM_", "YT_EMU_"))}
    r = subprocess.run([exe, "--tool", tool, sys.executable, os.path.join(ROOT, "tools", "sanitize_train_feed.py")],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=900)
    text = r.stdout.decode(errors="replace")
    if "Error: Device not supported" in text:
        pytest.skip("compute-sanitizer does not support this device here")
    assert "checks identical to the restatement" in text, text[-1500:]
    if tool == "racecheck":
        m = re.search(r"RACECHECK SUMMARY: (\d+) hazards? displayed", text)
        assert m and int(m.group(1)) == 0, text[-1500:]
    else:
        assert "ERROR SUMMARY: 0 errors" in text, text[-1500:]

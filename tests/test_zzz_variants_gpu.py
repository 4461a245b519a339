"""Every selectable kernel variant on real hardware against the ORACLE (runs last: zzz).  tools/sanitize_small.py in a
subprocess with a hard timeout: tiny trainings (RESIDENT and forced STREAMING, roomy and tiny exchange segments /
table partitions) and encodes (vector word finder + word dedup + block-per-long-word, and the dropout kernel), each
compared with the oracle inside the script.  A difference, a crash or a hang FAILS."""
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


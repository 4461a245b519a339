"""The reference's OWN stress test (tests/unit_tests/stress_test.cpp, compiled unmodified against include/compat by
oracle/Makefile -> oracle/_ref/ref_stress_b200, linked with libyttm_b200.so) on the GPU: its asserts compare
learn_bpe_from_string with its learn_bpe_slow spec, encode_as_ids / encode_as_subwords with its decode_slow spec, batch
with single-sentence encoding, and the decode round trip (stress_test.cpp:313-493).  Runs last (zz)."""
import os
import subprocess

import pytest

from _bind import ROOT

pytestmark = pytest.mark.gpu
BIN = os.path.join(ROOT, "oracle", "_ref", "ref_stress_b200")


@pytest.mark.parametrize("args", [["manual"], ["base", "40"], ["parallel", "4"]])
def test_reference_stress_binary(product, tmp_path, args):
    if not os.path.exists(BIN):
        pytest.skip("oracle/_ref/ref_stress_b200 not built (needs /root/reference at build time)")
    r = subprocess.run([BIN] + args, cwd=tmp_path, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, r.stderr.decode(errors="replace")[-2000:]

"""The warp-specialised prefill kernel (csrc/prefill_ws.cu, selected with B200_PREFILL=ws) through the same prefill parity
tests as the default kernel: against the oracle (packed, paged prefix + chunk, block sizes, long causal with repeated
rescales, stale / neighbouring rows) and against flash-attn.  The library reads the switch once per process, so the tests
run in a child pytest with the variable set."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("poly", ["1", "0"])
def test_prefill_parity_suite_under_the_warp_specialised_kernel(poly):
    env = dict(os.environ, B200_PREFILL="ws", B200_PREFILL_POLY=poly)
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu", "-k", "prefill",
           os.path.join(ROOT, "tests", "test_gpu_kernels.py"), os.path.join(ROOT, "tests", "test_gpu_zz_flash_attn_parity.py")]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and " failed" not in r.stdout, r.stdout[-2000:]

"""GPU check of the tensor-parallel linear layer's choice between the fused GEMM + collective kernels and the GEMM followed by the
stand-alone collective, on ONE H100 with 2 virtual ranks: forward and backward in the reduce-scatter-out, SP-gather, all-reduce-out
and all-reduce-dgrad modes, fusion forced on and switched off.  Outputs and gradients within test_gpu_fused.py's bound of fp32
torch; ``n_fused`` shows which path ran.  tests/_linear_paths_worker.py runs the cases in a process of its own, because the harness
needs CUDA modules loaded eagerly from the start (see there)."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

from _linear_paths_worker import EXPECT_FUSED, MODES  # noqa: E402


@pytest.fixture(scope="module")
def results():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    proc = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "_linear_paths_worker.py")], capture_output=True, text=True,
                          timeout=550)
    out = proc.stdout + proc.stderr
    print(out[-6000:])
    assert proc.returncode == 0 and "LINEAR_DONE" in proc.stdout, out[-6000:]
    recs = [json.loads(ln[len("LINEAR_CASE "):]) for ln in proc.stdout.splitlines() if ln.startswith("LINEAR_CASE ")]
    return {(r["mode"], r["fused"]): r for r in recs}


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "unfused"])
@pytest.mark.parametrize("mode", MODES)
def test_linear_path(results, mode, fused):
    rec = results[(mode, fused)]
    assert rec["n_fused"] == [EXPECT_FUSED[mode] if fused else {}] * 2, rec
    assert rec["out_excess"] <= 0 and rec["dx_excess"] <= 0 and rec["dw_excess"] <= 0, rec

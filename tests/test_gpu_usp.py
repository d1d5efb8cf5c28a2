"""GPU checks of Ulysses and zigzag context parallelism on the same layer.

* The composed attention (``ulysses_cp_attention``), forward and backward, with sp x cp virtual ranks on one H100 at Llama-3.2-1B
  head shapes, (sp, cp) = (2, 2) at S = 8k, (2, 4) and (4, 2) at 16k, under both cp exchanges, against ONE flash-attn call on the
  natural-order sequence with the ring test's bounds (output and dq rel-L2 1e-2, dk / dv 2e-2), and the ring's merged LSE on the
  heads a rank holds after the exchange (max abs 1e-3).  tests/_usp_gpu_worker.py runs them in a process of its own, because the
  harness needs CUDA modules loaded eagerly from the start (see there).
* The strategies of tests/test_usp.py end to end through the CUDA path (skipped below the 4 or 8 GPUs they need)."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

from _usp_gpu_worker import ATTN_CASES, LSE_CASES  # noqa: E402


@pytest.fixture(scope="module")
def usp_results():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    proc = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "_usp_gpu_worker.py")], capture_output=True, text=True,
                          timeout=1100)
    out = proc.stdout + proc.stderr
    print(out[-6000:])
    assert proc.returncode == 0 and "USP_DONE" in proc.stdout, out[-6000:]
    recs = [json.loads(ln[len("USP_CASE "):]) for ln in proc.stdout.splitlines() if ln.startswith("USP_CASE ")]
    return {(r["kind"], r["sp"], r["cp"], r["S"], r["comm"]): r for r in recs}


@pytest.mark.parametrize("sp,cp,S,comm", ATTN_CASES, ids=["sp%d-cp%d-S%d-%s" % c for c in ATTN_CASES])
def test_usp_attention_matches_flash(usp_results, sp, cp, S, comm):
    obs = usp_results[("attention", sp, cp, S, comm)]
    assert obs["out_rel_l2"] < 1e-2 and obs["dq_rel_l2"] < 1e-2, obs
    assert obs["dk_rel_l2"] < 2e-2 and obs["dv_rel_l2"] < 2e-2, obs
    assert (obs["ring_pushes"] > 0) == (comm == "ring"), obs


@pytest.mark.parametrize("sp,cp,S", LSE_CASES, ids=["sp%d-cp%d-S%d" % c for c in LSE_CASES])
def test_usp_ring_lse_matches_flash(usp_results, sp, cp, S):
    obs = usp_results[("lse", sp, cp, S, "ring")]
    assert obs["lse_max_abs"] < 1e-3, obs


# ---- the strategies end to end --------------------------------------------------------------------------------------------
def _cases():
    from test_usp import PARAMS
    return PARAMS


@pytest.mark.parametrize("name,comm", _cases(), ids=["%s-%s" % p for p in _cases()])
def test_usp_strategy_cuda(name, comm):
    from test_usp import CASES, launch
    world, cfg = CASES[name]
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    rep = launch(world, dict(cfg), comm, backend="cuda")
    assert rep["max_grad_err"] < 3e-2
    if comm == "ring":
        assert rep["ring_pushes"] > 0

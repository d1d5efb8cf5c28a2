"""fp parity pinned to the REFERENCE RUNTIME, not only to HF: tests/golden/ref_runtime/<case>.json holds the per-step losses the
UNMODIFIED reference (PKU-DAIR/Hetu-Galvatron runtime: FSDP + Megatron layers + flash-attn, run on GPUs by
oracle/ref_runtime/run_ref.py) computes for 3 Adam steps of the tiny Llama of tests/golden/ckpt_llama_tiny under a parallel
strategy.  This repo's runtime, given the same weights (the same converted checkpoint), the same token stream and the same
optimizer, must reproduce them: the loss of step 0 (pure forward) and of the later steps (which fold in every gradient through
the optimizer) and, at every step, the norm of all gradient tensors of the job -- CPU host runtime within 1e-4 / 3e-4 / 3e-3
(observed 7e-6 / 4e-5 / 6e-4: both sides compute in bf16 with fp32 reductions and fp32 cross-entropy, as the reference's own
tests configure it, tests/utils/runtime_args.py:60-62), GPU product path within 2e-4 / 3e-4 / 3e-3 (north_star asks for 1e-3, the reference's own criterion against HF is 5e-3, tests/core/test_tp.py:121).
CPU: the host runtime on the oracle backend.  GPU (``-m gpu``): the product path through the C ABI."""
import glob
import json
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_host_runtime import launch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "ckpt_llama_tiny")
FIXTURES = {os.path.basename(p)[:-5]: json.load(open(p)) for p in sorted(glob.glob(os.path.join(HERE, "golden", "ref_runtime", "*.json")))}


def _ours(fx, backend):
    over = {k: (bool(v) if k in ("sequence_parallel", "use_ulysses") else v) for k, v in fx["overrides"].items()}
    cfg = dict(over, load=GOLDEN, adam_weight_decay=0.0, lr=1e-3, reduce_in_fp32=bool(fx.get("reduce_in_fp32", 0)), _iters=fx["steps"], _tol=float("inf") if backend == "cuda" else 3e-2)
    return launch(fx["world"], cfg, backend=backend)


def _check(fx, rep, tol_step0, tol_later, tol_gnorm):
    ref, got = fx["losses"], rep["losses"]
    assert len(got) == len(ref)
    dl = [abs(a - b) / abs(b) for a, b in zip(got, ref)]
    dg = [abs(a - b) / abs(b) for a, b in zip(rep["grad_norms_all_ranks"], fx["grad_norms_all_ranks"])]
    assert dl[0] <= tol_step0, (ref, got)
    assert max(dl[1:]) <= tol_later, (ref, got)
    assert ref[-1] < ref[0] or fx["steps"] < 3            # the reference run itself trains
    # every gradient of the job, as the optimizers of the two runtimes see them (shards once, replicas once per holder)
    assert max(dg) <= tol_gnorm, (fx["grad_norms_all_ranks"], rep["grad_norms_all_ranks"])


@pytest.mark.skipif(not FIXTURES, reason="no reference-runtime fixtures committed")
@pytest.mark.parametrize("case", sorted(FIXTURES) or ["none"])
def test_host_runtime_matches_reference_runtime(case):
    fx = FIXTURES[case]
    if fx["world"] > 4:
        pytest.skip("large world")
    _check(fx, _ours(fx, "oracle"), 1e-4, 3e-4, 3e-3)        # observed: 7e-6, 4e-5, 6e-4


@pytest.mark.gpu
@pytest.mark.skipif(not FIXTURES, reason="no reference-runtime fixtures committed")
@pytest.mark.parametrize("case", sorted(FIXTURES) or ["none"])
def test_product_path_matches_reference_runtime(case):
    fx = FIXTURES[case]
    if not torch.cuda.is_available() or torch.cuda.device_count() < fx["world"]:
        pytest.skip("needs %d GPU(s)" % fx["world"])
    _check(fx, _ours(fx, "cuda"), 2e-4, 3e-4, 3e-3)

"""Tied input / output embeddings (C14) of the GPT family across pipeline stages, on the CPU over gloo, against the HF-pinned oracle
(loss 5e-3 rel, per-parameter gradients 3e-2 rel-L2, one AdamW step; the worker also asserts that the two copies of the matrix are
bit-identical after construction and after the step).  The forms the reference's own pipeline corpus runs GPT in
(tests/core/test_pp.py: pp 2 and pp 4, both schedules, tied), and the optimizer / gradient-precision variants whose gradient path
differs: the fused optimizer's deferred norm and step passes, and fp32 gradient buffers."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
_PORT = [33300]


def launch(world, config, timeout=900, backend="oracle"):
    from _launch import launch_ranks
    _PORT[0] += 1
    return launch_ranks("_tied_worker", world, config, _PORT[0] + os.getpid() % 500, timeout=timeout, backend=backend)


TIED = dict(_family="gpt", untie_embeddings_and_output_weights=False)

CASES = {
    "gpt_tied_pp4_gpipe_chunks8": (4, dict(TIED, _spec=dict(n_layer=4), pp_deg=4, chunks=8, pipeline_type="gpipe", global_train_batch_size=8)),
    "gpt_tied_pp4_1f1b_chunks8": (4, dict(TIED, _spec=dict(n_layer=4), pp_deg=4, chunks=8, pipeline_type="pipedream_flush", global_train_batch_size=8)),
    # the fused optimizer consumes the gradient inside the reduce-scatter: no gradient tensor to compare, the step is checked
    "gpt_tied_pp2_fused_clip": (2, dict(TIED, pp_deg=2, chunks=2, fused_optimizer=True, clip_grad=1.0, _tol=float("inf"))),
    "gpt_tied_pp2_reduce_fp32": (2, dict(TIED, pp_deg=2, chunks=2, reduce_in_fp32=True)),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_tied_across_stages(name):
    world, cfg = CASES[name]
    rep = launch(world, dict(cfg))
    assert rep["tied"]
    assert rep["max_grad_err"] < cfg.get("_tol", 3e-2)
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])

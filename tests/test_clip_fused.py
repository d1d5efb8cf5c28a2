"""Gradient clipping with the fused optimizer (``fused_optimizer=True`` + ``clip_grad``) on the CPU over gloo: over the clipping
strategies of tests/test_optimizer_utils.py, world 1 and zero3 without the slot pool, three steps of the deferred fused update clipped
by ``clip_grad_norm`` follow the torch optimizer clipped the same way -- per-step norms, later losses and the final fp32 masters --
with a norm that bites (max_norm 0.05), and no fp32 gradient buffer outside the units that need one.  A deferred step without a
``clip_grad_norm`` call is the immediate fused update."""
import os
import sys
import tempfile

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_optimizer_utils import CLIP  # noqa: E402

_PORT = [31400]

STRATEGIES = dict(CLIP, world1=(1, {}), dp2_zero3_nopool_ckpt=(2, dict(sdp=1, embed_sdp=1, zero3_pool_slots=0, global_checkpoint=1)))


def run(world, over, arm, backend="oracle", timeout=900):
    from _launch import launch_ranks
    _PORT[0] += 1
    tmp = tempfile.mkdtemp(prefix="hgb_clip_")
    rep = launch_ranks("_clip_worker", world, dict(over, _arm=arm, _dump=os.path.join(tmp, "m")), _PORT[0] + os.getpid() % 500,
                       timeout=timeout, backend=backend)
    masters = []
    for r in range(world):
        path = os.path.join(tmp, "m.rank%d" % r)
        masters.append(torch.load(path, weights_only=True))
        os.remove(path)
    os.rmdir(tmp)
    rep["masters"] = torch.cat([m[k].reshape(-1) for m in masters for k in sorted(m)])
    return rep


def rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("name", sorted(STRATEGIES))
def test_fused_clip_matches_torch_clip(name):
    world, over = STRATEGIES[name]
    fused, ref = run(world, over, "fused_clip"), run(world, over, "torch_clip")
    assert ref["norms"][0] > 0.05                       # the coefficient is below 1: clipping changes the update
    for a, b in zip(fused["norms"], ref["norms"]):
        assert abs(a - b) <= 1e-5 * b, (fused["norms"], ref["norms"])
    for a, b in zip(fused["losses"][1:], ref["losses"][1:]):
        assert abs(a - b) <= 1e-5 * abs(b), (fused["losses"], ref["losses"])
    assert rel(fused["masters"], ref["masters"]) <= 1e-5
    assert abs(fused["norms"][0] - fused["oracle_norm0"]) <= 2e-2 * fused["oracle_norm0"]
    # no fp32 gradient buffer except on pooled zero3 and replicated DDP units
    assert all(needed for _, needed in fused["fp32_grad_units"]), fused["fp32_grad_units"]


@pytest.mark.parametrize("name", ["world1", "dp2_zero3", "tp2_dp2_zero2"])
def test_deferred_step_without_clip_call_is_the_immediate_update(name):
    world, over = STRATEGIES[name]
    deferred, immediate = run(world, over, "fused_defer"), run(world, over, "fused")
    assert rel(deferred["masters"], immediate["masters"]) <= 1e-5
    for a, b in zip(deferred["losses"], immediate["losses"]):
        assert abs(a - b) <= 1e-5 * abs(b)

"""GPU checks of context parallelism in the GPT family.

* hidden-state dropout under zigzag context parallelism: ``bias_dropout_add`` over a rank's token runs (one launch of the existing
  bg_dropout_add_fwd / bg_dropout_bwd per run) reproduces that rank's rows of ONE whole-sequence launch bit for bit, forward and dx,
  for c = 2, 4, 8 with and without a Megatron-SP slice; dbias matches the fp64 sum of the rank's rows to fp32 summation noise;
* the ring schedule and the gathered path's per-chunk prefix calls at GPT head shapes (GPT-3 6.7B's 32 heads of 128, MHA, and
  GPT-2 small's 12 of 64) for c virtual ranks on one device, against ONE flash-attn call on the un-zigzagged sequence, within
  tests/test_gpu_cp_ring.py's bounds -- kernel level, as that file builds it;
* the strategies of tests/test_gpt_cp.py end to end through the CUDA path (skipped below the GPU count they need)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _dropout_ref as dref  # noqa: E402
from test_gpu_cp_ring import Ring, _interleave, _rel, _unzigzag, _zigzag, bg  # noqa: E402,F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
BF = torch.bfloat16


class _G:
    def __init__(self, size, rank):
        self.size, self.rank = size, rank

    def rank_in_group(self):
        return self.rank


@pytest.fixture(scope="module")
def be():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from hetu_galvatron_b200.core.runtime import world
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend
    world.get_rank()
    b = CudaBackend(arena_bytes=1 << 24)
    yield b
    b.close()


@pytest.mark.parametrize("c,t", [(2, 1), (4, 1), (8, 1), (2, 2), (4, 2), (8, 2)])
def test_dropout_runs_match_one_whole_sequence_launch(be, monkeypatch, c, t):
    from hetu_galvatron_b200.core.runtime.redistribute import local_positions
    from hetu_galvatron_b200.core.runtime.tensor_parallel import random as rnd
    from hetu_galvatron_b200.gpt_hf.GPTModel_tensor_parallel import row_runs
    monkeypatch.setattr(rnd, "get_backend", lambda: be)
    seed, it, site, sample_base, p = 1234, 5, 7, 3, 0.1
    S, b, h = 1024, 2, 512
    g = torch.Generator(device="cuda").manual_seed(c * 10 + t)
    x, res, dy = [torch.randn(S, b, h, device="cuda", generator=g).to(BF) for _ in range(3)]
    bias = torch.randn(h, device="cuda", generator=g)
    y_full = be.dropout_add_fwd(x, bias, res, p, seed, it, site, 0, sample_base)
    dx_full, _ = be.dropout_bwd(dy, p, seed, it, site, 0, sample_base, with_bias=True)
    rnd.begin_iteration(seed, it, sample_base)
    rows = S // (c * t)
    for r in range(c):
        for k in range(t):
            runs = row_runs(rows, _G(c, r), None, _G(t, k) if t > 1 else None)
            assert len(runs) <= 2
            pos = local_positions(S, c, r)[k * rows:(k + 1) * rows]
            idx = pos.cuda()
            xl, rl = x[idx].clone().requires_grad_(True), res[idx].clone().requires_grad_(True)
            bl = bias.clone().requires_grad_(True)
            y = rnd.bias_dropout_add(xl, bl, rl, p, site, runs)
            y.backward(dy[idx])
            torch.cuda.synchronize()
            assert torch.equal(y, y_full[idx]), (r, k, runs)
            assert torch.equal(xl.grad, dx_full[idx]), (r, k, runs)
            keep = dref.keep_mask(seed, it, site, pos.numpy(), sample_base + np.arange(b), h, p)
            want = torch.where(keep, dy[idx].cpu().double() * float(dref.scale(p)), torch.zeros((), dtype=torch.float64)).sum((0, 1))
            assert torch.allclose(bl.grad.cpu().double(), want, rtol=1e-5, atol=1e-4), float((bl.grad.cpu().double() - want).abs().max())


def _gather_path(be, q_loc, k, v, dout_loc, c, scale):
    """the gathered exchange's compute per rank: its two zigzag chunks against the K/V prefix up to each chunk's end (the all-gather
    and its reduce-scatter are the plain collectives); -> (out per rank, dq per rank, dk, dv summed over ranks)"""
    kg, vg = k.clone().requires_grad_(True), v.clone().requires_grad_(True)
    outs, dqs = [], []
    for r in range(c):
        q = q_loc[r].clone().requires_grad_(True)
        half = q.shape[1] // 2
        o = torch.cat([be.attention_prefix(q[:, :half], kg[:, :(r + 1) * half], vg[:, :(r + 1) * half], scale),
                       be.attention_prefix(q[:, half:], kg[:, :(2 * c - r) * half], vg[:, :(2 * c - r) * half], scale)], 1)
        o.backward(dout_loc[r])
        outs.append(o.detach())
        dqs.append(q.grad)
    return outs, dqs, kg.grad, vg.grad


@pytest.mark.parametrize("n,d", [(32, 128), (12, 64)], ids=["gpt3_6.7b_32x128", "gpt2_12x64"])
@pytest.mark.parametrize("c,S", [(2, 8192), (4, 16384), (8, 32768)])
def test_ring_and_gather_match_flash_at_gpt_heads(bg, n, d, c, S):
    from flash_attn.flash_attn_interface import _flash_attn_backward, _flash_attn_forward
    from hetu_galvatron_b200.core.runtime.tensor_parallel import transformer as tr
    b, scale = 1, d ** -0.5
    W = Ring(bg, c, b * (S // c) * n * d)           # MHA: K/V carry every head
    try:
        g = torch.Generator(device="cuda").manual_seed(13)
        q, k, v, dout = [torch.randn(b, S, n, d, device="cuda", generator=g).to(BF) for _ in range(4)]
        out_ref, lse_ref, _, _ = _flash_attn_forward(q, k, v, 0.0, scale, causal=True, window_size_left=-1, window_size_right=-1,
                                                     softcap=0.0, alibi_slopes=None, return_softmax=False)
        dq_ref, dk_ref, dv_ref = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        _flash_attn_backward(dout, q, k, v, out_ref, lse_ref, dq_ref, dk_ref, dv_ref, 0.0, scale, True, -1, -1, 0.0, None, False)
        loc = [[_zigzag(t, c, r) for t in (q, k, v, dout)] for r in range(c)]
        res = _interleave([tr.ring_attention_fwd(W.be, W.rings[r], *loc[r][:3], scale) for r in range(c)])
        grads = _interleave([tr.ring_attention_bwd(W.be, W.rings[r], loc[r][3], *loc[r][:3], res[r][0], res[r][1], scale)
                             for r in range(c)])
        W.check()
        ring = {"out": _unzigzag([o for o, _ in res], c)}
        ring["dq"], ring["dk"], ring["dv"] = [_unzigzag([gr[i] for gr in grads], c) for i in range(3)]
        outs, dqs, dk_g, dv_g = _gather_path(W.be, [lc[0] for lc in loc], k, v, [lc[3] for lc in loc], c, scale)
        gather = {"out": _unzigzag(outs, c), "dq": _unzigzag(dqs, c), "dk": dk_g, "dv": dv_g}
        ref = {"out": out_ref, "dq": dq_ref, "dk": dk_ref, "dv": dv_ref}
        for name, got in (("ring", ring), ("gather", gather)):
            obs = {key + "_rel_l2": _rel(got[key], ref[key]) for key in ref}
            print("GPT_CP_OBS %s n=%d d=%d c=%d S=%d %s" % (name, n, d, c, S, obs), flush=True)
            assert obs["out_rel_l2"] < 1e-2, (name, obs)
            assert obs["dq_rel_l2"] < 2e-2 and obs["dk_rel_l2"] < 2e-2 and obs["dv_rel_l2"] < 2e-2, (name, obs)
    finally:
        W.close()


def _cases():
    from test_gpt_cp import PARAMS
    return PARAMS


@pytest.mark.parametrize("name,comm", _cases(), ids=["%s-%s" % p for p in _cases()])
def test_gpt_cp_strategy_cuda(name, comm):
    from test_gpt_cp import CASES, _check, launch
    world, cfg = CASES[name]
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    rep = launch(world, dict(cfg, cp_comm=comm), backend="cuda")
    _check(rep, world, cfg, comm)

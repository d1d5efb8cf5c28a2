"""GPU checks of the dropout row kernels (bg_dropout_add_fwd / bg_dropout_bwd through CudaBackend) against the torch fp32
restatement of tests/_dropout_ref.py -- masks, forward output and dx bit-identical, dbias within fp32 summation noise, one launch
equal to two launches over row halves -- and the GPT / BERT families with hidden dropout against the oracle with the same masks on
the GPU path (multi-GPU cases skip below the GPU count they need)."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _dropout_ref as dref  # noqa: E402
from test_dropout import CASES, launch  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
BF = torch.bfloat16


def _need(n):
    if not torch.cuda.is_available() or torch.cuda.device_count() < n:
        pytest.skip("needs %d GPU(s)" % n)


@pytest.fixture(scope="module")
def be():
    _need(1)
    from hetu_galvatron_b200.core.runtime import world
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend
    world.get_rank()
    b = CudaBackend(arena_bytes=1 << 24)
    yield b
    b.close()


def _keep(seed, it, site, s, b, h, p, seq_base, sample_base):
    return dref.keep_mask(seed, it, site, seq_base + np.arange(s), sample_base + np.arange(b), h, p)


# (s, b, h): rows = s * b; 1063 * 3 rows is not a multiple of the CTA count of any grid
SHAPES = [(64, 2, 128), (1063, 3, 256), (17, 1, 4096), (8, 4, 8)]
COORDS = [(1234, 0, 4, 0, 0, 0.1), (7, 13, 2, 512, 6, 0.5), (0xFFFFFFFF, 0xFFFF, 0x7FFFFFFF, 3, 1000, 0.01), (42, 1, 0, 96, 0, 0.9)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("coords", COORDS)
def test_mask_and_forward_bit_identical(be, shape, coords):
    seed, it, site, seq_base, sample_base, p = coords
    s, b, h = shape
    g = torch.Generator(device="cpu").manual_seed(s * 131 + h)
    x, r = torch.randn(s, b, h, generator=g).to(BF), torch.randn(s, b, h, generator=g).to(BF)
    keep = _keep(seed, it, site, s, b, h, p, seq_base, sample_base)
    # mask alone: x = 1, no bias, no residual -> y = keep * bf16(scale)
    ones = torch.ones(s, b, h, dtype=BF, device="cuda")
    y1 = be.dropout_add_fwd(ones, None, None, p, seed, it, site, seq_base, sample_base).cpu()
    assert torch.equal(y1 != 0, keep)
    for bias in (None, torch.randn(h, generator=g), torch.randn(h, generator=g).to(BF)):
        for res in (None, r):
            got = be.dropout_add_fwd(x.cuda(), None if bias is None else bias.cuda(), None if res is None else res.cuda(), p, seed, it,
                                     site, seq_base, sample_base).cpu()
            want = dref.dropout_add_ref(x, bias, res, keep, p)
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (float((got.float() - want.float()).abs().max()))


@pytest.mark.parametrize("shape", SHAPES)
def test_backward_bit_identical(be, shape):
    s, b, h = shape
    seed, it, site, seq_base, sample_base, p = 99, 3, 5, 40, 2, 0.2
    dy = torch.randn(s, b, h, generator=torch.Generator().manual_seed(5)).to(BF)
    keep = _keep(seed, it, site, s, b, h, p, seq_base, sample_base)
    dx, db = be.dropout_bwd(dy.cuda(), p, seed, it, site, seq_base, sample_base, with_bias=True)
    want_dx, want_db = dref.dropout_bwd_ref(dy, keep, p)
    assert torch.equal(dx.cpu().view(torch.int16), want_dx.view(torch.int16))
    tol = 1e-5 * (dy.float().abs().reshape(-1, h).sum(0) / (1 - p)) + 1e-6
    assert ((db.cpu() - want_db).abs() <= tol).all()
    dx2, none = be.dropout_bwd(dy.cuda(), p, seed, it, site, seq_base, sample_base, with_bias=False)
    assert none is None and torch.equal(dx2, dx)


def test_one_launch_equals_two_half_launches(be):
    s, b, h = 300, 2, 1024
    seed, it, site, p = 5, 8, 11, 0.3
    g = torch.Generator().manual_seed(1)
    x, r, bias = torch.randn(s, b, h, generator=g).to(BF).cuda(), torch.randn(s, b, h, generator=g).to(BF).cuda(), torch.randn(h, generator=g).cuda()
    full = be.dropout_add_fwd(x, bias, r, p, seed, it, site, 10, 4)
    h0 = be.dropout_add_fwd(x[:120], bias, r[:120], p, seed, it, site, 10, 4)
    h1 = be.dropout_add_fwd(x[120:], bias, r[120:], p, seed, it, site, 130, 4)
    assert torch.equal(full, torch.cat([h0, h1]))
    # ... and the output does not depend on the grid: fewer CTAs per launch, same bits
    old = be.bg.get_tunable("local_ctas")
    try:
        be.bg.set_tunable("local_ctas", 7)
        assert torch.equal(be.dropout_add_fwd(x, bias, r, p, seed, it, site, 10, 4), full)
    finally:
        be.bg.set_tunable("local_ctas", old)


def test_bad_arguments_are_status_codes(be):
    x = torch.zeros(4, 1, 12, dtype=BF, device="cuda")
    with pytest.raises(be.bg.BgError, match="multiple of 8"):
        be.dropout_add_fwd(x, None, None, 0.1, 1, 0, 0, 0, 0)
    with pytest.raises(be.bg.BgError, match=r"\[0, 1\)"):
        be.dropout_add_fwd(torch.zeros(4, 1, 16, dtype=BF, device="cuda"), None, None, 1.0, 1, 0, 0, 0, 0)


WORLD1 = ["gpt_world1", "gpt_world1_ckpt_chunks2"]
WORLD2 = ["gpt_tp2", "gpt_tp2_megatron_sp", "gpt_dp2_zero3", "gpt_pp2_1f1b", "bert_tp2_megatron_sp", "bert_ulysses2"]
WORLD4 = ["gpt_baseline3_pp2_tp2_sp_zero2", "bert_baseline4_ulysses2_dp2"]


@pytest.mark.parametrize("name", WORLD1 + WORLD2 + WORLD4)
def test_family_parity_with_hidden_dropout_on_gpus(name):
    world, cfg = CASES[name]
    _need(world)
    rep = launch(world, dict(cfg), backend="cuda")
    assert rep["max_grad_err"] < 3e-2 and rep["launches"] > 0
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])


def test_attention_dropout_one_gpu_is_finite_and_reproducible():
    _need(1)
    cfg = dict(_mode="loss", _family="gpt", _spec=dict(attn_pdrop=0.1, resid_pdrop=0.1, embd_pdrop=0.1), seed=1234, chunks=2)
    a = launch(1, dict(cfg), backend="cuda")["loss"]
    b = launch(1, dict(cfg), backend="cuda")["loss"]
    assert math.isfinite(a) and a == b

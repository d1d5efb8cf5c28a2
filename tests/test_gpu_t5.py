"""The T5 family on the GPU: the cross-attention relayout pair against exact references, its argument checks, the encoder-gradient
addend of the key_value dgrad, and the family through the CUDA backend.

  * bg_cross_attn_qkv_fwd / _bwd at t5-small / base / large / 3B geometry (head dim 64 and 128, 4 to 32 heads per rank, s_q != s_k
    both ways, odd batches): q, k, v, dq_mixed and dkv_mixed bit for bit against the torch restatement (tests/_t5_backend.py), the
    bias gradients within fp32 summation error of float64;
  * bad arguments return status codes before any launch;
  * at tensor-parallel degree 1 the pass-through gradient of the encoder output rides in the dgrad GEMM's epilogue: the result is
    GEMM-then-add within one bf16 rounding, and the backward of the key_value projection runs its two GEMMs and no elementwise add;
  * the tiny T5 of tests/test_t5.py through the CUDA backend against the oracle, with and without checkpointing; the multi-GPU
    cases skip below their device count."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _fp_check import BF, _bits, assert_within, gamma  # noqa: E402

gpu = pytest.mark.gpu
EINVAL = -1
UB = 2.0 ** -8              # unit roundoff of bf16


@pytest.fixture(scope="module")
def be():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from hetu_galvatron_b200.core.runtime import backend as backend_mod
    backend = backend_mod.CudaBackend(comm=None, arena_bytes=1 << 20)
    previous = backend_mod._BACKEND
    backend_mod.set_backend(backend)             # (the autograd functions reach the backend through get_backend())
    yield backend
    backend_mod.set_backend(previous)


# (heads per rank, head dim, s_q, s_k, batch): t5-small tp 1 / t5-base tp 1 / t5-large tp 4 / t5-3B tp 1 / t5-3B tp 8
GEOMS = [(8, 64, 512, 128, 3), (12, 64, 128, 512, 1), (4, 64, 512, 512, 5), (32, 128, 128, 512, 3), (4, 128, 512, 128, 7)]


@gpu
@pytest.mark.parametrize("heads,hn,s_q,s_k,b", GEOMS)
def test_cross_attn_relayout_is_exact(be, heads, hn, s_q, s_k, b):
    from _t5_backend import cross_attn_qkv_bwd, cross_attn_qkv_fwd
    g = torch.Generator(device="cuda").manual_seed(heads * 1000 + s_q + b)
    qm = torch.randn(s_q, b, heads * hn, device="cuda", generator=g).to(BF)
    kvm = torch.randn(s_k, b, heads * 2 * hn, device="cuda", generator=g).to(BF)
    qb = torch.randn(heads * hn, device="cuda", generator=g).to(BF)
    kvb = torch.randn(heads * 2 * hn, device="cuda", generator=g).to(BF)
    for biases in ((qb, kvb), (None, None)):
        got = be.cross_attn_qkv_fwd(qm, biases[0], kvm, biases[1], heads, hn)
        want = cross_attn_qkv_fwd(qm.cpu(), None if biases[0] is None else qb.cpu(), kvm.cpu(), None if biases[1] is None else kvb.cpu(),
                                  heads, hn)
        for a, w in zip(got, want):
            assert a.shape == w.shape and torch.equal(_bits(a.cpu()), _bits(w))
    dq = torch.randn(b, s_q, heads, hn, device="cuda", generator=g).to(BF)
    dk, dv = [torch.randn(b, s_k, heads, hn, device="cuda", generator=g).to(BF) for _ in range(2)]
    dqm, dkvm, dqb, dkvb = be.cross_attn_qkv_bwd(dq, dk, dv)
    wqm, wkvm, _, _ = cross_attn_qkv_bwd(dq.cpu(), dk.cpu(), dv.cpu())
    assert torch.equal(_bits(dqm.cpu()), _bits(wqm)) and torch.equal(_bits(dkvm.cpu()), _bits(wkvm))
    for got_b, rows in ((dqb, wqm), (dkvb, wkvm)):
        r = rows.double().reshape(-1, rows.shape[-1])
        assert_within(got_b.cpu(), r.sum(0), gamma(r.shape[0]) * r.abs().sum(0), "cross-attention dbias")


@gpu
def test_bad_arguments_return_status_codes(be):
    """Checked before any launch (the pointers are never dereferenced)."""
    L, A, M = be.bg.lib(), 0x10000, 0x10001
    assert L.bg_cross_attn_qkv_fwd(A, A, A, A, A, A, A, 0, 128, 3, 8, 64, None) == EINVAL            # s_q 0
    assert L.bg_cross_attn_qkv_fwd(A, A, A, A, A, A, A, 512, 128, 0, 8, 64, None) == EINVAL          # batch 0
    assert L.bg_cross_attn_qkv_fwd(A, A, A, A, A, A, A, 512, 128, 3, 8, 60, None) == EINVAL          # head dim % 8
    assert L.bg_cross_attn_qkv_fwd(A, M, A, A, A, A, A, 512, 128, 3, 8, 64, None) == EINVAL          # misaligned bias
    assert L.bg_cross_attn_qkv_fwd(None, A, A, A, A, A, A, 512, 128, 3, 8, 64, None) == EINVAL       # null input
    assert L.bg_cross_attn_qkv_bwd(A, A, A, A, A, A, 0, 512, 128, 3, 8, 64, None) == EINVAL          # n_partial 0
    assert L.bg_cross_attn_qkv_bwd(A, A, A, A, A, None, 4, 512, 128, 3, 8, 64, None) == EINVAL       # null partials
    assert L.bg_cross_attn_qkv_bwd(A, A, A, M, A, A, 4, 512, 128, 3, 8, 64, None) == EINVAL          # misaligned dq_mixed


@gpu
def test_encoder_gradient_rides_in_the_dgrad_epilogue(be):
    """t5-large's key_value projection at tp 1 ([s_enc x b, 1024] x [2048, 1024]): d(encoder output) = dgrad + the pass-through
    gradient from one GEMM with the addend, within one bf16 rounding of GEMM-then-add; its backward launches the dgrad and wgrad
    GEMMs and no elementwise kernel (no aten::add in the profile)."""
    from hetu_galvatron_b200.core.runtime.tensor_parallel.transformer import _CrossKvFn
    g = torch.Generator(device="cuda").manual_seed(7)
    s, b, h = 512, 3, 1024
    enc = torch.randn(s, b, h, device="cuda", generator=g).to(BF).requires_grad_(True)
    weight = (torch.randn(2 * h, h, device="cuda", generator=g) * 0.03).to(BF).requires_grad_(True)
    kv, passthrough = _CrossKvFn.apply(enc, weight, False, None)
    dkv = torch.randn(kv.shape, device="cuda", generator=g).to(BF)
    dpass = torch.randn(passthrough.shape, device="cuda", generator=g).to(BF)
    torch.cuda.synchronize()
    n0 = be.launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
        torch.autograd.backward([kv, passthrough], [dkv, dpass])
    torch.cuda.synchronize()
    assert be.launch_count() - n0 == 2                                 # dgrad (+ addend) and wgrad
    assert not [e.name for e in prof.events() if e.name in ("aten::add", "aten::add_")]
    d2, w2, a2 = dkv.reshape(-1, 2 * h), weight.detach(), dpass.reshape(-1, h)
    fused = enc.grad.reshape(-1, h).double()
    gemm = be.gemm(d2, w2, "nn").double()                               # the same kernel without the addend: the same fp32 sums
    plain = (gemm + a2.double()).to(BF).double()                        # GEMM, round, add, round
    # fused = rnd(acc + a), plain = rnd(rnd(acc) + a): they differ by the GEMM output's rounding and the two final roundings
    assert bool(((fused - plain).abs() <= UB * (gemm.abs() + fused.abs() + plain.abs())).all())
    exact = d2.double() @ w2.double() + a2.double()
    bound = UB * exact.abs() + gamma(2 * h + 1) * (d2.double().abs() @ w2.double().abs() + a2.double().abs())
    assert bool(((fused - exact).abs() <= bound).all())


def _launch(world, cfg):
    from _launch import launch_ranks
    return launch_ranks("_t5_worker", world, cfg, 29300 + os.getpid() % 500 + world, timeout=1800, backend="cuda")


def _check(rep):
    assert rep["max_grad_err"] < 3e-2
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])


@gpu
def test_tiny_t5_on_one_gpu():
    """the tiny T5 through the CUDA backend; the checkpointed run equals the plain one; the masked-mean loss with -1 labels"""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    plain = _launch(1, dict(global_train_batch_size=4))
    _check(plain)
    ckpt = _launch(1, dict(global_train_batch_size=4, global_checkpoint=1))
    _check(ckpt)
    assert ckpt["loss"] == plain["loss"] and ckpt["max_grad_err"] == plain["max_grad_err"]
    _check(_launch(1, dict(global_train_batch_size=4, chunks=2, _masked=True)))


def _row_strategy(tps, pp_division, chunks, gbs, pipeline_type="pipedream_flush", vtp=1):
    from test_t5 import row_strategy
    return row_strategy(tps, pp_division, chunks, gbs, pipeline_type=pipeline_type, vtp=vtp)


MULTI = {"tp2_megatron_sp": (2, dict(global_tp_deg=2, vocab_tp=2, global_train_batch_size=4, sequence_parallel=True)),
         "dp2_zero3_ckpt": (2, dict(global_train_batch_size=8, sdp=1, global_checkpoint=1)),
         "pp2_gpipe_split_inside_decoder": (2, dict(_strategy=[[1] * 4, [3, 1], 3, 8, "gpipe"])),
         "pp2_1f1b_split_at_encoder_decoder_boundary": (2, dict(_strategy=[[1] * 4, [2, 2], 2, 8, "pipedream_flush"]))}


@gpu
@pytest.mark.parametrize("name", sorted(MULTI))
def test_tiny_t5_multi_gpu(name):
    world, cfg = MULTI[name]
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    cfg = dict(cfg)
    if "_strategy" in cfg:
        cfg["_strategy"] = _row_strategy(*cfg["_strategy"])
    _check(_launch(world, cfg))

"""Swin's relative-position bias on the GPU: its two kernels against exact references, their argument checks, one attention block
against float64 autograd, and the tiny Swin with the bias through the CUDA backend against the oracle.

  * bg_swin_rel_bias_fwd: bit for bit against the torch restatement (tests/_swin_rpb.py) at Swin-H (window 7) and Swin-L (window
    12) geometry, heads 6 .. 64, shifted and not, micro-batches 1 and odd, bf16 and fp32 tables;
  * bg_swin_rel_bias_bwd: within 1e-5 rel of the float64 sum (and within fp32 summation error of it entry by entry), bit for bit
    the same over two launches, and the same from the padded rows the memory-efficient attention kernel returns;
  * the attention call with the bias runs the memory-efficient kernel (torch.profiler kernel names, printed) and its q, k, v and
    table gradients match float64 autograd."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _fp_check import BF, _bits, assert_within, gamma  # noqa: E402

gpu = pytest.mark.gpu
EINVAL, EUNSUPPORTED = -1, -7


@pytest.fixture(scope="module")
def be():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend
    return CudaBackend(comm=None, arena_bytes=1 << 20)


@pytest.fixture(scope="module")
def ref():
    from _swin_rpb import SwinRelBiasOracleBackend
    return SwinRelBiasOracleBackend.__new__(SwinRelBiasOracleBackend)      # (its Swin methods are pure torch)


def _layout(res, window, shift):
    from hetu_galvatron_b200.swin.SwinModel_tensor_parallel import WindowLayout
    return WindowLayout(res, window, shift)


# (res, window, shift, mb, heads): Swin-H stages 0 / 1 / 2 / 3, Swin-L stages 0 / 1 / 3
GEOMS = [(56, 7, 3, 1, 8), (56, 7, 3, 3, 8), (28, 7, 3, 5, 16), (14, 7, 3, 7, 32), (7, 7, 0, 1, 64), (7, 7, 0, 33, 64),
         (96, 12, 6, 1, 6), (48, 12, 6, 3, 12), (12, 12, 0, 5, 48)]


@gpu
@pytest.mark.parametrize("table_dtype", [BF, torch.float32], ids=["bf16_table", "fp32_table"])
@pytest.mark.parametrize("res,window,shift,mb,heads", GEOMS)
def test_rel_bias_fwd_is_the_restatement(be, ref, res, window, shift, mb, heads, table_dtype):
    lay = _layout(res, window, shift)
    index, mask, _, _ = lay.rel_maps("cuda")
    g = torch.Generator(device="cuda").manual_seed(res * heads + mb)
    table = torch.randn((2 * window - 1) ** 2, heads, device="cuda", generator=g).to(table_dtype)
    got = be.swin_rel_bias_fwd(table, index, mask, mb, lay.n_windows, window)
    want = ref.swin_rel_bias_fwd(table.cpu(), index.cpu(), mask.cpu() if mask is not None else None, mb, lay.n_windows, window)
    assert got.shape == want.shape == (mb * lay.n_windows, heads, window ** 2, window ** 2)
    assert torch.equal(_bits(got.cpu()), _bits(want))
    base = got._base if got._base is not None else got
    assert not base[..., window ** 2:].any()                          # the padding columns are written, zero
    assert (torch.isinf(got).any().item()) == (shift > 0)


@gpu
@pytest.mark.parametrize("res,window,shift,mb,heads", GEOMS)
def test_rel_bias_bwd_against_float64(be, res, window, shift, mb, heads):
    lay = _layout(res, window, shift)
    index, _, cells, offsets = lay.rel_maps("cuda")
    L = window * window
    g = torch.Generator(device="cuda").manual_seed(res * heads + mb + 1)
    dbias = torch.randn(mb * lay.n_windows, heads, L, L, device="cuda", generator=g).to(BF)
    got = be.swin_rel_bias_bwd(dbias, cells, offsets, lay.n_windows, window)
    again = be.swin_rel_bias_bwd(dbias, cells, offsets, lay.n_windows, window)
    assert torch.equal(_bits(got), _bits(again))                       # fixed summation order
    d = dbias.double().sum(0).reshape(heads, L * L).t()
    a = dbias.double().abs().sum(0).reshape(heads, L * L).t()
    n_table = (2 * window - 1) ** 2
    want = torch.zeros(n_table, heads, dtype=torch.float64, device="cuda").index_add_(0, index.long(), d)
    mag = torch.zeros_like(want).index_add_(0, index.long(), a)
    k = dbias.shape[0] + L + be.norm_partials
    assert_within(got, want, gamma(k) * mag, "dtable")
    assert float((got.double() - want).norm() / want.norm()) < 1e-5
    # the rows the memory-efficient attention kernel returns: padded to 64 columns, sliced
    padded = torch.zeros(*dbias.shape[:3], (L + 63) // 64 * 64, dtype=BF, device="cuda")
    padded[..., :L] = dbias
    assert torch.equal(_bits(be.swin_rel_bias_bwd(padded[..., :L], cells, offsets, lay.n_windows, window)), _bits(got))


@gpu
def test_rel_bias_bad_arguments_return_status_codes(be):
    """Checked before any launch (the pointers are never dereferenced)."""
    L, A, M = be.bg.lib(), 0x10000, 0x10001
    before = L.bg_launch_count()
    assert L.bg_swin_rel_bias_fwd(A, 0, A, None, A, 0, 64, 8, 7, 49, 56, None) == EINVAL          # mb 0
    assert L.bg_swin_rel_bias_fwd(A, 0, A, None, A, 2, 64, 0, 7, 49, 56, None) == EINVAL          # no heads
    assert L.bg_swin_rel_bias_fwd(A, 0, A, None, A, 2, 64, 8, 7, 48, 56, None) == EINVAL          # L != window^2
    assert L.bg_swin_rel_bias_fwd(A, 0, A, None, A, 2, 64, 8, 7, 49, 52, None) == EINVAL          # ld % 8
    assert L.bg_swin_rel_bias_fwd(A, 0, A, None, A, 2, 64, 8, 7, 49, 48, None) == EINVAL          # ld < L
    assert L.bg_swin_rel_bias_fwd(A, 5, A, None, A, 2, 64, 8, 7, 49, 56, None) == EUNSUPPORTED    # table dtype
    assert L.bg_swin_rel_bias_fwd(None, 0, A, None, A, 2, 64, 8, 7, 49, 56, None) == EINVAL       # null table
    assert L.bg_swin_rel_bias_fwd(M, 0, A, None, A, 2, 64, 8, 7, 49, 56, None) == EINVAL          # misaligned bf16 table
    assert L.bg_swin_rel_bias_fwd(A + 2, 1, A, None, A, 2, 64, 8, 7, 49, 56, None) == EINVAL      # misaligned fp32 table
    assert L.bg_swin_rel_bias_fwd(A, 0, A + 2, None, A, 2, 64, 8, 7, 49, 56, None) == EINVAL      # misaligned index
    assert L.bg_swin_rel_bias_fwd(A, 0, A, None, A + 8, 2, 64, 8, 7, 49, 56, None) == EINVAL      # bias not 16-B aligned
    assert L.bg_swin_rel_bias_fwd(A, 0, A, None, A, 2, 64, 70000, 7, 49, 56, None) == EUNSUPPORTED  # heads > 65535
    assert L.bg_swin_rel_bias_fwd(A, 0, A, None, A, 2, 4, 8, 16, 256, 256, None) == EUNSUPPORTED  # 16 x 16 window
    assert L.bg_swin_rel_bias_bwd(A, A, A, A, 0, 2, 64, 8, 7, 49, 56, None) == EINVAL             # n_partial 0
    assert L.bg_swin_rel_bias_bwd(A, A, A, A, 65536, 2, 64, 8, 7, 49, 56, None) == EINVAL         # n_partial > 65535
    assert L.bg_swin_rel_bias_bwd(A, A, A, A, 4, 2, 64, 8, 12, 49, 56, None) == EINVAL            # L != window^2
    assert L.bg_swin_rel_bias_bwd(A + 8, A, A, A, 4, 2, 64, 8, 7, 49, 56, None) == EINVAL         # dbias not 16-B aligned
    assert L.bg_swin_rel_bias_bwd(A, None, A, A, 4, 2, 64, 8, 7, 49, 56, None) == EINVAL          # null cells
    assert L.bg_swin_rel_bias_bwd(A, A, A + 1, A, 4, 2, 64, 8, 7, 49, 56, None) == EINVAL         # misaligned offsets
    assert L.bg_swin_rel_bias_bwd(A, A, A, A + 2, 4, 2, 64, 8, 7, 49, 56, None) == EINVAL         # misaligned partials
    assert L.bg_launch_count() == before


@gpu
@pytest.mark.parametrize("res,window,shift,mb,heads,hn", [(14, 7, 3, 3, 8, 40), (7, 7, 0, 2, 16, 40), (24, 12, 6, 2, 6, 32)])
def test_attention_block_with_bias_against_float64(be, res, window, shift, mb, heads, hn):
    """q, k, v [mb * nW, L, heads, hn] and the table through _RelBiasFn + CudaBackend.attention: the output and the q / k / v / table
    gradients against float64 autograd of softmax(q k^T / sqrt(hn) + table[index] + shift mask) v (rel-L2 2e-2; bf16 inputs)."""
    from torch.profiler import ProfilerActivity, profile
    from hetu_galvatron_b200.core.runtime import backend as backend_mod
    from hetu_galvatron_b200.swin.SwinModel_tensor_parallel import _RelBiasFn
    lay = _layout(res, window, shift)
    L, nw = window * window, lay.n_windows
    g = torch.Generator(device="cuda").manual_seed(res + heads)
    q, k, v = [torch.randn(mb * nw, L, heads, hn, device="cuda", generator=g).to(BF).requires_grad_(True) for _ in range(3)]
    table = (torch.randn((2 * window - 1) ** 2, heads, device="cuda", generator=g)).to(BF).requires_grad_(True)
    dout = torch.randn(mb * nw, L, heads, hn, device="cuda", generator=g).to(BF)
    prev = backend_mod._BACKEND
    backend_mod.set_backend(be)
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            mask = _RelBiasFn.apply(table, lay, mb)
            out = be.attention(q, k, v, False, hn ** -0.5, window_bias=mask)
            out.backward(dout)
            torch.cuda.synchronize()
    finally:
        backend_mod.set_backend(prev)
    names = sorted({e.key for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA})
    print("kernels:", names)
    assert any("swin_rel_bias_fwd" in n for n in names) and any("swin_rel_bias_bwd" in n for n in names)
    assert any("fmha_cutlassF" in n or "efficient_attention" in n for n in names), names      # memory-efficient forward
    assert any("fmha_cutlassB" in n or "efficient_attention" in n for n in names), names      # ... and backward
    assert not any("cudnn" in n.lower() for n in names), names
    qd, kd, vd, td = [t.detach().double().requires_grad_(True) for t in (q, k, v, table)]
    index = lay.rel_maps("cuda")[0].long()
    bias = td[index].t().reshape(1, heads, L, L)
    scores = qd.transpose(1, 2) @ kd.transpose(1, 2).transpose(-1, -2) * hn ** -0.5 + bias
    if shift:
        m = lay.rel_maps("cuda")[1].bool().repeat(mb, 1, 1)[:, None]
        scores = scores.masked_fill(m, float("-inf"))
    want = (torch.softmax(scores, -1) @ vd.transpose(1, 2)).transpose(1, 2)
    want.backward(dout.double())
    rel = lambda a, b: float((a.double() - b).norm() / b.norm())  # noqa: E731
    errs = dict(out=rel(out, want), dq=rel(q.grad, qd.grad), dk=rel(k.grad, kd.grad), dv=rel(v.grad, vd.grad),
                dtable=rel(table.grad, td.grad))
    print("rel-L2:", errs)
    assert max(errs.values()) < 2e-2, errs


def _launch(world, cfg):
    from _launch import launch_ranks
    return launch_ranks("_swin_rpb_worker", world, cfg, 29700 + os.getpid() % 500 + world, timeout=1800, backend="cuda")


@gpu
def test_tiny_swin_with_bias_on_one_gpu():
    """the tiny Swin (224 px, window 7) with the bias through the CUDA backend against the oracle; micro-batch 7 pads stages 2 and 3;
    the checkpointed run (the bias recomputed) computes the plain run's loss (the memory-efficient backward may add in any order, so
    the gradients are held to the oracle's bar, not to each other's bits)"""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    plain = _launch(1, dict(global_train_batch_size=7))
    ckpt = _launch(1, dict(global_train_batch_size=7, global_checkpoint=1))
    print("plain:", plain, "\ncheckpointed:", ckpt)
    for rep in (plain, ckpt):
        assert rep["tokens_run"] == [3136, 784, 200, 56]
        assert rep["max_grad_err"] < 3e-2 and rep["table_grad_err"] < 3e-2 and rep["table_grad_max"] > 0.0
        assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
        assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])
    assert ckpt["loss"] == plain["loss"]

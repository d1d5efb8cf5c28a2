"""The Swin family on the GPU: its kernels against exact references, their argument checks, and the family through the CUDA backend.

Kernels (through the backend's thin wrappers over the C ABI), at Swin-H / Swin-L geometry (head dim 40 and 32, widths 192 .. 2560,
merged rows up to 4 x 2560 = 10240 columns), with odd micro-batches and padded token counts:
  * window QKV relayout, window merge and their backwards: bit for bit against the torch restatement (tests/_swin_backend.py, the
    same token maps); the dbias column sums within fp32 summation error of float64;
  * merge + LayerNorm: bit for bit equal to bg_layernorm_fwd on the gathered rows where that kernel takes the width (so it inherits
    tests/test_gpu_ops.py's correct-rounding bar), against float64 with that test's bounds otherwise and with the added bias; backward
    against float64 with the LayerNorm test's bounds, and the scatter leaves no row unwritten;
  * mean-pool: within fp32 summation error of float64, its backward bit for bit;
  * drop path: bit for bit against the torch Philox restatement for bf16 and fp32 biases.
Bad arguments return status codes before any launch.  Then the tiny Swin of tests/test_swin.py through the CUDA backend on one GPU
against the oracle, with the padding tokens' gradient exactly zero and checkpointing changing nothing; the multi-GPU cases skip below
their device count."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _fp_check import BF, F64, U, _bits, assert_rounded, assert_within, gamma  # noqa: E402

gpu = pytest.mark.gpu
NAN = float("nan")
EINVAL, EUNSUPPORTED = -1, -7


@pytest.fixture(scope="module")
def be():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend
    return CudaBackend(comm=None, arena_bytes=1 << 20)


@pytest.fixture(scope="module")
def ref():
    from _swin_backend import SwinOracleBackend
    return SwinOracleBackend.__new__(SwinOracleBackend)      # (its Swin methods are pure torch and need no process group)


def _layout(res, window, shift):
    from hetu_galvatron_b200.swin.SwinModel_tensor_parallel import WindowLayout
    lay = WindowLayout(res, window, shift)
    tmap, inv = lay.maps("cuda")
    return lay, tmap, inv


# (res, window, shift, t_run, mb, heads, head dim): Swin-H stages 0 / 2 (shifted, padded 196 -> 200) / 3, Swin-L stage 1
GEOMS = [(56, 7, 3, 3136, 3, 4, 40), (14, 7, 3, 200, 5, 8, 40), (7, 7, 0, 56, 7, 16, 40), (48, 12, 6, 2304, 2, 6, 32)]


@gpu
@pytest.mark.parametrize("res,window,shift,t_run,mb,heads,hn", GEOMS)
def test_window_relayouts_are_exact(be, ref, res, window, shift, t_run, mb, heads, hn):
    lay, tmap, inv = _layout(res, window, shift)
    g = torch.Generator(device="cuda").manual_seed(res + mb)
    mixed = torch.randn(t_run * mb, heads * 3 * hn, device="cuda", generator=g).to(BF)
    bias = torch.randn(heads * 3 * hn, device="cuda", generator=g).to(BF)
    got = be.swin_window_qkv_fwd(mixed, bias, tmap, inv, lay.n_windows, mb, heads, hn)
    want = ref.swin_window_qkv_fwd(mixed, bias, tmap, inv, lay.n_windows, mb, heads, hn)
    for a, b in zip(got, want):
        assert torch.equal(_bits(a), _bits(b))
    dq, dk, dv = [torch.randn_like(t, dtype=torch.float32).to(BF) for t in got]
    dmixed, dbias = be.swin_window_qkv_bwd(dq, dk, dv, tmap, inv, lay.n_windows, mb, t_run)
    wdm, wdb = ref.swin_window_qkv_bwd(dq, dk, dv, tmap, inv, lay.n_windows, mb, t_run)
    assert torch.equal(_bits(dmixed), _bits(wdm))
    assert not dmixed[res * res * mb:].any()
    terms = wdm.double()
    k = -(-t_run * mb // be.norm_partials) + be.norm_partials
    assert_within(dbias, terms.sum(0), gamma(k) * terms.abs().sum(0), "qkv dbias")
    ctx = torch.randn(mb * lay.n_windows, window * window, heads, hn, device="cuda", generator=g).to(BF)
    rows = be.swin_window_merge_fwd(ctx, tmap, inv, lay.n_windows, mb, t_run)
    assert torch.equal(_bits(rows), _bits(ref.swin_window_merge_fwd(ctx, tmap, inv, lay.n_windows, mb, t_run)))
    assert not rows[res * res:].any()
    drows = torch.randn_like(rows, dtype=torch.float32).to(BF)
    drows[res * res:] = NAN                                  # padding-token rows are never read
    dwin = be.swin_window_merge_bwd(drows, tmap, inv, lay.n_windows, mb, heads, hn)
    assert torch.equal(_bits(dwin), _bits(ref.swin_window_merge_bwd(drows, tmap, inv, lay.n_windows, mb, heads, hn)))


def _ln_bounds(v, w, b, eps, mean, rstd, n):
    """float64 reference and slack of a LayerNorm forward, as tests/test_gpu_ops.py::test_layernorm_fwd_bwd states them"""
    D = 8 * -(-n // (8 * 256)) + 10          # additions on the longest path of the block-wide sum (test_gpu_ops._tree_depth)
    e32 = float(np.float32(eps))
    m = v.mean(-1, keepdim=True)
    var = (v - m).pow(2).mean(-1, keepdim=True)
    r = (var + e32).rsqrt()
    dm = gamma(D) * v.abs().mean(-1, keepdim=True) + gamma(2) * m.abs()
    dv = (gamma(D + 6) * (var + dm * dm + e32) + dm * dm) / (var + e32)
    dr = dv / 2 + 4 * U
    t = (v - m) * r * w
    yr = t + b
    em = w.abs() * r * dm
    return yr, (em + t.abs() * dr) * (1 + gamma(3)) + gamma(4) * (t.abs() + em + yr.abs()), D


def _check_ln_bwd(be, dx, dw, db, vd, gd, w, mean, rstd, D, what):
    """the LayerNorm backward against float64 from the kernel's mean / rstd, with tests/test_gpu_ops.py's bounds; dw / db are the
    fp32 partial sums rounded to the weight's bf16"""
    n = vd.shape[0]
    mk, rk = mean[:n].double()[:, None], rstd[:n].double()[:, None]
    xh = (vd - mk) * rk
    gw = gd * w.double()
    s1, s2 = gw.mean(-1, keepdim=True), (gw * xh).mean(-1, keepdim=True)
    dvr = rk * (gw - s1 - xh * s2)
    edx = rk * (gamma(3) * (gw.abs() + s1.abs()) + gamma(4) * (xh * s2).abs() + gamma(D + 3) * gw.abs().mean(-1, keepdim=True)
                + xh.abs() * gamma(D + 6) * (gw * xh).abs().mean(-1, keepdim=True))
    assert_rounded(dx, dvr, edx, what + " dx")
    k = -(-n // be.norm_partials) + be.norm_partials
    assert_rounded(dw, (gd * xh).sum(0), gamma(k + 3) * (gd * xh).abs().sum(0), what + " dw")
    assert_rounded(db, gd.sum(0), gamma(k) * gd.abs().sum(0), what + " db")
    return dvr


@gpu
@pytest.mark.parametrize("res,c,mb,t_out_run", [(56, 320, 3, 784), (28, 640, 5, 200), (14, 1280, 7, 56), (14, 2560, 2, 56),
                                               (96, 192, 2, 2304), (24, 1536, 3, 144)])
def test_patch_merge_layernorm(be, ref, res, c, mb, t_out_run):
    """r = 2: Swin-H merges (C 320 / 640 / 1280; 2560 for the widest row the kernel takes) and Swin-L's first and last."""
    g = torch.Generator(device="cuda").manual_seed(res * c + mb)
    x = torch.randn(res * res * mb + 8, c, device="cuda", generator=g).to(BF)       # 8 padding-token rows after the real ones
    w = (1 + 0.1 * torch.randn(4 * c, device="cuda", generator=g)).to(BF)
    b = (0.1 * torch.randn(4 * c, device="cuda", generator=g)).to(BF)
    y, mean, rstd = be.swin_merge_ln_fwd(x, None, w, b, 1e-5, mb, res, res, 2, False, t_out_run)
    idx, v = ref._gathered(x, None, mb, res, res, 2, False)
    t_out = idx.shape[0]
    assert not y[t_out:].any() and not mean[t_out * mb:].any() and not rstd[t_out * mb:].any()
    rows = v.reshape(-1, 4 * c).to(BF)
    if 4 * c <= 8192:                          # bg_layernorm_fwd's widest row: the same arithmetic, so the same bits
        yl, ml, rl = be.layernorm_fwd(rows, w, b, 1e-5)
        assert torch.equal(_bits(y[:t_out].reshape(-1, 4 * c)), _bits(yl)) and torch.equal(mean[:t_out * mb], ml)
    yr, slack, D = _ln_bounds(v.reshape(-1, 4 * c).double(), w.double(), b.double(), 1e-5, mean, rstd, 4 * c)
    assert_rounded(y[:t_out].reshape(-1, 4 * c), yr, slack, "merge y")
    dy = torch.randn(t_out_run, mb, 4 * c, device="cuda", generator=g).to(BF)
    dy[t_out:] = NAN                                          # padding-token rows are never read
    dx, dw, db, dab = be.swin_merge_ln_bwd(dy, x, None, w, mean, rstd, mb, res, res, 2, False)
    assert dab is None and not dx[res * res * mb:].any()
    dx_g = dx.reshape(-1, c)[idx.reshape(-1)].reshape(-1, 4 * c)
    _check_ln_bwd(be, dx_g, dw, db, v.reshape(-1, 4 * c).double(), dy[:t_out].reshape(-1, 4 * c).double(), w, mean, rstd, D, "merge")


@gpu
@pytest.mark.parametrize("b,c,side", [(3, 320, 56), (1, 192, 96), (5, 128, 8)])
def test_embedding_bias_layernorm(be, ref, b, c, side):
    """r = 1 with the patch bias: the patch GEMM's (sample, patch) rows -> SBH rows, + bias, LayerNorm; zero padding rows."""
    g = torch.Generator(device="cuda").manual_seed(b * c)
    n = b * side * side
    rows_pad = (n + 7) // 8 * 8 + 8
    x = torch.randn(rows_pad, c, device="cuda", generator=g).to(BF)
    bias = torch.randn(c, device="cuda", generator=g).to(BF)
    w = (1 + 0.1 * torch.randn(c, device="cuda", generator=g)).to(BF)
    lb = (0.1 * torch.randn(c, device="cuda", generator=g)).to(BF)
    t_run = side * side + 8
    y, mean, rstd = be.swin_merge_ln_fwd(x, bias, w, lb, 1e-5, b, side, side, 1, True, t_run)
    idx, v = ref._gathered(x, bias, b, side, side, 1, True)
    assert not y[side * side:].any()
    vd = x[:n].double().view(b, side * side, c).transpose(0, 1).reshape(-1, c) + bias.double()
    yr, slack, D = _ln_bounds(vd, w.double(), lb.double(), 1e-5, mean, rstd, c)
    assert_rounded(y[:side * side].reshape(-1, c), yr, slack + gamma(1) * vd.abs() * w.double().abs() * rstd[:n].double()[:, None], "y")
    dy = torch.randn(t_run, b, c, device="cuda", generator=g).to(BF)
    dx, dw, db, dab = be.swin_merge_ln_bwd(dy, x, bias, w, mean, rstd, b, side, side, 1, True)
    assert not dx[n:].any()
    dx_sbh = dx[:n].view(b, side * side, c).transpose(0, 1).reshape(-1, c)
    dvr = _check_ln_bwd(be, dx_sbh, dw, db, vd, dy[:side * side].reshape(-1, c).double(), w, mean, rstd, D, "embedding")
    assert_within(dab, dvr.sum(0), gamma(n + 2) * dvr.abs().sum(0) + 1e-3 * rstd[:n].double().max() * U * n, "dbias")


@gpu
@pytest.mark.parametrize("tokens,t_run,mb,c", [(49, 56, 64, 2560), (49, 49, 63, 2560), (144, 144, 5, 1536), (196, 200, 3, 1280)])
def test_mean_pool(be, tokens, t_run, mb, c):
    g = torch.Generator(device="cuda").manual_seed(tokens * mb)
    x = torch.randn(t_run, mb, c, device="cuda", generator=g).to(BF)
    x[tokens:] = NAN                                          # padding tokens are never read
    rows_out = (mb + 7) // 8 * 8
    y = be.swin_mean_pool_fwd(x, tokens, rows_out)
    assert not y[mb:].any()
    xd = x[:tokens].double()
    assert_rounded(y[:mb], xd.mean(0), gamma(tokens + 1) * xd.abs().mean(0), "pooled")
    dy = torch.randn(rows_out, c, device="cuda", generator=g).to(BF)
    dx = be.swin_mean_pool_bwd(dy, tokens, t_run, mb)
    want = (dy[:mb].float() / tokens).to(BF)
    assert torch.equal(_bits(dx[:tokens]), _bits(want.unsqueeze(0).expand(tokens, mb, c))) and not dx[tokens:].any()


@gpu
@pytest.mark.parametrize("bias_dtype", [BF, torch.float32], ids=["bf16_bias", "fp32_bias"])
@pytest.mark.parametrize("s,b,h,p", [(3136, 3, 320, 0.1), (56, 63, 2560, 0.3), (200, 5, 1280, 0.5)])
def test_drop_path_is_the_philox_restatement(be, ref, bias_dtype, s, b, h, p):
    g = torch.Generator(device="cuda").manual_seed(s + b)
    x, res = [torch.randn(s, b, h, device="cuda", generator=g).to(BF) for _ in range(2)]
    bias = torch.randn(h, device="cuda", generator=g).to(bias_dtype)
    args = (p, 1234, 7, 3 * 5 + 1, 40)
    y = be.drop_path_add_fwd(x, bias, res, *args)
    want = ref.drop_path_add_fwd(x.cpu(), bias.cpu(), res.cpu(), *args)
    assert torch.equal(_bits(y.cpu()), _bits(want))
    dy = torch.randn(s, b, h, device="cuda", generator=g).to(BF)
    dx, db = be.drop_path_add_bwd(dy, *args, True)
    wdx, wdb = ref.drop_path_add_bwd(dy.cpu(), *args, True)
    assert torch.equal(_bits(dx.cpu()), _bits(wdx))
    assert_within(db.cpu(), wdb.double(), gamma(s * b) * wdx.double().abs().reshape(-1, h).sum(0), "drop path dbias")


@gpu
def test_bad_arguments_return_status_codes(be):
    """Checked before any launch (the pointers are never dereferenced)."""
    L, A, M = be.bg.lib(), 0x10000, 0x10001
    assert L.bg_swin_window_qkv_fwd(A, A, A, A, A, A, 3, 196, 192, 4, 49, 8, 40, None) == EINVAL            # tokens_run < tokens
    assert L.bg_swin_window_qkv_fwd(A, A, A, A, A, A, 3, 196, 200, 4, 48, 8, 40, None) == EINVAL            # 4 x 48 != 196
    assert L.bg_swin_window_qkv_fwd(A, A, A, A, A, A, 3, 196, 200, 4, 49, 8, 36, None) == EINVAL            # head dim % 8
    assert L.bg_swin_window_qkv_fwd(M, A, A, A, A, A, 3, 196, 200, 4, 49, 8, 40, None) == EINVAL            # misaligned
    assert L.bg_swin_window_qkv_bwd(A, A, A, A, A, 0, A, 3, 196, 200, 4, 49, 8, 40, None) == EINVAL         # n_partial 0
    assert L.bg_swin_window_merge_fwd(A, A, A, A, 0, 196, 200, 4, 49, 320, None) == EINVAL                  # mb 0
    assert L.bg_swin_window_merge_bwd(A, A, A, A, 3, 196, 200, 4, 49, 324, None) == EINVAL                  # cols % 8
    assert L.bg_swin_merge_ln_fwd(A, None, A, A, A, A, A, 3, 14, 14, 3, 0, 600, 320, 56, 1e-5, None) == EINVAL     # r = 3
    assert L.bg_swin_merge_ln_fwd(A, None, A, A, A, A, A, 3, 7, 7, 2, 0, 147, 320, 16, 1e-5, None) == EINVAL       # 7 is odd
    assert L.bg_swin_merge_ln_fwd(A, None, A, A, A, A, A, 3, 14, 14, 2, 0, 500, 320, 56, 1e-5, None) == EINVAL     # rows_in < 588
    assert L.bg_swin_merge_ln_fwd(A, None, A, A, A, A, A, 3, 14, 14, 2, 0, 588, 320, 48, 1e-5, None) == EINVAL     # 48 < 49
    assert L.bg_swin_merge_ln_fwd(A, None, A, A, A, A, A, 3, 14, 14, 2, 0, 588, 2568, 56, 1e-5, None) == EUNSUPPORTED
    assert L.bg_swin_merge_ln_bwd(A, A, A, A, A, A, A, A, A, None, 4, 3, 14, 14, 2, 0, 588, 320, None) == EINVAL   # bias w/o dbias
    assert L.bg_swin_mean_pool_fwd(A, A, 49, 56, 63, 60, 2560, None) == EINVAL                              # rows_out < mb
    assert L.bg_swin_mean_pool_bwd(A, A, 49, 48, 63, 2560, None) == EINVAL                                  # tokens_run < tokens
    assert L.bg_drop_path_add_fwd(A, A, 1, A, A, 10, 320, 3, 0, 0.1, 1, 0, 4, None) == EINVAL                # rows % b_loc
    assert L.bg_drop_path_add_fwd(A, A, 1, A, A, 9, 320, 3, 0, 1.0, 1, 0, 4, None) == EINVAL                 # p = 1
    assert L.bg_drop_path_add_fwd(A, A, 9, A, A, 9, 320, 3, 0, 0.1, 1, 0, 4, None) == EUNSUPPORTED           # bias dtype
    assert L.bg_drop_path_add_bwd(A, A, None, 0, 9, 320, 3, 0, 0.1, 1, 0, 4, None) == EINVAL                 # n_partial 0


def _launch(world, cfg):
    from _launch import launch_ranks
    return launch_ranks("_swin_worker", world, cfg, 29400 + os.getpid() % 500 + world, timeout=1800, backend="cuda")


def _check(rep, tokens_run):
    assert rep["tokens_run"] == tokens_run
    assert rep["max_grad_err"] < 3e-2
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])
    assert rep["classifier_pad_rows_max"] == 0.0


@gpu
def test_tiny_swin_on_one_gpu():
    """the tiny Swin (224 px, window 7) through the CUDA backend; micro-batch 7 pads stages 2 and 3 (200 and 56 tokens); the
    checkpointed run equals the plain one; with drop path 0.3 the same oracle masks, with and without checkpointing."""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    plain = _launch(1, dict(global_train_batch_size=7))
    _check(plain, [3136, 784, 200, 56])
    ckpt = _launch(1, dict(global_train_batch_size=7, global_checkpoint=1))
    _check(ckpt, [3136, 784, 200, 56])
    assert ckpt["loss"] == plain["loss"] and ckpt["max_grad_err"] == plain["max_grad_err"]
    drop = _launch(1, dict(global_train_batch_size=8, _spec=dict(drop_path_rate=0.3)))
    _check(drop, [3136, 784, 196, 49])
    drop_ckpt = _launch(1, dict(global_train_batch_size=8, global_checkpoint=1, _spec=dict(drop_path_rate=0.3)))
    _check(drop_ckpt, [3136, 784, 196, 49])         # the recompute draws the forward's drop-path masks
    assert drop_ckpt["loss"] == drop["loss"] and drop_ckpt["max_grad_err"] == drop["max_grad_err"]


@gpu
def test_padding_token_gradient_is_exactly_zero():
    """Swin-H/224's stage 0 never pads (3136 x m is a multiple of 8), so a 168-px image (a 42 x 42 grid, 1764 tokens) at
    micro-batch 1: stage 0 runs 1768 tokens and the gradient reaching the embedding's 4 padding rows is exactly zero."""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    rep = _launch(1, dict(global_train_batch_size=1, _check_padded_token_grad=True,
                          _spec=dict(image_size=168, depths=[2, 2], num_heads=[1, 2])))
    assert rep["tokens_run"][0] == 1768 and rep["pad_token_grad_max"] == 0.0 and rep["real_token_grad_max"] > 0.0
    assert rep["max_grad_err"] < 3e-2


TP_HEADS = dict(num_heads=[2, 4, 8, 16])
MULTI = {"tp2_vtp2": (2, dict(global_tp_deg=2, vocab_tp=2, global_train_batch_size=8, _spec=TP_HEADS)),
         "dp2_zero3_ckpt": (2, dict(global_train_batch_size=16, sdp=1, global_checkpoint=1)),
         "pp2_1f1b": (2, dict(pp_deg=2, chunks=2, global_train_batch_size=16)),
         "drop_path_tp2": (2, dict(global_tp_deg=2, vocab_tp=2, global_train_batch_size=8, _spec=dict(TP_HEADS, drop_path_rate=0.3)))}


@gpu
@pytest.mark.parametrize("name", sorted(MULTI))
def test_tiny_swin_multi_gpu(name):
    world, cfg = MULTI[name]
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    _check(_launch(world, dict(cfg)), [3136, 784, 196, 49])

"""GPU parity of the local fused kernels (through the C ABI) against float64 restatements of the reference ops, computed from the
same bf16 / fp32 inputs the kernels read: RMSNorm (flash_attn.ops.rms_norm semantics, LlamaModel_tensor_parallel.py:2,48), LayerNorm
with bias (torch.nn.LayerNorm of the GPT / BERT families), bias + GeLU in the tanh and the erf form (oracle/gpt_bert_ref.py::gelu),
swiglu (transformer.py:122-124), the QKV split + RoPE + relayout chain (transformer.py:731-767,842-867 + megatron
apply_rotary_pos_emb), and the vocab-parallel cross entropy (cross_entropy.py:14-152).

The rule for a bf16 output: it is the correctly rounded float64 value, up to the kernel's fp32 evaluation error,
    |got - ref| <= 1/2 ulp_bf16 + eps_fp32,
where eps_fp32 is derived, next to each assertion, from the formula the kernel evaluates: every fp32 rounding contributes
u = 2^-24 times the magnitude of what it rounds, a block-wide sum over D levels contributes D u times the sum of the magnitudes of
its terms, and CUDA's documented bounds hold for the library functions (rsqrtf, tanhf, erff: 2 ulp; __expf: 2 + floor(1.173 |x|)
ulp; an fp32 ulp is at most 2 u relative).  fp32 outputs get bounds of the same kind.  A kernel that truncates instead of
rounding to nearest even, or is off by one bf16 ulp, fails.  Every output buffer starts as NaN, so an element the kernel does not
write fails too."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _fp_check import BF, F64, U, _bits, assert_rounded, assert_within, gamma, ulp_f32  # noqa: E402
pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
NAN = float("nan")


@pytest.fixture(scope="module")
def bg():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import hetu_galvatron_b200._bg as bg
    bg.lib()
    return bg


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, NAN, device="cuda", dtype=dtype)


def _f32_rel(c):
    """relative difference between the fp32 literal a kernel uses and the exact constant c"""
    return abs(float(np.float32(c)) - c) / abs(c)


def _tree_depth(cols, threads=256, per_vec=8):
    """additions on the longest path of a block-wide fp32 sum over a row of `cols`: a thread adds its up to
    ceil(cols / (per_vec * threads)) vectors of per_vec terms one by one, then two 32-lane butterflies add 5 levels each"""
    return per_vec * -(-cols // (per_vec * threads)) + 10


def _with_local_ctas(bg, n, fn):
    old = bg.get_tunable("local_ctas")
    try:
        bg.set_tunable("local_ctas", n)
        return fn()
    finally:
        bg.set_tunable("local_ctas", old)


@pytest.mark.parametrize("n,scale,acc", [(8, 1.0, False), (4096 * 8 + 8, 0.5, True), (1 << 22, 1.0, False)])
@pytest.mark.parametrize("sd,dd", [(torch.float32, BF), (BF, torch.float32), (BF, BF), (torch.float32, torch.float32)])
def test_cast(bg, n, scale, acc, sd, dd):
    src = (torch.randn(n, device="cuda") * 2).to(sd)
    dst0 = torch.randn(n, device="cuda").to(dd) if acc else _nan(n, dtype=dd)
    dst = dst0.clone()
    bg.cast(src, dst, scale=scale, accumulate=acc)
    prod = src.double() * scale
    ref = prod + (dst0.double() if acc else 0)
    if dd == BF and not acc and scale == 1.0:
        assert torch.equal(dst.view(torch.int16), src.to(BF).view(torch.int16))
    elif dd == BF:
        # fl(fl(src * scale) + dst0): one rounding of the product, one of the sum
        assert_rounded(dst, ref, U * prod.abs() + U * ref.abs())
    else:
        torch.testing.assert_close(dst, ref.float(), rtol=1e-6, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------------------------
# RMSNorm
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols", [(1, 8), (37, 128), (1000, 4096), (64, 8192), (50, 3072), (301, 5120), (2500, 2048)])
def test_rmsnorm_fwd_bwd(bg, rows, cols):
    eps = 1e-5
    x = torch.randn(rows, cols, device="cuda").to(BF)
    w = (1 + 0.1 * torch.randn(cols, device="cuda")).to(BF)
    dy = torch.randn(rows, cols, device="cuda").to(BF)
    y, rstd = _nan(rows, cols, dtype=BF), _nan(rows)
    bg.check(bg.lib().bg_rmsnorm_fwd(_p(x), _p(w), _p(y), _p(rstd), rows, cols, eps, _s()))
    D = _tree_depth(cols)
    xd, wd, gd = x.double(), w.double(), dy.double()
    ms = xd.pow(2).mean(-1, keepdim=True) + float(np.float32(eps))
    r = ms.rsqrt()
    # ms: squares (1 rounding) summed over D levels, / n, + eps -> gamma(D + 3) relative (all terms >= 0);
    # rsqrtf: half of that plus its own 2 ulp (4 u)
    dr = gamma(D + 3) / 2 + 4 * U
    assert_within(rstd, r.squeeze(-1), dr * r.squeeze(-1), "rstd")
    yr = xd * r * wd
    # y = x * rstd * w: rstd's error and two roundings
    assert_rounded(y, yr, yr.abs() * (dr + gamma(3)), "y")

    # backward from the kernel's own rstd (an input of the backward kernel)
    npart = 64
    rk = rstd.double()[:, None]
    xh = xd * rk
    gw = gd * wd
    dot = (gw * xh).mean(-1, keepdim=True)
    dxr = rk * (gw - xh * dot)
    dx, dwp = _nan(rows, cols, dtype=BF), _nan(npart, cols)
    bg.check(bg.lib().bg_rmsnorm_bwd(_p(dy), _p(x), _p(w), _p(rstd), _p(dx), _p(dwp), rows, cols, npart, _s()))
    # dot: terms g*w*xhat (3 roundings) summed over D levels, / n (1); dx = rstd * (g*w - x*rstd*dot): cancellation is inherent,
    # so the slack is absolute, u times the magnitudes of the terms
    ddot = gamma(D + 4) * (gw * xh).abs().mean(-1, keepdim=True)
    assert_rounded(dx, dxr, rk * (gamma(3) * (gw.abs() + (xh * dot).abs()) + xh.abs() * ddot), "dx")
    # dw: each CTA adds dy * xhat (2 roundings) of its <= ceil(rows / npart) rows one by one; the partials are added here in fp64
    k = -(-rows // npart)
    terms = gd * xh
    assert_within(dwp.double().sum(0), terms.sum(0), gamma(k + 2) * terms.abs().sum(0), "dw")
    assert not dwp[rows:].any()


# ---------------------------------------------------------------------------------------------------------------------------
# LayerNorm with bias
# ---------------------------------------------------------------------------------------------------------------------------
def _ln_inputs(kind, rows, cols):
    if kind == "normal":
        return torch.randn(rows, cols, device="cuda").to(BF)
    if kind == "offset":      # a one-pass E[x^2] - mean^2 variance loses every digit here; the two-pass one does not
        return (300 + 0.5 * torch.randn(rows, cols, device="cuda")).to(BF)
    return torch.randn(rows, 1, device="cuda").to(BF).expand(rows, cols).contiguous()     # constant rows: variance 0


def _ln_fwd(bg, x, w, b, eps):
    rows, cols = x.shape
    y, mean, rstd = _nan(rows, cols, dtype=BF), _nan(rows), _nan(rows)
    bg.check(bg.lib().bg_layernorm_fwd(_p(x), _p(w), _p(b), _p(y), _p(mean), _p(rstd), rows, cols, eps, _s()))
    return y, mean, rstd


def _ln_bwd(bg, dy, x, w, mean, rstd, npart):
    rows, cols = x.shape
    dx, dwp, dbp = _nan(rows, cols, dtype=BF), _nan(npart, cols), _nan(npart, cols)
    bg.check(bg.lib().bg_layernorm_bwd(_p(dy), _p(x), _p(w), _p(mean), _p(rstd), _p(dx), _p(dwp), _p(dbp), rows, cols, npart, _s()))
    return dx, dwp, dbp


@pytest.mark.parametrize("eps", [1e-5, 1e-12])
@pytest.mark.parametrize("rows,cols", [(1, 8), (8192, 768), (8192, 1024), (1057, 4096), (3, 1600), (5, 2056), (64, 8192)])
def test_layernorm_fwd_bwd(bg, rows, cols, eps):
    """GPT-2 small (h 768, bsz 8 x seq 1024), BERT-large (h 1024), 6.7B (h 4096, one row more than local_ctas CTAs), odd and
    ragged widths (257 vectors: one thread owns a second one) and the widest row; eps of GPT (1e-5) and of BERT (1e-12)."""
    n = cols
    D = _tree_depth(cols)
    e32 = float(np.float32(eps))
    g = torch.Generator(device="cuda").manual_seed(rows * 7 + cols)
    w = (1 + 0.1 * torch.randn(cols, device="cuda", generator=g)).to(BF)
    b = (0.1 * torch.randn(cols, device="cuda", generator=g)).to(BF)
    wd, bd = w.double(), b.double()
    for kind in ("normal", "offset", "constant"):
        x = _ln_inputs(kind, rows, cols)
        dy = torch.randn(rows, cols, device="cuda").to(BF)
        y, mean, rstd = _ln_fwd(bg, x, w, b, eps)
        # the launch geometry does not change a bit: one CTA owns a row, its reduction tree is fixed
        y3, mean3, rstd3 = _with_local_ctas(bg, 3, lambda: _ln_fwd(bg, x, w, b, eps))
        for got, again in ((y, y3), (mean, mean3), (rstd, rstd3)):
            assert torch.equal(_bits(got), _bits(again)), kind

        xd = x.double()
        m = xd.mean(-1, keepdim=True)
        var = (xd - m).pow(2).mean(-1, keepdim=True)
        r = (var + e32).rsqrt()
        # mean = fl(sum) * fl(1/n): the sum over D levels errs by gamma(D) sum|x|, the scaling by 2 roundings
        dm = gamma(D) * xd.abs().mean(-1, keepdim=True) + gamma(2) * m.abs()
        # variance: (x - mean)^2 (3 roundings with the subtraction) summed over D levels, * fl(1/n), + eps -> gamma(D + 6)
        # relative, plus the shift dm^2 that the kernel's mean adds to the sum of squares; rsqrtf: half of it plus 2 ulp (4 u)
        dv = (gamma(D + 6) * (var + dm * dm + e32) + dm * dm) / (var + e32)
        dr = dv / 2 + 4 * U
        assert_within(mean, m.squeeze(-1), dm.squeeze(-1), f"{kind} mean")
        assert_within(rstd, r.squeeze(-1), (dr * r).squeeze(-1), f"{kind} rstd")
        t = (xd - m) * r * wd
        yr = t + bd
        # y = fl(fl(fl(x - mean) * rstd) * w) + b: the mean's error scaled by rstd * w, rstd's relative error on t, 4 roundings
        em = wd.abs() * r * dm
        assert_rounded(y, yr, (em + t.abs() * dr) * (1 + gamma(3)) + gamma(4) * (t.abs() + em + yr.abs()), f"{kind} y")
        if kind == "constant":
            # the fp32 sum of a constant bf16 row is exact and sum * fl(1/n) gives the value back: x - mean is exactly 0
            assert torch.equal(mean, x[:, 0].float()), kind
            assert torch.equal(_bits(y), _bits(b.expand(rows, cols))), kind
            r0 = torch.full_like(rstd, e32, dtype=F64).rsqrt()
            assert ((rstd.double() - r0).abs() <= 2 * ulp_f32(r0)).all(), (rstd[:4], r0[:4])       # rsqrtf: 2 ulp
        del xd, m, var, r, t, yr, em

        # backward from the kernel's mean and rstd (inputs of the backward kernel)
        xd, gd = x.double(), dy.double()
        mk, rk = mean.double()[:, None], rstd.double()[:, None]
        xh = (xd - mk) * rk
        gw = gd * wd
        s1 = gw.mean(-1, keepdim=True)
        s2 = (gw * xh).mean(-1, keepdim=True)
        dxr = rk * (gw - s1 - xh * s2)
        # s1: terms g*w (1 rounding) over D levels, * fl(1/n) (2); s2: terms g*w*xhat (4 with xhat's 2) over D levels, * fl(1/n)
        ds1 = gamma(D + 3) * gw.abs().mean(-1, keepdim=True)
        ds2 = gamma(D + 6) * (gw * xh).abs().mean(-1, keepdim=True)
        # dx = rstd * (g*w - s1 - xhat * s2): cancellation is inherent, the slack is absolute: u times the terms' magnitudes,
        # plus the reductions' errors
        edx = rk * (gamma(3) * (gw.abs() + s1.abs()) + gamma(4) * (xh * s2).abs() + ds1 + xh.abs() * ds2)
        dwr, dbr = (gd * xh).sum(0), gd.sum(0)
        dws, dbs = (gd * xh).abs().sum(0), gd.abs().sum(0)
        dx0 = None
        for npart in (1, 7, 396, rows + 5):
            dx, dwp, dbp = _ln_bwd(bg, dy, x, w, mean, rstd, npart)
            if dx0 is None:
                assert_rounded(dx, dxr, edx, f"{kind} dx")
                dx0 = dx
            else:           # one CTA owns a row and its reduction tree is fixed: the number of CTAs does not change a bit
                assert torch.equal(_bits(dx), _bits(dx0)), (kind, npart)
            # a CTA adds the dy * xhat (3 roundings with xhat's 2) and dy of its <= ceil(rows / npart) rows one by one;
            # the bound scales with the column sums of |terms|.  The partials are added here in fp64.
            k = -(-rows // npart)
            assert_within(dwp.double().sum(0), dwr, gamma(k + 3) * dws, f"{kind} dw, {npart} partials")
            assert_within(dbp.double().sum(0), dbr, gamma(k) * dbs, f"{kind} db, {npart} partials")
            if npart > rows:                    # CTAs that visit no row write zeros
                assert not dwp[rows:].any() and not dbp[rows:].any(), (kind, npart)
        del xd, gd, mk, rk, xh, gw, s1, s2, dxr, edx, ds1, ds2
    torch.cuda.empty_cache()


def test_layernorm_bwd_without_rows(bg):
    """rows = 0: nothing to normalise, but every partial row is written, with zeros."""
    cols = 1024
    x = torch.empty(0, cols, device="cuda", dtype=BF)
    w = torch.ones(cols, device="cuda", dtype=BF)
    for npart in (1, 5):
        dx, dwp, dbp = _ln_bwd(bg, x, x, w, _nan(0), _nan(0), npart)
        torch.cuda.synchronize()
        assert torch.equal(dwp, torch.zeros_like(dwp)) and torch.equal(dbp, torch.zeros_like(dbp)), npart


# ---------------------------------------------------------------------------------------------------------------------------
# bias + GeLU
# ---------------------------------------------------------------------------------------------------------------------------
_C_TANH = math.sqrt(2 / math.pi)       # the kernel's 0.79788456f
_A_TANH = 0.044715
_B_TANH = 3 * _A_TANH * _C_TANH       # the kernel's 0.1070322243f
_C_ERF = 1 / math.sqrt(2)              # 0.70710678f
_C_PDF = 1 / math.sqrt(2 * math.pi)    # 0.3989422804f


def _gelu64(v, tanh_form):
    return F.gelu(v, approximate="tanh" if tanh_form else "none")


def _dgelu64(v, tanh_form):
    v = v.detach().requires_grad_(True)
    return torch.autograd.grad(_gelu64(v, tanh_form), v, torch.ones_like(v))[0]


def _input_slack(f, v):
    """the output's change when v = x + b moves by its fp32 rounding (u |v|): the propagated error of that rounding"""
    h = U * v.abs()
    f0 = f(v)
    return torch.maximum((f(v + h) - f0).abs(), (f(v - h) - f0).abs())


def _gelu_eps(v, dy, tanh_form, rounded_input):
    """fp32 evaluation error of the kernel's gelu (dy None) or dy * gelu' at the float64 v (see GeluTanh / GeluErf in bg_ops.cu)."""
    av = v.abs()
    if tanh_form:
        # z = c*v*(1 + a*v*v): 5 roundings and the two fp32 literals; t = tanhf(z): its 2 ulp (4 u) plus z's error through tanh'
        z = _C_TANH * v * (1 + _A_TANH * v * v)
        t = torch.tanh(z)
        dt = (1 - t * t) * z.abs() * (_f32_rel(_C_TANH) + _f32_rel(_A_TANH) + gamma(5)) + 4 * U * t.abs()
        if dy is None:
            # v*0.5*(1 + t): the sum and the product round once each; in the negative tail 1 + t cancels (absolute slack)
            y = 0.5 * v * (1 + t)
            eps = 0.5 * av * (dt + U * (1 + t).abs()) + U * y.abs()
        else:
            # 0.5*v*((1 - t*t)*(c + b*v*v)) + 0.5*(1 + t)
            a_ = 1 - t * t
            bb = _C_TANH + _B_TANH * v * v
            da = 2 * t.abs() * dt + U * (t * t + a_.abs())
            db = _C_TANH * _f32_rel(_C_TANH) + _B_TANH * v * v * (_f32_rel(_B_TANH) + gamma(2)) + U * bb
            d1 = 0.5 * av * (da * bb + a_ * db + gamma(2) * a_ * bb)
            d2 = 0.5 * (dt + U * (1 + t).abs())
            gp = 0.5 * v * a_ * bb + 0.5 * (1 + t)
            eps = dy.abs() * (d1 + d2 + gamma(2) * gp.abs())
    else:
        # e = erff(v*c): its 2 ulp (4 u) plus the argument's 2 roundings (literal + product) through erf'
        al = _C_ERF * v
        e = torch.erf(al)
        de = 2 / math.sqrt(math.pi) * torch.exp(-al * al) * al.abs() * (_f32_rel(_C_ERF) + U) + 4 * U * e.abs()
        if dy is None:
            y = 0.5 * v * (1 + e)
            eps = 0.5 * av * (de + U * (1 + e).abs()) + U * y.abs()
        else:
            # 0.5*(1 + e) + v*c'*__expf(-0.5*v*v): __expf's 2 + floor(1.173 |w|) ulp and its argument's rounding (|w| u)
            w = 0.5 * v * v
            t2 = _C_PDF * av * torch.exp(-w)
            dexp = 2 * U * (2 + torch.floor(1.173 * w)) + U * w
            gp = 0.5 * (1 + e) - t2 * torch.sign(-v)
            eps = dy.abs() * (0.5 * (de + U * (1 + e).abs()) + t2 * (_f32_rel(_C_PDF) + gamma(2) + dexp) + gamma(2) * gp.abs())
    if rounded_input:
        f = (lambda u_: _gelu64(u_, tanh_form)) if dy is None else (lambda u_: dy * _dgelu64(u_, tanh_form))
        eps = eps + _input_slack(f, v)
    return eps


def _bias_gelu(bg, x, bias, dy, tanh_form):
    out = _nan(*x.shape, dtype=BF)
    bg.check(bg.lib().bg_bias_gelu(_p(x), _p(bias) if bias is not None else None, _p(dy) if dy is not None else None, _p(out),
                                   x.shape[0], x.shape[1], 1 if tanh_form else 0, _s()))
    return out


@pytest.mark.parametrize("tanh_form", [True, False], ids=["tanh", "erf"])
@pytest.mark.parametrize("rows,cols", [(1, 8), (3, 24), (8192, 3072), (8192, 4096), (2048, 8192), (1000, 16384)])
def test_bias_gelu(bg, rows, cols, tanh_form):
    """GPT-2 small / BERT-large / 6.7B-at-tp-2 / 6.7B ffn widths and a ragged row (3 vectors of 8).  x + b walks a deterministic
    grid over [-12.5, 12.5] with an exact 0: the negative tail [-6, -2] is the only region where the tanh and the erf form
    differ by more than half a bf16 ulp, so a grid is what tells the forms apart."""
    N = rows * cols
    grid = torch.linspace(-12, 12, N, device="cuda", dtype=F64).to(BF).view(rows, cols)
    col = torch.arange(cols, device="cuda", dtype=F64)
    bias = (0.5 * torch.sin(0.7 * col + 0.3)).to(BF)       # distinct per column and per 8-column vector
    dy = torch.randn(rows, cols, device="cuda").to(BF)
    for b in (bias, None):
        x = grid.clone()
        mid = (rows // 2, cols // 2)
        x[mid] = -b[mid[1]] if b is not None else 0.0      # x + b == 0 exactly
        y = _bias_gelu(bg, x, b, None, tanh_form)
        dx = _bias_gelu(bg, x, b, dy, tanh_form)
        y7 = _with_local_ctas(bg, 7, lambda: _bias_gelu(bg, x, b, None, tanh_form))
        dx7 = _with_local_ctas(bg, 7, lambda: _bias_gelu(bg, x, b, dy, tanh_form))
        assert torch.equal(_bits(y), _bits(y7)) and torch.equal(_bits(dx), _bits(dx7))     # the grid does not change a bit
        what = "%s, bias %s" % ("tanh" if tanh_form else "erf", "bf16" if b is not None else "none")
        chunk = max(1, (1 << 21) // cols)          # float64 reference and bound a slice of rows at a time
        for r0 in range(0, rows, chunk):
            sl = slice(r0, r0 + chunk)
            v = x[sl].double() + (b.double() if b is not None else 0.0)
            gd = dy[sl].double()
            assert_rounded(y[sl], _gelu64(v, tanh_form), _gelu_eps(v, None, tanh_form, b is not None), what + " forward")
            assert_rounded(dx[sl], gd * _dgelu64(v, tanh_form), _gelu_eps(v, gd, tanh_form, b is not None), what + " backward")
        assert y[mid].item() == 0.0 and dx[mid].item() == 0.5 * dy[mid].item()   # gelu(0) = 0, gelu'(0) = 1/2 in both forms
        del v, gd
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------------
# swiglu
# ---------------------------------------------------------------------------------------------------------------------------
def _expf_rel(x):
    """relative error bound of __expf(x): 2 + floor(1.173 |x|) fp32 ulp (CUDA's intrinsic bound), an ulp <= 2 u relative"""
    return 2 * U * (2 + torch.floor(1.173 * x.abs()))


@pytest.mark.parametrize("rows,ffn", [(1, 8), (33, 256), (2048, 14336), (3, 1792), (4097, 3584)])
def test_swiglu(bg, rows, ffn):
    gu = torch.randn(rows, 2 * ffn, device="cuda").to(BF)
    dy = torch.randn(rows, ffn, device="cuda").to(BF)
    y = _nan(rows, ffn, dtype=BF)
    bg.check(bg.lib().bg_swiglu_fwd(_p(gu), _p(y), rows, ffn, _s()))
    g, u = torch.chunk(gu.double(), 2, dim=-1)
    d = dy.double()
    sg = torch.sigmoid(g)
    sm = torch.sigmoid(-g)                   # e / (1 + e) with e = exp(-g): how 1 + e passes on e's relative error
    # sigmoid = 1 / (1 + __expf(-g)): __expf's error through 1 + e, plus the sum's and the division's roundings
    dsg = sm * _expf_rel(g) + gamma(2)
    yr = g * sg * u
    # y = fl(fl(g / fl(1 + e)) * u)
    assert_rounded(y, yr, yr.abs() * (dsg + gamma(1)), "y")
    dgu = _nan(rows, 2 * ffn, dtype=BF)
    bg.check(bg.lib().bg_swiglu_bwd(_p(dy), _p(gu), _p(dgu), rows, ffn, _s()))
    du = d * g * sg
    h = 1 - sg
    q = g * h
    dg = d * u * sg * (1 + q)
    # du = fl(fl(d * g) * sg); dg = ((d*u)*sg) * (1 + g*(1 - sg)): 1 - sg cancels for large g (absolute slack from sg's error)
    dh = sg * dsg + U * h
    p_ = (d * u * sg).abs()
    edg = p_ * (g.abs() * dh + gamma(2) * (q.abs() + (1 + q).abs())) + (dg.abs()) * (dsg + gamma(3))
    assert_rounded(dgu[:, :ffn], dg, edg, "dgate")
    assert_rounded(dgu[:, ffn:], du, du.abs() * (dsg + gamma(2)), "dup")


# ---------------------------------------------------------------------------------------------------------------------------
# QKV split + RoPE + relayout
# ---------------------------------------------------------------------------------------------------------------------------
def _rotate_half(x):
    x1, x2 = torch.chunk(x, 2, dim=-1)
    return torch.cat((-x2, x1), dim=-1)


def _ref_qkv_rope(mixed, cos, sin, ng, r, hn):
    """transformer.py:731-767 split, :853-854 apply_rotary_pos_emb (t*cos + rotate_half(t)*sin), :864 rearrange.  Also returns
    the magnitude |t*cos| + |rotate_half(t)*sin| of the two products summed per element (the rounding scale)."""
    s, b = mixed.shape[:2]
    m = mixed.view(s, b, ng, (r + 2) * hn)
    q, k, v = torch.split(m, [r * hn, hn, hn], dim=3)
    q = q.reshape(s, b, ng * r, hn)
    c = torch.cat([cos, cos], -1)[:, None, None, :]
    sn = torch.cat([sin, sin], -1)[:, None, None, :]
    mag = [(t * c).abs() + (_rotate_half(t) * sn).abs() for t in (q, k)]
    q = q * c + _rotate_half(q) * sn
    k = k * c + _rotate_half(k) * sn
    return [t.permute(1, 0, 2, 3).contiguous() for t in (q, k, v)], [t.permute(1, 0, 2, 3).contiguous() for t in mag]


@pytest.mark.parametrize("s,b,ng,r,hn", [(16, 1, 1, 1, 16), (64, 2, 2, 4, 64), (512, 1, 8, 4, 128), (40, 2, 16, 4, 128), (3000, 1, 1, 4, 128)])
def test_qkv_rope_fwd_bwd(bg, s, b, ng, r, hn):
    from oracle.collectives_ref import rope_tables
    mixed = torch.randn(s, b, ng * (r + 2) * hn, device="cuda").to(BF)
    cos, sin = [t.cuda().contiguous() for t in rope_tables(s, hn, offset=3)]
    q = _nan(b, s, ng * r, hn, dtype=BF)
    k = _nan(b, s, ng, hn, dtype=BF)
    v = _nan(b, s, ng, hn, dtype=BF)
    bg.check(bg.lib().bg_qkv_rope(_p(mixed), _p(q), _p(k), _p(v), _p(cos), _p(sin), s, b, ng, r, hn, 0, _s()))
    mf = mixed.double().requires_grad_(True)
    (qf, kf, vf), (mq, mk) = _ref_qkv_rope(mf, cos.double(), sin.double(), ng, r, hn)
    # a*cos -/+ b*sin: two products and a sum, each rounded once
    assert_rounded(q, qf.detach(), gamma(2) * mq.detach(), "q")
    assert_rounded(k, kf.detach(), gamma(2) * mk.detach(), "k")
    assert torch.equal(v.view(torch.int16), vf.detach().to(BF).view(torch.int16))
    dq, dk, dv = [torch.randn_like(t).to(BF) for t in (qf, kf, vf)]
    ((qf * dq.double()).sum() + (kf * dk.double()).sum() + (vf * dv.double()).sum()).backward()
    # the transpose rotates by -theta: the same two products per element, so the same bound, from |dq| and |dk|
    with torch.no_grad():
        mg = torch.zeros_like(mf)
        c = torch.cat([cos, cos], -1).double()[:, None, None, :]
        sn = torch.cat([sin, sin], -1).double()[:, None, None, :]
        mv = mg.view(s, b, ng, (r + 2) * hn)
        for t, lo, hi in ((dq.double().permute(1, 0, 2, 3).reshape(s, b, ng, r * hn), 0, r * hn),
                          (dk.double().permute(1, 0, 2, 3).reshape(s, b, ng, hn), r * hn, (r + 1) * hn)):
            tt = t.view(s, b, ng, -1, hn)
            mv[..., lo:hi] = ((tt * c[:, :, :, None]).abs() + (_rotate_half(tt) * sn[:, :, :, None]).abs()).view(s, b, ng, hi - lo)
    dm = _nan(*mixed.shape, dtype=BF)
    bg.check(bg.lib().bg_qkv_rope(_p(dm), _p(dq), _p(dk), _p(dv), _p(cos), _p(sin), s, b, ng, r, hn, 1, _s()))
    assert_rounded(dm, mf.grad, gamma(2) * mg, "dmixed")


# ---------------------------------------------------------------------------------------------------------------------------
# vocab-parallel cross entropy
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,vocab,parts", [(5, 64, 1), (64, 1000 * 8, 4), (512, 128256, 1), (128, 128256, 8)])
@pytest.mark.parametrize("dtype", [BF, torch.float32])
def test_vocab_parallel_cross_entropy(bg, rows, vocab, parts, dtype):
    """`parts` vocab shards handled sequentially on one device: the MAX / SUM all-reduces between the kernels are
    done here with torch, exactly where cross_entropy.py:22-30 / :61-89 puts them.  Random targets, then targets pinned to the
    first and the last column of every shard and to the last vocab id -- where `target - vocab_start` indexing goes wrong."""
    vl = vocab // parts
    edges = sorted({e for i in range(parts) for e in (i * vl, i * vl + vl - 1)} | {vocab - 1})
    for target in (torch.randint(0, vocab, (rows,), device="cuda"),
                   torch.tensor(edges, device="cuda").repeat(-(-rows // len(edges)))[:rows].contiguous()):
        _cross_entropy_case(bg, rows, vocab, parts, dtype, target)


def _expf_arg_rel(xs):
    """relative error of __expf(fl(x - max)): __expf's own bound and the subtraction's rounding (|x - max| u), which is not exact
    even for bf16 logits (a small logit minus a large max needs more than 24 significant bits)"""
    return _expf_rel(xs) + U * xs.abs()


def _cross_entropy_case(bg, rows, vocab, parts, dtype, target):
    L = bg.lib()
    vl = vocab // parts
    logits = (torch.randn(rows, vocab, device="cuda") * 3).to(dtype)
    shards = [logits[:, i * vl:(i + 1) * vl].contiguous() for i in range(parts)]
    code = bg.dtype_code(dtype)
    E = 8 if dtype == BF else 4
    D = E * -(-vl // (E * 512)) + 10            # the block-wide sums: 512 threads, E elements per 16-B vector
    maxes = []
    for sh in shards:
        m = _nan(rows)
        bg.check(L.bg_ce_rowmax(_p(sh), code, _p(m), rows, vl, _s()))
        maxes.append(m)
    gmax = torch.stack(maxes).max(0).values
    assert torch.equal(gmax, logits.float().max(-1).values)
    outs = []
    for i, sh in enumerate(shards):
        o = _nan(rows, 2)
        bg.check(L.bg_ce_sumexp(_p(sh), code, _p(target), _p(gmax), _p(o), rows, vl, i * vl, _s()))
        outs.append(o)
        xs = sh.double() - gmax.double()[:, None]
        es = xs.exp()
        # the terms exp(x - max), each within its __expf bound, summed over D levels
        rel = _expf_arg_rel(xs)
        assert_within(o[:, 0], es.sum(-1), (es * (rel + gamma(D) * (1 + rel))).sum(-1), f"shard {i} sum")
        local = target - i * vl
        mine = (local >= 0) & (local < vl)
        pred = torch.where(mine, xs.gather(1, local.clamp(0, vl - 1)[:, None]).squeeze(1), torch.zeros_like(xs[:, 0]))
        # target logit - max: one rounding; exactly 0 when the target is outside this shard
        assert_within(o[:, 1], pred, U * pred.abs(), f"shard {i} target logit")
        assert torch.equal(o[~mine, 1], torch.zeros_like(o[~mine, 1]))
    tot = torch.stack(outs).sum(0).contiguous()
    loss = torch.log(tot[:, 0]) - tot[:, 1]
    ld = logits.double()
    want = F.cross_entropy(ld, target, reduction="none")
    torch.testing.assert_close(loss.double(), want, rtol=2e-5, atol=2e-5)
    gl = torch.rand(rows, device="cuda")
    for i, sh in enumerate(shards):
        bg.check(L.bg_ce_bwd(_p(sh), code, _p(target), _p(gmax), _p(tot), _p(gl), rows, vl, i * vl, _s()))
        # from the kernel's inputs: max, the summed (sum, target logit) pairs and grad_loss
        xs = ld[:, i * vl:(i + 1) * vl] - gmax.double()[:, None]
        p = xs.exp() / tot[:, 0].double()[:, None]
        local = target - i * vl
        mine = (local >= 0) & (local < vl)
        oh = torch.zeros_like(p)
        oh[mine.nonzero().squeeze(1), local[mine]] = 1.0
        g = gl.double()[:, None]
        ref = (p - oh) * g
        # p = __expf(x - max) * fl(1/sum): __expf's bound and 2 roundings; p - 1 and * g round once each (p - 1 cancels: absolute)
        eps = g.abs() * (p * (_expf_arg_rel(xs) + gamma(2)) + U * (p - oh).abs()) + U * ref.abs()
        if dtype == BF:
            assert_rounded(sh, ref, eps, f"shard {i} dlogits")
        else:
            assert_within(sh, ref, eps, f"shard {i} dlogits")

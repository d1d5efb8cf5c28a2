"""The ViT family on the GPU: its four kernels against exact references, their argument checks, and the family through the CUDA backend.

Kernels (through the C ABI), at ViT-B / ViT-H widths (768, 1280), b in {1, 3, 8, 80} and s_run in {197, 200}:
  * bg_vit_patchify: the einops relayout "b c (h p1) (w p2) -> b (h w) (p1 p2 c)" bit for bit (fp32 pixels rounded once), zero tails;
  * bg_vit_embed_fwd: the float64 sum correctly rounded to bf16 up to its two fp32 roundings, padding rows zero, and with dropout on
    exactly the mask bg_dropout_add_fwd draws at the same (seed, iteration, site, token, sample) coordinates;
  * bg_vit_embed_bwd: dpatch bit-exact (bg_dropout_bwd's dx with dropout), the column sums within fp32 summation error of float64,
    padding-token rows of dy never read (they hold NaN here);
  * bg_bias_tanh forward and backward against float64 (tests/_fp_check.py's rule).
Bad arguments return BG_EINVAL / BG_EUNSUPPORTED before any launch (checked in a child process that sees no device)."""
import ctypes
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _fp_check import BF, F64, U, assert_rounded, assert_within, gamma  # noqa: E402

gpu = pytest.mark.gpu
NAN = float("nan")
SEED, ITER, SITE = 1234, 7, 0


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


def _ceil8(n):
    return (n + 7) // 8 * 8


def _einops(pixels, patch):
    b, c, hgt, wid = pixels.shape
    x = pixels.reshape(b, c, hgt // patch, patch, wid // patch, patch).permute(0, 2, 4, 3, 5, 1)
    return x.reshape(b * (hgt // patch) * (wid // patch), patch * patch * c)


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("b,c,img,patch", [(1, 3, 224, 16), (3, 3, 224, 16), (8, 3, 224, 16), (5, 3, 32, 8), (2, 8, 16, 4)])
def test_patchify_is_the_einops_relayout(bg, dtype, b, c, img, patch):
    g = torch.Generator(device="cuda").manual_seed(b * 31 + img)
    pixels = torch.randn(b, c, img, img, device="cuda", generator=g).to(dtype)
    n = b * (img // patch) ** 2
    rows_pad = _ceil8(n) + 8                     # (one more block of 8: the tail must be written, whatever its length)
    out = torch.full((rows_pad, patch * patch * c), NAN, device="cuda", dtype=BF)
    bg.check(bg.lib().bg_vit_patchify(_p(pixels), bg.dtype_code(dtype), _p(out), b, c, img, img, patch, rows_pad, _s()))
    torch.cuda.synchronize()
    want = _einops(pixels, patch).to(BF)
    assert torch.equal(out[:n].view(torch.int16), want.view(torch.int16))
    assert torch.equal(out[n:], torch.zeros_like(out[n:]))


def _embed_inputs(b, h, n_patches, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rows_pad = _ceil8(b * n_patches)
    r = lambda *shape: torch.randn(*shape, device="cuda", generator=g).to(BF)  # noqa: E731
    return r(rows_pad, h), r(h), r(h), r(n_patches + 1, h), rows_pad


def _keep_mask(bg, s_run, b, h, p, sample_base):
    """bg_dropout_add_fwd on ones: scale where kept, 0 where dropped -> bool [s_run, b, h]"""
    ones = torch.ones(s_run, b, h, device="cuda", dtype=BF)
    y = torch.empty_like(ones)
    bg.check(bg.lib().bg_dropout_add_fwd(_p(ones), None, 0, None, _p(y), s_run * b, h, b, 0, sample_base, p, SEED, ITER, SITE, _s()))
    return y != 0


SHAPES = [(h, b, s_run) for h in (768, 1280) for b in (1, 3, 8, 80) for s_run in (197, 200)]


@gpu
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("h,b,s_run", SHAPES)
def test_embed_fwd_is_the_rounded_sum(bg, h, b, s_run, p):
    n_patches, sample_base = 196, 5
    patch, bias, cls, pos, _ = _embed_inputs(b, h, n_patches, h + b + s_run)
    y = torch.full((s_run, b, h), NAN, device="cuda", dtype=BF)
    bg.check(bg.lib().bg_vit_embed_fwd(_p(patch), _p(bias), _p(cls), _p(pos), _p(y), b, n_patches, s_run, h, sample_base, p, SEED, ITER,
                                       SITE, _s()))
    torch.cuda.synchronize()
    S = n_patches + 1
    pd, bd, cd, qd = patch.double(), bias.double(), cls.double(), pos.double()
    ref = torch.empty(S, b, h, dtype=F64, device="cuda")
    mag = torch.empty_like(ref)
    ref[0] = qd[0] + cd
    mag[0] = qd[0].abs() + cd.abs()
    rows = pd[:b * n_patches].view(b, n_patches, h).transpose(0, 1)
    ref[1:] = rows + (qd[1:] + bd)[:, None]
    mag[1:] = rows.abs() + (qd[1:].abs() + bd.abs())[:, None]
    eps = gamma(2) * mag                                  # (pos + bias) rounded in fp32, then + patch rounded in fp32
    if p > 0:
        keep = _keep_mask(bg, s_run, b, h, p, sample_base)[:S]
        scale = float(torch.tensor(1.0 / (1.0 - p), dtype=torch.float32))
        # dropped elements are 0 and kept ones the scaled sum (checked below), so a mask that differs from bg_dropout_add_fwd's
        # fails wherever the sum is not exactly 0 (random bf16 inputs do sum to exactly 0 now and then: y != 0 is not the mask)
        assert not y[:S][~keep].any(), "an element bg_dropout_add_fwd drops is kept"
        ref = torch.where(keep, ref * scale, torch.zeros_like(ref))
        eps = torch.where(keep, gamma(3) * mag * scale, torch.zeros_like(eps))
    assert_rounded(y[:S], ref, eps, "embed_fwd h %d b %d" % (h, b))
    assert torch.equal(y[S:], torch.zeros_like(y[S:]))


@gpu
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("h,b,s_run", SHAPES)
def test_embed_bwd_sums_and_dpatch(bg, h, b, s_run, p):
    n_patches, sample_base, S = 196, 3, 197
    rows_pad = _ceil8(b * n_patches) + 8
    g = torch.Generator(device="cuda").manual_seed(7 * h + b + s_run)
    dy = torch.randn(s_run, b, h, device="cuda", generator=g).to(BF)
    dy[S:] = NAN                                          # padding tokens: never read
    dpatch = torch.full((rows_pad, h), NAN, device="cuda", dtype=BF)
    dpos = torch.full((S, h), NAN, device="cuda")
    npart = 17
    dbp = torch.full((npart, h), NAN, device="cuda")
    bg.check(bg.lib().bg_vit_embed_bwd(_p(dy), _p(dpatch), _p(dpos), _p(dbp), npart, b, n_patches, s_run, rows_pad, h, sample_base, p, SEED,
                                       ITER, SITE, _s()))
    torch.cuda.synchronize()
    if p > 0:       # g = bg_dropout_bwd's dx at the same coordinates (bit for bit)
        gdx = torch.empty(S, b, h, device="cuda", dtype=BF)
        bg.check(bg.lib().bg_dropout_bwd(_p(dy), _p(gdx), None, 1, S * b, h, b, 0, sample_base, p, SEED, ITER, SITE, _s()))
        keep = _keep_mask(bg, S, b, h, p, sample_base)
        scale = float(torch.tensor(1.0 / (1.0 - p), dtype=torch.float32))
        gd = torch.where(keep, dy[:S].float() * scale, torch.zeros((), device="cuda")).double()   # the fp32 values the sums add
    else:
        gdx, gd = dy[:S], dy[:S].double()
    n = b * n_patches
    assert torch.equal(dpatch[:n].view(torch.int16), gdx[1:].transpose(0, 1).reshape(n, h).view(torch.int16))
    assert torch.equal(dpatch[n:], torch.zeros_like(dpatch[n:]))
    ref_pos, mag_pos = gd.sum(1), gd.abs().sum(1)
    assert_within(dpos, ref_pos, gamma(max(b - 1, 1)) * mag_pos, "dpos h %d b %d" % (h, b))
    dbias = dbp.double().sum(0)                          # (the caller's sum of the partials, here in float64)
    assert_within(dbias, ref_pos[1:].sum(0), gamma(b + n_patches) * mag_pos[1:].sum(0), "dbias h %d b %d" % (h, b))


@gpu
@pytest.mark.parametrize("backward", [False, True], ids=["fwd", "bwd"])
@pytest.mark.parametrize("rows,cols", [(8, 768), (8, 1280), (80, 768), (80, 1280), (24, 64)])
def test_bias_tanh_against_float64(bg, rows, cols, backward):
    g = torch.Generator(device="cuda").manual_seed(rows + cols)
    x = (2 * torch.randn(rows, cols, device="cuda", generator=g)).to(BF)
    bias = torch.randn(cols, device="cuda", generator=g).to(BF)
    dy = torch.randn(rows, cols, device="cuda", generator=g).to(BF)
    out = torch.full((rows, cols), NAN, device="cuda", dtype=BF)
    bg.check(bg.lib().bg_bias_tanh(_p(x), _p(bias), _p(dy) if backward else None, _p(out), rows, cols, _s()))
    torch.cuda.synchronize()
    v = x.double() + bias.double()
    t = torch.tanh(v)
    # fp32: x + b rounded (u |v|, through tanh' <= 1), tanhf within 2 ulp (<= 4u |t|)
    dt = U * v.abs() + 4 * U * t.abs()
    if not backward:
        assert_rounded(out, t, dt, "bias_tanh fwd")
    else:
        gd = dy.double()
        # 1 - t^2 from the fp32 t: 2 |t| dt, plus the roundings of t*t, 1 - t*t and the product
        assert_rounded(out, gd * (1 - t * t), gd.abs() * (2 * t.abs() * dt + 3 * U), "bias_tanh bwd")


# ---- argument checks (no device in the child: a call that slips past validation fails at its launch) -------------------------------
_BAD_CALLS = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from hetu_galvatron_b200 import _bg
L = _bg.lib()
A, M = 0x10000, 0x10002            # a 16-B aligned and a misaligned address; neither is ever dereferenced
EINVAL, EUNSUPPORTED = -1, -7
out = []
def call(want_rc, name, *args):
    before = L.bg_launch_count()
    rc = getattr(L, name)(*args)
    out.append(dict(call="%s%r" % (name, args), got=[rc, L.bg_launch_count() - before], want=[want_rc, 0],
                    msg=L.bg_last_error().decode()))
PF, EF, EB, TH = "bg_vit_patchify", "bg_vit_embed_fwd", "bg_vit_embed_bwd", "bg_bias_tanh"
call(EUNSUPPORTED, PF, A, 2, A, 1, 3, 224, 224, 16, 200, None)           # pixel dtype
call(EINVAL, PF, A, 1, A, 1, 3, 224, 224, 15, 200, None)                 # 224 % 15
call(EINVAL, PF, A, 1, A, 0, 3, 224, 224, 16, 200, None)                 # batch 0
call(EINVAL, PF, A, 1, A, 1, 3, 12, 12, 2, 40, None)                     # p*p*C = 12
call(EINVAL, PF, A, 1, A, 1, 3, 224, 224, 16, 192, None)                 # rows_pad < 196
call(EINVAL, PF, A, 1, A, 1, 3, 224, 224, 16, 199, None)                 # rows_pad % 8
call(EINVAL, PF, 0x10001, 1, A, 1, 3, 224, 224, 16, 200, None)           # fp32 pixels misaligned
call(EINVAL, PF, A, 1, M, 1, 3, 224, 224, 16, 200, None)                 # out misaligned
E = (196, 200, 768, 0, 0.0, 1, 2, 0, None)                               # n_patches, s_run, h, sample_base, p, seed, iteration, site
for i in range(5):                                                       # patch_out, bias, cls, pos, y
    p = [A] * 5; p[i] = M
    call(EINVAL, EF, *p, 2, *E)
    p[i] = None
    call(EINVAL, EF, *p, 2, *E)
for bad in ((2, 196, 196, 768), (2, 0, 200, 768), (0, 196, 200, 768), (2, 196, 200, 12), (2, 196, 200, 0)):
    call(EINVAL, EF, A, A, A, A, A, *bad, 0, 0.0, 1, 2, 0, None)
    call(EINVAL, EB, A, A, A, A, 4, bad[0], bad[1], bad[2], 400, bad[3], 0, 0.0, 1, 2, 0, None)
for prob in (1.0, -0.1):
    call(EINVAL, EF, A, A, A, A, A, 2, 196, 200, 768, 0, prob, 1, 2, 0, None)
    call(EINVAL, EB, A, A, A, A, 4, 2, 196, 200, 392, 768, 0, prob, 1, 2, 0, None)
for i in range(4):                                                       # dy, dpatch, dpos, dbias_partial
    p = [A] * 4; p[i] = M
    call(EINVAL, EB, *p, 4, 2, 196, 200, 392, 768, 0, 0.0, 1, 2, 0, None)
for rows_pad, npart in ((390, 4), (388, 4), (392, 0), (392, 65536)):
    call(EINVAL, EB, A, A, A, A, npart, 2, 196, 200, rows_pad, 768, 0, 0.0, 1, 2, 0, None)
for i in range(4):                                                       # x, bias, dy, out
    p = [A] * 4; p[i] = M
    call(EINVAL, TH, *p, 8, 768, None)
for rows, cols in ((8, 0), (8, 12), (-1, 768)):
    call(EINVAL, TH, A, None, None, A, rows, cols, None)
print(json.dumps(out))
"""


def test_vit_kernels_reject_bad_arguments():
    """Every shape, dtype, alignment and dropout-argument error of the four ViT entries is a status code, before any launch."""
    import __graft_entry__ as ge
    from hetu_galvatron_b200 import _bg
    if not os.path.exists(_bg.LIB_PATH):
        ge.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _BAD_CALLS, ROOT], env=env, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    calls = json.loads(res.stdout.strip().splitlines()[-1])
    assert len(calls) == 8 + 10 + 10 + 4 + 4 + 4 + 4 + 3
    bad = [c for c in calls if c["got"] != c["want"]]
    assert not bad, bad


# ---- the family through the CUDA backend ---------------------------------------------------------------------------------------------
def _need(world):
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip("needs %d GPU(s)" % world)


def _cases():
    from test_vit import CASES
    cases = dict(CASES)
    # ViT/16 geometry (224 px, 196 patches + CLS = 197 tokens) at micro-batch 1: the layers run 200 tokens
    cases["vit16_geometry_microbatch1_s_run200"] = (1, dict(chunks=2, global_train_batch_size=2, _check_padded_token_grad=True,
                                                            _spec=dict(image_size=224, patch_size=16)), 200)
    return cases


CASES = _cases()


@gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(CASES))
def test_vit_family_cuda(name):
    world, cfg, s_run = CASES[name]
    _need(world)
    from test_vit import launch
    rep = launch(world, dict(cfg), backend="cuda")
    assert rep["s_run"] == s_run
    assert rep["max_grad_err"] < 3e-2
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])
    assert rep["classifier_pad_rows_max"] == 0.0
    if cfg.get("_check_padded_token_grad"):
        # the padding tokens' rows of the gradient reaching the embedding are exactly zero
        assert rep["pad_token_grad_max"] == 0.0 and rep["real_token_grad_max"] > 0.0

"""GPU parity of the wgmma/TMA GEMM (through the C ABI) against torch fp32 matmul of the same bf16 inputs.
Covers the three layouts of the Megatron linear layer (layers.py:417 fwd TN, :462 dgrad NN, :534 wgrad NT), ragged
edges (TMA zero-fill / clipping), accumulate mode, and the Llama-3-8B shapes of BASELINE config (2)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
BF = torch.bfloat16


@pytest.fixture(scope="module")
def bg():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import hetu_galvatron_b200._bg as bg
    bg.lib()
    return bg


def run(bg, layout, m, n, k, accumulate=False, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a_shape = (k, m) if layout == 2 else (m, k)
    b_shape = (n, k) if layout == 0 else (k, n)
    a = torch.randn(a_shape, device="cuda", generator=g).to(BF)
    b = torch.randn(b_shape, device="cuda", generator=g).to(BF)
    c0 = torch.randn(m, n, device="cuda", generator=g).to(BF)
    c = c0.clone()
    bg.gemm_bf16(a, b, c, m, n, k, layout, accumulate=accumulate)
    af = a.float().t() if layout == 2 else a.float()
    bf = b.float().t() if layout == 0 else b.float()
    want = af @ bf + (c0.float() if accumulate else 0)
    return c, want, k


def check(c, want, k):
    got = c.float()
    err = (got - want).abs()
    # fp32 accumulation, one bf16 rounding of the result (+ tiny slack for summation order over k)
    tol = want.abs() * 2 ** -7 + 1e-3 * (k ** 0.5)
    assert (err <= tol).all(), f"max err {float(err.max())}, bad {int((err > tol).sum())}/{err.numel()}"


@pytest.mark.parametrize("layout", [0, 1, 2])
@pytest.mark.parametrize("m,n,k", [(128, 256, 64), (256, 512, 256), (8, 8, 8), (136, 264, 72), (384, 256, 4096 + 64),
                                   (1024, 1000, 520), (2048, 768, 1792)])
def test_gemm_layouts_and_edges(bg, layout, m, n, k):
    check(*run(bg, layout, m, n, k, seed=m + n + k + layout))


@pytest.mark.parametrize("layout", [0, 1, 2])
def test_gemm_accumulate(bg, layout):
    check(*run(bg, layout, 512, 776, 320, accumulate=True, seed=5))


@pytest.mark.parametrize("layout,m,n,k", [
    (0, 8192, 6144, 4096),    # QKV projection fwd
    (0, 8192, 28672, 4096),   # gate+up fwd
    (0, 8192, 4096, 14336),   # down fwd
    (1, 8192, 4096, 6144),    # QKV dgrad
    (2, 28672, 4096, 8192),   # gate+up wgrad
    (2, 4096, 14336, 8192),   # down wgrad
])
def test_gemm_llama3_8b_shapes_vs_cublas(bg, layout, m, n, k):
    """Full BASELINE sizes: compare with torch.matmul (cuBLAS bf16, fp32 accumulate) -- both round once to bf16."""
    g = torch.Generator(device="cuda").manual_seed(1)
    a_shape = (k, m) if layout == 2 else (m, k)
    b_shape = (n, k) if layout == 0 else (k, n)
    a = (torch.randn(a_shape, device="cuda", generator=g) * 0.5).to(BF)
    b = (torch.randn(b_shape, device="cuda", generator=g) * 0.5).to(BF)
    c = torch.empty(m, n, device="cuda", dtype=BF)
    bg.gemm_bf16(a, b, c, m, n, k, layout)
    want = torch.matmul(a.t() if layout == 2 else a, b.t() if layout == 0 else b)
    diff = (c.float() - want.float()).abs()
    scale = want.float().abs().mean()
    assert float(diff.max()) <= float(scale) * 0.05 + 0.5, (float(diff.max()), float(scale))
    assert float(diff.mean()) <= float(scale) * 2 ** -8

"""The plain GEMM runs 256-wide tiles (wgmma m64n256k16) for N > 128 and 128-wide tiles (m64n128k16) for N <= 128.  Both
walk every output element's k loop in the same order, so a 128-column slice of a product, computed on its own by the
narrow tile, must equal the same columns of the full product computed by the wide tile bit for bit.  The shapes cover a
flagship projection and MLP down-projection, a ragged output (4360 = 17 wide tiles + 8 columns, M and K off the tile
grid) and the smallest outputs that take the wide tile (136: one wide tile, 120 columns of it out of bounds; 264: a
second wide tile with 8 live columns)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _fp_check import assert_rounded, gemm_eps  # noqa: E402
pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
BF = torch.bfloat16


@pytest.fixture(scope="module")
def bg():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import hetu_galvatron_b200._bg as bg
    bg.lib()
    return bg


@pytest.mark.parametrize("epilogue", [None, "acc", "addend"])
@pytest.mark.parametrize("layout", [0, 1, 2])
@pytest.mark.parametrize("m,n,k", [(8192, 3072, 2048), (8192, 2048, 8192), (2056, 4360, 520), (1032, 136, 264), (1032, 264, 1032)])
def test_wide_tile_matches_narrow_slices(bg, layout, m, n, k, epilogue):
    g = torch.Generator(device="cuda").manual_seed(m + n + k + layout)
    a = (torch.randn((k, m) if layout == 2 else (m, k), device="cuda", generator=g) * 0.5).to(BF)
    b = (torch.randn((n, k) if layout == 0 else (k, n), device="cuda", generator=g) * 0.5).to(BF)
    c0 = torch.randn(m, n, device="cuda", generator=g).to(BF)

    def gemm(bb, cc0, nn):
        c = cc0.clone()
        if epilogue == "addend":
            bg.gemm_bf16_add(a, bb, c, cc0, m, nn, k, layout)
        else:
            bg.gemm_bf16(a, bb, c, m, nn, k, layout, accumulate=epilogue == "acc")
        return c

    full = gemm(b, c0, n)
    for c_lo in range(0, n, 128):
        c_hi = min(n, c_lo + 128)
        bs = (b[c_lo:c_hi] if layout == 0 else b[:, c_lo:c_hi]).contiguous()
        part = gemm(bs, c0[:, c_lo:c_hi].contiguous(), c_hi - c_lo)
        torch.cuda.synchronize()
        assert torch.equal(part, full[:, c_lo:c_hi]), (c_lo, c_hi)
    ad, bd = (a.double().t() if layout == 2 else a.double()), (b.double().t() if layout == 0 else b.double())
    ref, s = ad @ bd, ad.abs() @ bd.abs()
    if epilogue:
        ref, s = ref + c0.double(), s + c0.double().abs()
    assert_rounded(full, ref, gemm_eps(k, s))       # the fp32 accumulation bound, then one correct bf16 rounding

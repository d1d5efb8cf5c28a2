"""The plain GEMM walks its tiles in a raster chosen from the output width (2 m-blocks per sweep over n up to 32 n-blocks,
8 above).  The raster only orders tiles: each tile's k loop is the same, so a column slice of a product computed on
its own (under another raster) must equal the same slice of the full product bit for bit.  The 8192 x 8192 output is
rastered with 8 m-blocks per sweep, its 2048-wide column slices with 2; so is the ragged 4360-wide one (35 n-blocks) against
its 1024-wide slices."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _fp_check import assert_rounded, gemm_eps  # noqa: E402
pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
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
@pytest.mark.parametrize("m,n,k,cols", [(8192, 8192, 2048, 2048), (2056, 4360, 520, 1024)])
def test_column_slices_match_full_product(bg, layout, m, n, k, cols, epilogue):
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
    for c_lo in range(0, n, cols):
        c_hi = min(n, c_lo + cols)
        bs = (b[c_lo:c_hi] if layout == 0 else b[:, c_lo:c_hi]).contiguous()
        part = gemm(bs, c0[:, c_lo:c_hi].contiguous(), c_hi - c_lo)
        torch.cuda.synchronize()
        assert torch.equal(part, full[:, c_lo:c_hi]), (c_lo, c_hi)
    ad, bd = (a.double().t() if layout == 2 else a.double()), (b.double().t() if layout == 0 else b.double())
    ref, s = ad @ bd, ad.abs() @ bd.abs()
    if epilogue:
        ref, s = ref + c0.double(), s + c0.double().abs()
    assert_rounded(full, ref, gemm_eps(k, s))       # the fp32 accumulation bound, then one correct bf16 rounding

"""GPU checks of the wgmma/TMA GEMM (through the C ABI) against float64 references of the same bf16 inputs.  Covers the three
layouts of the Megatron linear layer (layers.py:417 fwd TN, :462 dgrad NN, :534 wgrad NT), both tile widths (the kernel runs
128-wide tiles for N <= 128 and 256-wide tiles above), and the four epilogues: plain, accumulate into C, add a separate addend,
and add an addend that aliases C.

Two references:
  - integer data: A and B integers in [-8, 8], addends integer-valued bf16 in [-4096, 4096].  Every product and every partial
    sum is an integer below 2^24, which fp32 holds exactly in any summation order, so the output must be the float64 result
    rounded to bf16 (round to nearest, ties to even) BIT FOR BIT.  Products with K >= 1000 must contain ties of both kinds, so a
    kernel that rounds ties away from zero fails as surely as one that truncates.
  - real data: N(0, 0.25) in bf16; the output must be within half a bf16 ulp of the float64 value plus the fp32 accumulation
    bound `gemm_eps` (tests/_fp_check.py).
Every output sits in the middle of a larger allocation between two guards of 128 sentinel rows, which must be bit-identical
after the call (TMA must clip every store to [M][N]); the non-accumulating epilogues start from NaN, so an element the kernel
never writes fails."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from _fp_check import BF, F64, assert_rounded, gemm_eps  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
EPILOGUES = ("plain", "acc", "add", "add_alias")
GUARD = 128                  # sentinel rows before and after C: one tile row
SENTINEL = 0x3F5A            # bf16 bits of 0.8515625


@pytest.fixture(scope="module")
def bg():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import hetu_galvatron_b200._bg as bg
    bg.lib()
    return bg


def _rand(shape, kind, g, lim=8):
    if kind == "int":
        return torch.randint(-lim, lim + 1, shape, device="cuda", generator=g).to(BF)
    return (torch.randn(shape, device="cuda", generator=g) * 0.5).to(BF)


def _operands(layout, m, n, k, kind, g):
    """the stored operands a, b of `layout` and their logical views A [M][K], B [K][N]"""
    a = _rand((k, m) if layout == 2 else (m, k), kind, g)
    b = _rand((n, k) if layout == 0 else (k, n), kind, g)
    return a, b, (a.t() if layout == 2 else a), (b.t() if layout == 0 else b)


def _addend(m, n, kind, g):
    return _rand((m, n), kind, g, lim=4096)


def _run(bg, layout, a, b, m, n, k, epilogue, c0=None):
    """C of one call, written into the middle of a guarded allocation; checks that the guards are untouched"""
    buf = torch.full(((m + 2 * GUARD) * n,), SENTINEL, device="cuda", dtype=torch.int16)
    c = buf[GUARD * n:(GUARD + m) * n].view(BF).view(m, n)
    if epilogue in ("acc", "add_alias"):
        c.copy_(c0)
    else:
        c.fill_(float("nan"))
    if epilogue in ("plain", "acc"):
        bg.gemm_bf16(a, b, c, m, n, k, layout, accumulate=epilogue == "acc")
    else:
        bg.gemm_bf16_add(a, b, c, c if epilogue == "add_alias" else c0, m, n, k, layout)
    torch.cuda.synchronize()
    for what, guard in (("before", buf[:GUARD * n]), ("after", buf[(GUARD + m) * n:])):
        bad = int((guard != SENTINEL).sum())
        assert bad == 0, "%d elements of the guard %s C were written" % (bad, what)
    return c


def _tie_kinds(ref):
    """(ties that round down to even, ties that round up to even) among the exact integer results `ref` (|ref| < 2^24, so
    fp32 holds them; bf16 keeps the upper 16 bits of the fp32 pattern)"""
    bits = ref.float().view(torch.int32)
    tie = (bits & 0xFFFF) == 0x8000
    odd = ((bits >> 16) & 1) == 1
    return int((tie & ~odd).sum()), int((tie & odd).sum())


def _assert_exact(got, ref, what):
    want = ref.to(BF)
    bad = got.view(torch.int16) != want.view(torch.int16)
    if bad.any():
        i = int(bad.reshape(-1).nonzero()[0])
        pytest.fail("%s: %d / %d elements differ from the correctly rounded result; first at flat index %d: got %r want %r "
                    "(exact %r)" % (what, int(bad.sum()), bad.numel(), i, got.reshape(-1)[i].item(), want.reshape(-1)[i].item(),
                                    ref.reshape(-1)[i].item()))


def _check_all_epilogues(bg, layout, m, n, k, kind, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a, b, A, B = _operands(layout, m, n, k, kind, g)
    c0 = _addend(m, n, kind, g)
    Ad, Bd = A.to(F64), B.to(F64)
    prod = Ad @ Bd
    s = Ad.abs() @ Bd.abs() if kind == "real" else None
    for epi in EPILOGUES:
        got = _run(bg, layout, a, b, m, n, k, epi, c0)
        ref = prod if epi == "plain" else prod + c0.to(F64)
        what = "%s layout %d %dx%dx%d %s" % (kind, layout, m, n, k, epi)
        if kind == "int":
            assert ref.abs().max() < 2 ** 24
            _assert_exact(got, ref, what)
            if k >= 1000:
                down, up = _tie_kinds(ref)
                assert down > 0 and up > 0, (what, down, up)
        else:
            # |fp32 result - ref| <= gemm_eps(k, |A| @ |B| (+ |addend|)); the bf16 rounding adds half an ulp
            assert_rounded(got, ref, gemm_eps(k, s if epi == "plain" else s + c0.to(F64).abs()), what)


# Edges: M 8 (a tail inside consumer warpgroup 0), 64 (exactly one warpgroup), 72 (one row group into warpgroup 1), 128 (a full
# tile), 136 (8 rows into the next tile), 200, 1032 (9 m-blocks: a ragged raster group); N 8, 64, 120 (tails inside a 64-column
# store chunk), 128 (the widest 128-wide tile), 136 (one 256-wide tile with 8 live columns in its 3rd chunk), 192 (a wide tile
# whose 4th store chunk is skipped), 264, 4360 (18 wide n-blocks: group_m = 16, 8 live columns in the last); K 8, 64, 72,
# 1000, 4160 (tails inside and across the 64-deep k-block).  2056 x 4360 is 306 tiles: more than SMs, so CTAs loop over
# different numbers of tiles and reuse their staging buffers.
EDGE_SHAPES = [(8, 8, 8), (64, 64, 64), (72, 120, 72), (128, 128, 1000), (136, 136, 4160), (200, 192, 1000), (1032, 264, 72),
               (8, 4360, 64), (1032, 4360, 1000), (2056, 4360, 4160)]


@pytest.mark.parametrize("layout", [0, 1, 2])
@pytest.mark.parametrize("m,n,k", EDGE_SHAPES)
def test_gemm_edges_integer_exact(bg, layout, m, n, k):
    _check_all_epilogues(bg, layout, m, n, k, "int", seed=m * 7 + n * 3 + k + layout)


@pytest.mark.parametrize("layout", [0, 1, 2])
@pytest.mark.parametrize("m,n,k", EDGE_SHAPES)
def test_gemm_edges_real(bg, layout, m, n, k):
    _check_all_epilogues(bg, layout, m, n, k, "real", seed=m * 5 + n * 11 + k + layout)


@pytest.mark.parametrize("layout", [0, 1, 2])
def test_gemm_deterministic(bg, layout):
    m, n, k = 2056, 4360, 4160
    g = torch.Generator(device="cuda").manual_seed(layout)
    a, b, _, _ = _operands(layout, m, n, k, "real", g)
    c0 = _addend(m, n, "real", g)
    for epi in EPILOGUES:
        first, second = (_run(bg, layout, a, b, m, n, k, epi, c0) for _ in range(2))
        assert torch.equal(first.view(torch.int16), second.view(torch.int16)), epi


def _samples(extent, block, per_block, g):
    """per_block random indices from every `block`-sized block of range(extent)"""
    idx = []
    for lo in range(0, extent, block):
        width = min(block, extent - lo)
        idx += (lo + torch.randperm(width, generator=g)[:per_block]).tolist()
    return torch.tensor(idx, device="cuda")


@pytest.mark.parametrize("layout,m,n,k", [
    (0, 8192, 6144, 4096),    # QKV projection fwd
    (0, 8192, 28672, 4096),   # gate+up fwd
    (0, 8192, 4096, 14336),   # down fwd
    (1, 8192, 4096, 6144),    # QKV dgrad
    (2, 28672, 4096, 8192),   # gate+up wgrad
    (2, 4096, 14336, 8192),   # down wgrad
])
def test_gemm_llama3_8b_shapes(bg, layout, m, n, k):
    """The BASELINE sizes.  A full float64 product costs up to 2 TFLOP here, so the check samples: 2 random rows of every
    128-row block against all columns, and 2 random columns of every 256-column block against all rows -- every tile is checked
    in both directions."""
    gs = torch.Generator().manual_seed(m + n + k)
    rows, cols = _samples(m, 128, 2, gs), _samples(n, 256, 2, gs)
    for kind in ("int", "real"):
        g = torch.Generator(device="cuda").manual_seed(m + n + k + layout)
        a, b, A, B = _operands(layout, m, n, k, kind, g)
        got = _run(bg, layout, a, b, m, n, k, "plain")
        Bd = B.to(F64)
        for what, sel, ra, rb in (("rows", (rows, slice(None)), A[rows].to(F64), Bd),
                                  ("cols", (slice(None), cols), A.to(F64), Bd[:, cols])):
            ref = ra @ rb
            label = "%s layout %d %dx%dx%d sampled %s" % (kind, layout, m, n, k, what)
            if kind == "int":
                _assert_exact(got[sel], ref, label)
            else:
                assert_rounded(got[sel], ref, gemm_eps(k, ra.abs() @ rb.abs()), label)
            del ref, ra, rb


def test_gemm_index_width(bg):
    """M * N = 17408 * 131072 > 2^31 elements: a 32-bit element index would wrap from row 16384 on.  Every such row is checked,
    plus 2 sampled rows of every 128-row block before it, for the plain and the accumulating epilogue."""
    m, n, k = 17408, 131072, 64
    first_wide = (1 << 31) // n
    g = torch.Generator(device="cuda").manual_seed(17)
    a, b, A, B = _operands(0, m, n, k, "int", g)
    rows = torch.cat([_samples(first_wide, 128, 2, torch.Generator().manual_seed(3)),
                      torch.arange(first_wide, m, device="cuda")])
    prod = A[rows].to(F64) @ B.to(F64)
    c = torch.full((m, n), float("nan"), device="cuda", dtype=BF)
    try:
        bg.gemm_bf16(a, b, c, m, n, k, 0)
        torch.cuda.synchronize()
        _assert_exact(c[rows], prod, "plain")
        before = c[rows].to(F64)
        bg.gemm_bf16(a, b, c, m, n, k, 0, accumulate=True)
        torch.cuda.synchronize()
        _assert_exact(c[rows], prod + before, "accumulate")
    finally:
        del c
        torch.cuda.empty_cache()

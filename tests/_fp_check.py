"""Floating-point checks shared by the GPU kernel tests: a bf16 output must be the correctly rounded float64 value up to the
kernel's own fp32 evaluation error, and an fp32 output must be within a derived bound of the float64 value.

    |got - ref| <= 1/2 ulp_bf16 + eps        (assert_rounded)
    |got - ref| <= eps + 1/2 ulp_fp32       (assert_within)

eps is derived by each caller, next to its assertion, from the formula the kernel evaluates; U = 2^-24 is the unit roundoff of
fp32.  NaN anywhere fails, so an output buffer that starts as NaN also catches elements a kernel never writes."""
import torch

BF = torch.bfloat16
F64 = torch.float64
U = 2.0 ** -24              # unit roundoff of fp32


def gamma(k):
    """Higham's gamma_k = k u / (1 - k u): the relative error bound of k fp32 roundings in a row."""
    return k * U / (1 - k * U)


def _ulp(v, mant):
    """spacing of the floating-point numbers with `mant` explicit mantissa bits at |v|: 2^(floor(log2|v|) - mant)
    (normal range; the smallest normal's spacing below it)"""
    _, e = torch.frexp(v.double().abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(v, dtype=F64), e - 1 - mant)


def ulp_bf16(v):
    return _ulp(v, 7)


def ulp_f32(v):
    return _ulp(v, 23)


def _report(what, got, ref, err, tol, bad):
    i = int(torch.argmax(torch.where(bad, (err / tol).nan_to_num(float("inf")), torch.zeros_like(err))))
    flat = lambda t: t.reshape(-1)[i].item()  # noqa: E731
    return (f"{what}: {int(bad.sum())} / {bad.numel()} outside the bound; worst at flat index {i}: got {flat(got)} ref {flat(ref)} "
            f"err {flat(err):.3e} tol {flat(tol):.3e}")


def assert_rounded(got, ref, eps, what="bf16 output"):
    """bf16 `got` against the float64 `ref`: |got - ref| <= 1/2 ulp_bf16 + eps, the ulp the larger of got's and ref's (a result
    rounded up across a power of two is still correctly rounded).  NaN anywhere fails."""
    assert got.dtype == BF and ref.dtype == F64
    g = got.double()
    tol = 0.5 * torch.maximum(ulp_bf16(g), ulp_bf16(ref)) + eps
    err = (g - ref).abs()
    bad = ~(err <= tol)
    assert not bad.any(), _report(what, g, ref, err, tol, bad)


def assert_within(got, ref, eps, what="fp32 output"):
    """fp32 `got` against the float64 `ref`: |got - ref| <= eps + 1/2 ulp_fp32 (the final rounding of the fp32 result)."""
    g = got.double()
    tol = eps + 0.5 * ulp_f32(ref)
    err = (g - ref).abs()
    bad = ~(err <= tol)
    assert not bad.any(), _report(what, g, ref, err, tol, bad)


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF else t.view(torch.int32)


def gemm_eps(k, s):
    """fp32 error bound of one output of the wgmma GEMM (csrc/bg_gemm.cu) before its final bf16 rounding, for a K-long dot
    product whose |terms| sum to `s` (|A| @ |B|, plus |addend| when the epilogue adds one):
      - the bf16 products are exact in fp32;
      - each k16 wgmma adds its 16 products into the accumulator: up to four levels of rounding inside the group, one step
        per group, ceil(K / 16) groups;
      - the epilogue's add of the addend or the old C is one more rounding;
      - the tensor core's internal rounding is not documented, so each step is charged 2u instead of u.
    Hence (ceil(K / 16) + 4 + 1) * 2u * s."""
    return (-(-k // 16) + 5) * 2 * U * s

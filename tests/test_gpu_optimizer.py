"""The fused optimizer kernels of csrc/bg_coll.cu against float64 AdamW and float64 sums of squares, on virtual ranks.

Entries under test: the AdamW reduce-scatter (``bg_reduce_scatter_adamw``), its clipped form (``bg_reduce_scatter_adamw_clipped``),
the norm pass (``bg_reduce_scatter_sumsq``) and the local clipped step of pooled ZeRO-3 units (``bg_adamw_clipped``), for bf16
and fp32 gradient sources, on groups of 1, 2, 3, 4, 6 and 8 virtual ranks of one device (``BgComm.local_world``, comm_ctas 16),
with the FSDP pre/post-divide factors of ``oracle/collectives_ref.fsdp_divide_factors``.

The reference.  AdamW in float64 from the fp32 values the kernel reads:
  - the gradient is the kernel's own fp32 gradient, obtained bit for bit from the same sources with ``bg_reduce_scatter_acc``
    (fp32 dst, accumulate 0) at the same prescale and postscale.  For the clipped reduce-scatter the postscale is the fp32
    product fp32(postscale) * fp32(coef): the clipped kernel folds exactly that into its postscale at its start.  For the local
    step the gradient is fp32(g * coef), the one rounding the local kernel makes.  So the AdamW check does not inherit the
    collective's summation error, which tests/test_gpu_collectives.py bounds.
  - the hyperparameters are the fp32 values the ABI receives, not Python's doubles (at beta2 = 0.999, 1 - 0.999f is 1.3e-5
    relative away from 1 - 0.999: that difference is what the kernel computes, not an error).  1 - beta is exact in fp32 for
    every beta used here (0, or >= 1/2: Sterbenz), and the bias corrections are 1 - beta^t computed in double from the fp32
    betas, as the host code does before it rounds them to fp32.
  - each step's reference starts from the kernel's own fp32 (p, m, v) of the previous step, so errors do not compound.

The bounds (u = 2^-24, gamma_k = k u / (1 - k u), tiny = 2^-149 the fp32 subnormal spacing that bounds the absolute error of
one rounding below the normal range; the build is -O3 without fast-math, so sqrtf and / are correctly rounded, subnormals are
kept, and multiply-adds may be contracted).  c1 = 1 - b1, c2 = 1 - b2, s = lr / bc1, d = sqrt(v') / bc2s + eps:
  m' = b1 m + c1 g:                 |dm| <= gamma_3 (b1 |m| + c1 |g|) + 3 tiny         (absolute: the terms can cancel)
  v' = b2 v + c2 g^2:               |dv| <= gamma_4 (b2 v + c2 g^2) + 4 tiny           (both terms >= 0: relative)
  d:                                relative gamma_7 (v' to gamma_4 under the sqrt, the sqrt, bc2s rounded to fp32, the division,
                                    the add of eps), plus sqrt(4 tiny) / bc2s from an underflowed v'
  upd = s m' / d:                   |dupd| <= s |dm| / d + |upd| gamma_11 + s |m'| sqrt(4 tiny) / (bc2s d^2) + 3 tiny
                                    (s is rounded twice: bc1 to fp32 and the division; then the product, the quotient, d)
  p' = p (1 - lr wd) - upd:         |dp| <= |p| delta_decay + gamma_2 (|p decay| + |upd|) + |dupd| + 2 tiny,
                                    delta_decay = u lr wd + u decay (the fp32 decay 1 - lr wd: two roundings)
``_fp_check.assert_within`` adds half an fp32 ulp of the reference for the final rounding.

Bit-for-bit relations:
  - the clipped reduce-scatter with a null coefficient, and with coefficient 1, equals bg_reduce_scatter_adamw;
  - the pooled-unit path, bg_reduce_scatter_sumsq(dst=shard) then bg_adamw_clipped on that shard, equals the clipped
    reduce-scatter on the same sources at coefficient 1 (every group), and at any coefficient where the postscale is a power of
    two (groups of 1, 2, 4 and 8: (acc * ps) * coef and acc * (ps * coef) round alike).  With postscale 1 / 1.5 (groups of 3
    and 6) both paths are held to the float64 bound instead;
  - the norm pass's dst equals bg_reduce_scatter_acc's output;
  - the same step at comm_ctas 1, 3 and 16 gives the same (p, m, v) and the same fp32 shard.

Cases.  Hyperparameter sets: the defaults of this repository, the set of the older tests, lr = 0 (p comes back bit-identical
while m and v update), wd = 0, beta1 = beta2 = 0 and eps = 1e-3.  Steps 1, 2, 3 from zero moments, then 10, 1000, 10^6 and
2^31 + 5 from random state (signed m, v >= 0 with some v = 0).  Gradients N(0, sigma), sigma from 1e-6 to 1 over the steps,
with exact zeros, magnitudes log-uniform over [1e-30, 1e3], some of 1e18 (squares near the fp32 top) and, from random state,
a block where b1 m and c1 g cancel.  Shards: one 16-B vector, 4096 * 8 + 8, one vector before, at and after a whole grid-stride
span of the launch, and 2^24 + 24 elements for groups of at most 2.  Clip coefficients null, 1, 0.3 and 0.7 (whose fp32 product
with the postscale 1 / 1.5 is inexact).  Every state tensor is a view between sentinel guards, which must come back unchanged,
as must the sources.  Every case checks the device error flag.
"""
import contextlib
import math
import os
import sys

import pytest
import torch

# before any CUDA context exists in this process: a kernel waiting for a peer must never falsely order another stream behind it
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from _fp_check import BF, U, _bits, assert_within, gamma  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

F32, F64 = torch.float32, torch.float64
TINY = 2.0 ** -149           # spacing of the fp32 subnormals
GUARD = 1024                 # fp32 elements of every guard region
CTAS = 16
# Launch geometry of bg_coll.cu: kThreads = 128; the AdamW and sum-of-squares epilogues keep V = RsPlan<PMAX, kEpi>::V vectors
# in flight per thread and iteration (half of kInFlight = 8 below 8 peers, divided by PMAX = 2, 4 or 8, the smallest >= n);
# grid = min(ceil((vectors / V + 1) / 128), comm_ctas), local_ctas for a group of one.  The local step: one vector of 4.
THREADS, K_IN_FLIGHT = 128, 8
LARGE = (1 << 24) + 24

HYPER = {            # lr, beta1, beta2, eps, weight_decay
    "defaults": (1e-4, 0.9, 0.999, 1e-8, 0.01),
    "older_tests": (1e-2, 0.9, 0.95, 1e-8, 0.1),
    "lr0": (0.0, 0.9, 0.999, 1e-8, 0.01),
    "wd0": (1e-3, 0.9, 0.999, 1e-8, 0.0),
    "beta0": (1e-3, 0.0, 0.0, 1e-8, 0.01),
    "eps1e-3": (1e-3, 0.9, 0.999, 1e-3, 0.01),
}
ZERO_STEPS = (1, 2, 3)
STATE_STEPS = (10, 1000, 10 ** 6, (1 << 31) + 5)
COEFS = (None, 1.0, 0.3, 0.7)


def f32(x):
    return float(torch.tensor(x, dtype=F32))


def _pmax(n):
    return 2 if n <= 2 else 4 if n <= 4 else 8


def v_opt(n):
    return (K_IN_FLIGHT // 2 if _pmax(n) < 8 else K_IN_FLIGHT) // _pmax(n)


def comm_grid(vectors, v, cap=CTAS):
    return max(1, min(cap, -(-(vectors // v + 1) // THREADS)))


def shards(n, dt):
    """shard sizes (elements) at the edges of the launch: one vector, 4096 * 8 + 8, one vector before, at and after a whole
    grid-stride span of the capped grid (CTAS * 128 * V vectors), and 2^24 + 24 for groups of at most 2"""
    e = 8 if dt == BF else 4
    span = CTAS * THREADS * v_opt(n)
    assert comm_grid(span - 1, v_opt(n)) == CTAS
    out = {"vector": e, "mid": 4096 * 8 + 8, "span-1": (span - 1) * e, "span": span * e, "span+1": (span + 1) * e}
    if n <= 2:
        out["large"] = LARGE
    return out


SHARD_NAMES = ("vector", "mid", "span-1", "span", "span+1", "large")


@contextlib.contextmanager
def tunables(bg, **kv):
    old = {k: bg.get_tunable(k) for k in kv}
    try:
        for k, v in kv.items():
            bg.set_tunable(k, v)
        yield
    finally:
        for k, v in old.items():
            bg.set_tunable(k, v)


@pytest.fixture(scope="module")
def bg():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import hetu_galvatron_b200._bg as bg
    bg.lib()
    with tunables(bg, timeout_ms=20000, comm_ctas=CTAS, local_ctas=CTAS):
        yield bg


class World:
    """n virtual ranks with one symmetric source buffer each, sized once for the largest shard of the module and reused."""

    def __init__(self, bg, n):
        from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
        self.bg, self.n = bg, n
        self.src_bytes = n * max(max(shards(n, dt).values()) for dt in (BF, F32)) * 4
        self.comms = bg.BgComm.local_world(n, device=0, arena_bytes=self.src_bytes + (64 << 20))
        self.group = CommGroup(list(range(n)))
        self.streams = [torch.cuda.Stream() for _ in range(n)]
        self.sym = [c.sym_alloc(self.group, self.src_bytes) for c in self.comms]
        for c in self.comms:
            c.exchange()
        self.gen = torch.Generator(device="cuda").manual_seed(500 + n)
        self.pre, self.post = fsdp_factors(n)

    def run(self, fn):
        torch.cuda.synchronize()
        for r, c in enumerate(self.comms):
            with torch.cuda.stream(self.streams[r]):
                fn(r, c)
        torch.cuda.synchronize()
        for c in self.comms:
            assert c.error_flag() == 0

    def close(self):
        torch.cuda.synchronize()
        for c in self.comms:
            c.close()


def fsdp_factors(n):
    from oracle import collectives_ref
    return collectives_ref.fsdp_divide_factors(n)


@pytest.fixture(scope="module", params=[1, 2, 3, 4, 6, 8])
def world(request, bg):
    w = World(bg, request.param)
    yield w
    w.close()


# ---- data --------------------------------------------------------------------------------------------------------------------
def write_sources(w, shard, dt, sigma, huge=1e18):
    """Every member's source: N(0, sigma), with edge elements at fixed shard-relative positions i (so a one-vector shard has them
    too): i % 16 == 3 exact zeros; i % 16 in (5, 9) magnitudes log-uniform over [1e-30, 1e3]; i % 64 == 13 +-huge.  An edge value
    is held by member 0 alone, so the sum over the members is exact.  Returns a snapshot of the sources' bytes."""
    n, total = w.n, w.n * shard
    i = torch.arange(total, device="cuda") % shard
    vals = torch.randn(n, total, device="cuda", generator=w.gen) * sigma
    sign = torch.where(torch.rand(total, device="cuda", generator=w.gen) < 0.5, -1.0, 1.0)
    logu = sign * 10.0 ** (torch.rand(total, device="cuda", generator=w.gen) * 33 - 30)
    edge = ((i % 16 == 3) | (i % 16 == 5) | (i % 16 == 9) | (i % 64 == 13))
    first = torch.where(i % 16 == 3, 0.0, torch.where(i % 64 == 13, sign * huge, logu))
    vals[:, edge] = 0.0
    vals[0, edge] = first[edge]
    esz = 2 if dt == BF else 4
    for r in range(n):
        w.sym[r].view(dt, total).copy_(vals[r].to(dt))
    return [w.sym[r].u8[:total * esz].clone() for r in range(n)]


def check_sources(w, snap):
    for r in range(w.n):
        assert torch.equal(w.sym[r].u8[:snap[r].numel()], snap[r]), "source of rank %d changed" % r


class Guarded:
    """an fp32 tensor of `numel` elements between two sentinel guards of GUARD elements"""

    def __init__(self, numel, gen):
        self.numel = numel
        self.buf = torch.randint(-2 ** 31, 2 ** 31 - 1, (numel + 2 * GUARD,), dtype=torch.int32, device="cuda",
                                 generator=gen).view(F32)
        self.guards = self._guards().clone()
        self.t = self.buf[GUARD:GUARD + numel]

    def _guards(self):
        return torch.cat([self.buf[:GUARD], self.buf[GUARD + self.numel:]]).view(torch.int32)

    def check(self):
        assert torch.equal(self._guards(), self.guards), "guard overwritten"


def state_buffers(w, state):
    out = []
    for t in state:
        g = Guarded(t.numel(), w.gen)
        g.t.copy_(t)
        out.append(g)
    return out


def random_state(w, shard, sigma):
    """p ~ N(0, 1); m signed, ~ sigma; v >= 0, ~ sigma^2, exactly 0 where i % 16 == 11"""
    i = torch.arange(shard, device="cuda")
    p = torch.randn(shard, device="cuda", generator=w.gen)
    m = torch.randn(shard, device="cuda", generator=w.gen) * sigma
    v = (torch.randn(shard, device="cuda", generator=w.gen) * sigma) ** 2
    v[i % 16 == 11] = 0.0
    return [p, m, v]


# ---- the float64 reference and its bounds ------------------------------------------------------------------------------------
def fp32_hyper(h):
    """the fp32 values the ABI receives; 1 - beta is then exact in fp32 (beta = 0 or >= 1/2)"""
    lr, b1, b2, eps, wd = (f32(x) for x in h)
    for b in (b1, b2):
        assert f32(1.0 - b) == 1.0 - b
    return lr, b1, b2, eps, wd


def adamw_ref(p, m, v, g, h, step):
    """float64 AdamW from fp32 inputs and fp32 hyperparameters; returns (p', m', v') and their error bounds (module docstring)"""
    lr, b1, b2, eps, wd = fp32_hyper(h)
    p, m, v, g = (t.double() for t in (p, m, v, g))
    c1, c2 = 1.0 - b1, 1.0 - b2
    bc1, bc2s = 1.0 - b1 ** step, math.sqrt(1.0 - b2 ** step)
    m1 = b1 * m + c1 * g
    v1 = b2 * v + c2 * g * g
    d = v1.sqrt() / bc2s + eps
    s = lr / bc1
    upd = s * m1 / d
    decay = 1.0 - lr * wd
    p1 = p * decay - upd
    em = gamma(3) * (b1 * m.abs() + c1 * g.abs()) + 3 * TINY
    ev = gamma(4) * (b2 * v + c2 * g * g) + 4 * TINY
    eu = s * em / d + upd.abs() * gamma(11) + s * m1.abs() * math.sqrt(4 * TINY) / (bc2s * d * d) + 3 * TINY
    delta_decay = U * lr * wd + U * decay
    ep = p.abs() * delta_decay + gamma(2) * ((p * decay).abs() + upd.abs()) + eu + 2 * TINY
    return (p1, m1, v1), (ep, em, ev)


def check_step(what, got, state_in, g, h, step):
    """the kernel's (p, m, v) against float64 AdamW from state_in and the fp32 gradient g.  Elements whose reference moved by more
    than the bound prove they were written; there must be such elements in m wherever g is not zero."""
    refs, bounds = adamw_ref(*state_in, g, h, step)
    for name, out, ref, eps in zip("pmv", got, refs, bounds):
        assert_within(out, ref, eps, "%s %s at step %d" % (what, name, step))
    moved = (refs[1] - state_in[1].double()).abs() > bounds[1] + 0.5 * state_in[1].double().abs() * 2 * U
    assert int(moved.sum()) >= (g != 0).sum() // 2, (what, int(moved.sum()))


def acc_grad(w, shard, dt, postscales):
    """the fp32 gradient each rank's AdamW epilogue forms: bg_reduce_scatter_acc's fp32 output, accumulate 0"""
    out = [torch.full((shard,), float("nan"), device="cuda") for _ in range(w.n)]
    w.run(lambda r, c: c.reduce_scatter_acc(w.group, w.sym[r], dt, out[r], prescale=1.0 / w.pre, postscale=postscales[r]))
    return out


def pow2(x):
    return x > 0 and math.frexp(x)[0] == 0.5


def bits_equal(a, b):
    return torch.equal(_bits(a), _bits(b))


# ---- AdamW: the reduce-scatter, its clipped form, and the pooled-unit path ------------------------------------------------------
def run_paths(w, dt, shard, state, h, step, coef):
    """one step of the three paths from the same state: the AdamW reduce-scatter ("plain"), the clipped reduce-scatter ("clip")
    and the pooled-unit path ("pool": the norm pass writing the fp32 shard, then the local clipped step).  Returns the guarded
    outputs and the pooled path's fp32 shards."""
    n, bg = w.n, w.bg
    pre, post = 1.0 / w.pre, 1.0 / w.post
    coef_t = None if coef is None else torch.full((), coef, device="cuda")
    out = {k: [state_buffers(w, state[r]) for r in range(n)] for k in ("plain", "clip", "pool")}
    lr, b1, b2, eps, wd = h
    st = lambda k, r: [b.t for b in out[k][r]]  # noqa: E731
    w.run(lambda r, c: c.reduce_scatter_adamw(w.group, w.sym[r], dt, *st("plain", r), shard, pre, post, lr, b1, b2, eps, wd, step))
    w.run(lambda r, c: c.reduce_scatter_adamw_clipped(w.group, w.sym[r], dt, *st("clip", r), shard, pre, post, lr, b1, b2, eps, wd,
                                                      step, coef_t))
    flat = [Guarded(shard, w.gen) for _ in range(n)]
    parts = [torch.full((4 * CTAS + 36,), float("nan"), device="cuda") for _ in range(n)]
    w.run(lambda r, c: c.reduce_scatter_sumsq(w.group, w.sym[r], dt, shard, pre, post, parts[r], dst=flat[r].t))
    for r in range(n):
        bg.adamw_clipped(*st("pool", r), flat[r].t, lr, b1, b2, eps, wd, step, coef_t)
    torch.cuda.synchronize()
    for g in flat:
        g.check()
    for k in out:
        for r in range(n):
            for b in out[k][r]:
                b.check()
    return {k: [st(k, r) for r in range(n)] for k in out}, [g.t for g in flat]


@pytest.mark.parametrize("hyper", sorted(HYPER))
@pytest.mark.parametrize("dt", [BF, F32], ids=["bf16", "fp32"])
def test_adamw_against_float64(world, bg, dt, hyper):
    """steps 1-3 from zero moments and 10 .. 2^31 + 5 from random state, at one shard edge per (dtype, hyperparameter set), every
    clip coefficient in turn: every path within the float64 bound of the module docstring, and the bit-for-bit relations."""
    w, n = world, world.n
    h = HYPER[hyper]
    hi = sorted(HYPER).index(hyper)
    table = shards(n, dt)
    names = [k for k in SHARD_NAMES if k in table]
    shard = table[names[(hi + (dt == F32)) % len(names)]]
    post = f32(1.0 / w.post)
    if not pow2(post):          # the coefficient 0.7 then makes the clipped kernel's postscale product inexact
        assert f32(post * f32(0.7)) != post * f32(0.7)
    g0 = torch.Generator(device="cuda").manual_seed(hi)
    p0 = torch.randn(shard, device="cuda", generator=g0)
    state = [[p0.clone(), torch.zeros(shard, device="cuda"), torch.zeros(shard, device="cuda")] for _ in range(n)]
    lr, b1 = f32(h[0]), f32(h[1])
    for si, step in enumerate(ZERO_STEPS + STATE_STEPS):
        sigma = 10.0 ** (-6 + si)
        coef = COEFS[(si + hi) % len(COEFS)]
        snap = write_sources(w, shard, dt, sigma)
        g_plain = acc_grad(w, shard, dt, [post] * n)
        post_c = post if coef is None else f32(post * f32(coef))       # postscale *= *clip_coef, in fp32
        g_clip = acc_grad(w, shard, dt, [post_c] * n)
        if step in STATE_STEPS:
            state = [random_state(w, shard, sigma) for _ in range(n)]
            if b1 > 0:          # b1 m + c1 g cancels (to the rounding of m) where i % 16 == 7
                i = torch.arange(shard, device="cuda")
                for r in range(n):
                    sel = i % 16 == 7
                    state[r][1][sel] = (-(1.0 - b1) * g_plain[r][sel].double() / b1).float()
        outs, flat = run_paths(w, dt, shard, state, h, step, coef)
        check_sources(w, snap)
        c = 1.0 if coef is None else f32(coef)
        for r in range(n):
            assert bits_equal(flat[r], g_plain[r]), "the norm pass's fp32 shard is bg_reduce_scatter_acc's"
            g_pool = (g_plain[r].double() * c).float()                  # the local step's one rounding
            check_step("plain rank %d" % r, outs["plain"][r], state[r], g_plain[r], h, step)
            check_step("clip %s rank %d" % (coef, r), outs["clip"][r], state[r], g_clip[r], h, step)
            check_step("pool %s rank %d" % (coef, r), outs["pool"][r], state[r], g_pool, h, step)
            for i in range(3):
                if coef is None or coef == 1.0:
                    assert bits_equal(outs["clip"][r][i], outs["plain"][r][i]), ("clip == plain", coef, i)
                if coef is None or coef == 1.0 or pow2(post):
                    assert bits_equal(outs["pool"][r][i], outs["clip"][r][i]), ("pool == clip", coef, post, i)
            if lr == 0.0:
                assert bits_equal(outs["plain"][r][0], state[r][0]) and bits_equal(outs["clip"][r][0], state[r][0])
                assert bits_equal(outs["pool"][r][0], state[r][0])
        state = [[t.clone() for t in outs["plain"][r]] for r in range(n)]   # the next step starts from the kernel's own state


@pytest.mark.parametrize("dt", [BF, F32], ids=["bf16", "fp32"])
def test_adamw_grid_independent(world, bg, dt):
    """the same step from the same random state at comm_ctas (local_ctas for a group of one) 1, 3 and 16, on 2.5 grid-stride
    spans plus 3 vectors: bit-identical (p, m, v) on every path, and the same fp32 shard from the norm pass"""
    w, n = world, world.n
    e = 8 if dt == BF else 4
    shard = (5 * CTAS * THREADS * v_opt(n) // 2 + 3) * e
    write_sources(w, shard, dt, 1e-2)
    state = [random_state(w, shard, 1e-2) for _ in range(n)]
    res = []
    for ctas in (1, 3, 16):
        with tunables(bg, comm_ctas=ctas, local_ctas=ctas):
            outs, flat = run_paths(w, dt, shard, state, HYPER["defaults"], 10, 0.3)
        res.append((outs, flat))
    for outs, flat in res[1:]:
        for r in range(n):
            assert bits_equal(flat[r], res[0][1][r])
            for k in outs:
                for i in range(3):
                    assert bits_equal(outs[k][r][i], res[0][0][k][r][i]), (k, r, i)


# ---- the norm pass --------------------------------------------------------------------------------------------------------------
def skip_sets(shard):
    """skip-range sets for a shard: bounds are multiples of 8 inside the shard (s8 = its last multiple of 8 when the fp32 shard is
    not a whole number of 8-element groups)"""
    s8 = shard // 8 * 8
    sets = {"none": [], "empty": [(0, 0)], "empty_mid": [(s8 // 16 * 8, s8 // 16 * 8)]}
    if s8 >= 8:
        sets["first"] = [(0, 8)]
        sets["to_end"] = [(max(0, s8 - 24), s8)]
        sets["whole"] = [(0, s8)]
    if s8 >= 64:
        sets["adjacent"] = [(8, 24), (24, 40)]
        sets["overlap"] = [(16, 48), (32, 64), (40, 56)]
        step = s8 // 16 // 8 * 8
        sets["max_skip"] = [(k * step, k * step + 8) for k in range(16)]
    return sets


@pytest.mark.parametrize("shard_name", SHARD_NAMES)
@pytest.mark.parametrize("dt", [BF, F32], ids=["bf16", "fp32"])
def test_norm_pass_against_float64(world, bg, dt, shard_name):
    """The sum of the per-warp partials against the float64 sum of g_i^2 over the elements outside every skip range, g_i the fp32
    shard the same call writes to dst (itself bg_reduce_scatter_acc's output, bit for bit).  g_i^2 is exact in float64; what is
    left is one fp32 rounding per warp partial (u * total) and float64 rounding: the per-thread fma chains of k elements, the
    five warp-shuffle levels, the sum of the W partials here and the reference's own sum of the shard's squares, hence
    u * total + (k + 5 + W + shard) * 2^-53 * total.  A range covering the whole shard gives exactly 0.  The partials past the
    launch's 4 * grid warps are zero, and nothing before them is NaN.  The partials are fp32, so the large edge values are 1e15
    here (a warp's sum of squares of 1e18 gradients exceeds the fp32 range)."""
    w, n = world, world.n
    table = shards(n, dt)
    if shard_name not in table:
        pytest.skip("2^24 elements per rank only for groups of at most 2")
    shard = table[shard_name]
    e = 8 if dt == BF else 4
    post = f32(1.0 / w.post)
    snap = write_sources(w, shard, dt, 1e-2, huge=1e15)
    want_dst = acc_grad(w, shard, dt, [post] * n)
    nvec = shard // e
    grid = comm_grid(nvec, v_opt(n))
    k = -(-nvec // (grid * THREADS)) * e
    n_parts = 4 * CTAS + 36
    for name, ranges in skip_sets(shard).items():
        dst = [Guarded(shard, w.gen) for _ in range(n)]
        parts = [torch.full((n_parts,), float("nan"), device="cuda") for _ in range(n)]
        w.run(lambda r, c: c.reduce_scatter_sumsq(w.group, w.sym[r], dt, shard, 1.0 / w.pre, post, parts[r], ranges, dst=dst[r].t))
        check_sources(w, snap)
        keep = torch.ones(shard, dtype=torch.bool, device="cuda")
        for lo, hi in ranges:
            keep[lo:hi] = False
        for r in range(n):
            dst[r].check()
            assert bits_equal(dst[r].t, want_dst[r]), name
            assert not torch.isnan(parts[r][:4 * grid]).any(), name
            assert bool((parts[r][4 * grid:] == 0).all()), (name, "tail of partials not zeroed")
            got = float(parts[r].double().sum())
            want = float((dst[r].t.double()[keep] ** 2).sum())
            if not bool(keep.any()):
                assert got == 0.0, (name, got)
                continue
            tol = U * want + (k + 5 + 4 * grid + shard) * 2.0 ** -53 * want
            assert abs(got - want) <= tol, (name, r, got, want, abs(got - want) / want)

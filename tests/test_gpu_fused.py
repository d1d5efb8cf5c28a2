"""GPU parity of the fused GEMM + collective kernels (through the C ABI), on ONE H100: n virtual ranks (n contexts, n arenas) on
the device, every rank's kernels on its own streams, so the real cross-rank protocol runs -- partial tiles TMA-stored into the
owner's arena, per-tile / per-block arrival counters, the tile reducer's broadcast and exit barrier, the chunk-signalled push
kernel beside the gathering GEMM.  Checked against float64 references of the same bf16 operands, with integer data (exact:
every partial and every sum is an integer below 2^24) and with real data (a derived bound), and against the plain wgmma GEMM:

  GEMM + reduce-scatter (C8)   == bf16(sum_r bf16(P_r)) of every rank's partial P_r: bit for bit (integers), run-to-run identical
  GEMM + all-reduce (C5/C6)    == the same rows on EVERY member, bit-identical across members, runs and the reduce-scatter
  all-gather + GEMM (C7)       == plain GEMM on the concatenated operand, BIT-EXACT (same tiles, same accumulation order), and
                                  the correctly rounded exact product (integers)

Results start as NaN and are followed by sentinel guards (also after the partial region peers store into), so an unwritten
element or a stray store fails.
The same operations at real NVLink scale are exercised by bench.py's path legs and scripts/test_fused_collectives.py (N GPUs)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from _fp_check import BF, assert_rounded, gamma, gemm_eps, ulp_bf16  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

FLAG_BYTES = 1 << 16
GUARD = 128                  # sentinel rows after each result region: one tile row
SENTINEL = 0x3F5A            # bf16 bits of 0.8515625


@pytest.fixture(scope="module")
def bg():
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import hetu_galvatron_b200._bg as bg
    bg.lib()
    bg.set_tunable("timeout_ms", 8000)
    bg.set_tunable("comm_ctas", 16)
    yield bg
    bg.set_tunable("comm_ctas", 132)


class World:
    def __init__(self, bg, n, arena=768 << 20):
        from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
        self.bg, self.n = bg, n
        self.comms = bg.BgComm.local_world(n, device=0, arena_bytes=arena)
        self.group = CommGroup(list(range(n)))
        self.streams = [torch.cuda.Stream() for _ in range(n)]
        # communication streams are HIGH priority (as in the backend): the CTA distributor serves a high-priority grid before a
        # low-priority one that is waiting for an SM (here: another virtual rank's 128-CTA GEMM), so a push kernel is never
        # stuck behind a GEMM that cannot be placed yet
        self.comm_streams = [torch.cuda.Stream(priority=-1) for _ in range(n)]

    def sym(self, nbytes):
        bufs = [c.sym_alloc(self.group, nbytes) for c in self.comms]
        for c in self.comms:
            c.exchange()
        for b in bufs:
            b.u8.zero_()
        return bufs

    def run(self, fn):
        torch.cuda.synchronize()
        for r, c in enumerate(self.comms):
            with torch.cuda.stream(self.streams[r]):
                fn(r, c)
        try:
            torch.cuda.synchronize()
        except Exception as exc:      # a device-side timeout traps the kernel; its who/where record survives in mapped host memory
            raise AssertionError("device fault: %s; error records %s" % (str(exc).splitlines()[0], [c.error_info() for c in self.comms]))
        for c in self.comms:
            assert c.error_flag() == 0, c.error_info()

    def close(self):
        torch.cuda.synchronize()
        for c in self.comms:
            c.close()


@pytest.fixture(scope="module", params=[2, 4])
def world(request, bg):
    w = World(bg, request.param)
    yield w
    w.close()


def _operands(n, m, nn, k, layout, seed, kind):
    """every rank's stored operands a_r, b_r of `layout` (M = m, the full product's rows) and their float64 partial products
    P_r = A_r op B_r with the sums of |terms| S_r = |A_r| op |B_r|"""
    g = torch.Generator(device="cpu").manual_seed(seed)

    def rand(*shape):
        if kind == "int":
            return torch.randint(-8, 9, shape, generator=g).to(torch.bfloat16).cuda()
        return (torch.randn(*shape, generator=g) * 0.5).to(torch.bfloat16).cuda()
    a = [rand(k, m) if layout == "nt" else rand(m, k) for _ in range(n)]
    b = [rand(nn, k) if layout == "tn" else rand(k, nn) for _ in range(n)]
    A = [x.double().t() if layout == "nt" else x.double() for x in a]
    B = [w.double().t() if layout == "tn" else w.double() for w in b]
    return a, b, [x @ w for x, w in zip(A, B)], [x.abs() @ w.abs() for x, w in zip(A, B)]


def _check_reduced(got, parts, sums, kind, k, what):
    """The fused reduce-scatter / all-reduce result is bf16(sum_r bf16(P_r)): every rank's partial tile is rounded to bf16 once
    when it is shipped, the owner sums the p partials in fp32 in rank order and rounds once more.
      int:  every term is an integer below 2^24, so the formula is exact in fp32 and the result must match it bit for bit.
      real: |result - sum_r P_r| <= sum_r (gemm_eps_r + 1/2 ulp_bf16(|P_r| + gemm_eps_r))   (each partial, then its rounding)
                                   + gamma(p) * sum_r 2 (|P_r| + gemm_eps_r)                   (the fp32 sum of the p partials)
            + half an ulp of the final rounding (assert_rounded)."""
    if kind == "int":
        assert max(float(x.abs().max()) for x in parts) > 256 and any(bool((x.to(BF).double() != x).any()) for x in parts), \
            "the partials must exercise their own bf16 rounding"
        want = sum(x.to(BF).double() for x in parts)
        assert float(want.abs().max()) < 2 ** 24
        bad = got.view(torch.int16) != want.to(BF).view(torch.int16)
        assert not bad.any(), "%s: %d / %d elements differ from bf16(sum_r bf16(P_r))" % (what, int(bad.sum()), bad.numel())
    else:
        e = [gemm_eps(k, s) for s in sums]
        t = [x.abs() + er for x, er in zip(parts, e)]
        eps = sum(er + 0.5 * ulp_bf16(tr) for er, tr in zip(e, t)) + gamma(len(parts)) * 2 * sum(t)
        assert_rounded(got, sum(parts), eps, what)


def _guarded(rows, nn):
    """a NaN-filled bf16 [rows][nn] tensor followed by a guard of GUARD sentinel rows; returns (tensor, guard)"""
    buf = torch.full(((rows + GUARD) * nn,), SENTINEL, device="cuda", dtype=torch.int16)
    t = buf[:rows * nn].view(BF).view(rows, nn)
    t.fill_(float("nan"))
    return t, buf[rows * nn:]


def _assert_guard(guard, what):
    bad = int((guard.view(torch.int16) != SENTINEL).sum())
    assert bad == 0, "%s: %d guard elements written" % (what, bad)


LAYOUT = {"tn": 0, "nn": 1, "nt": 2}
# the existing shapes, then K tails inside (72) and across (1000) the 64-deep k-block, 8-column tails of the 128-wide fused tile
# (8: one tile of 8 live columns; 136: a second tile of 8) and the NT layout
SCATTER_CASES = [(128, 256, 128, "tn"), (256, 512, 320, "tn"), (256, 264, 512, "nn"), (1024, 1024, 1024, "tn"),
                 (128, 8, 72, "tn"), (256, 136, 1000, "nt"), (128, 136, 72, "nn"), (256, 8, 1000, "nt"), (128, 136, 1000, "tn")]


@pytest.mark.parametrize("m_per,nn,k,layout", SCATTER_CASES)
def test_gemm_reduce_scatter(world, m_per, nn, k, layout):
    n = world.n
    m = m_per * n
    region, guard = m * nn * 2, GUARD * nn * 2
    bufs = world.sym(region + guard + FLAG_BYTES)        # [partials | guard | counters]
    for bf in bufs:
        bf.u8[region:region + guard].view(torch.int16).fill_(SENTINEL)
    code = LAYOUT[layout]
    for kind in ("int", "real"):
        a, b, parts, sums = _operands(n, m, nn, k, layout, 100 + m + nn + k, kind)
        outs = []
        for rep in range(2):
            out, out_guard = zip(*[_guarded(m_per, nn) for _ in range(n)])
            world.run(lambda r, c: c.gemm_reduce_scatter(world.group, a[r], b[r], m, nn, k, code, bufs[r], 0, region + guard, out[r]))
            for r in range(n):
                _assert_guard(out_guard[r], "after out, rank %d" % r)
                _assert_guard(bufs[r].u8[region:region + guard], "after the partials, rank %d" % r)
            outs.append(out)
        for r in range(n):
            rows = slice(r * m_per, (r + 1) * m_per)
            _check_reduced(outs[0][r], [x[rows] for x in parts], [x[rows] for x in sums], kind, k, "%s rank %d" % (kind, r))
            assert torch.equal(outs[0][r].view(torch.int16), outs[1][r].view(torch.int16))      # deterministic


@pytest.mark.parametrize("m_per,nn,k,layout", SCATTER_CASES)
def test_gemm_all_reduce(world, m_per, nn, k, layout):
    n = world.n
    m = m_per * n
    region, guard = m * nn * 2, GUARD * nn * 2
    res, flags = region + guard, 2 * (region + guard)
    bufs = world.sym(flags + FLAG_BYTES)                 # [partials | guard | result | guard | counters]
    for bf in bufs:
        for g0 in (region, res + region):
            bf.u8[g0:g0 + guard].view(torch.int16).fill_(SENTINEL)
    code = LAYOUT[layout]
    for kind in ("int", "real"):
        a, b, parts, sums = _operands(n, m, nn, k, layout, 200 + m + nn + k, kind)
        results = []
        for rep in range(2):
            for bf in bufs:
                bf.u8[res:res + region].view(torch.bfloat16).fill_(float("nan"))
            world.run(lambda r, c: c.gemm_all_reduce(world.group, a[r], b[r], m, nn, k, code, bufs[r], 0, flags, res))
            for r, bf in enumerate(bufs):
                for g0 in (region, res + region):
                    _assert_guard(bf.u8[g0:g0 + guard], "rank %d guard at byte %d" % (r, g0))
            results.append([bf.u8[res:res + region].view(torch.bfloat16).view(m, nn).clone() for bf in bufs])
        _check_reduced(results[0][0], parts, sums, kind, k, kind)
        for r in range(1, n):      # replicas bit-identical across the group
            assert torch.equal(results[0][r].view(torch.int16), results[0][0].view(torch.int16))
        assert torch.equal(results[1][0].view(torch.int16), results[0][0].view(torch.int16))    # and across runs
        # the fused all-reduce == fused reduce-scatter + exact all-gather: same bits as the reduce-scatter variant
        out = [torch.zeros(m_per, nn, device="cuda", dtype=torch.bfloat16) for _ in range(n)]
        world.run(lambda r, c: c.gemm_reduce_scatter(world.group, a[r], b[r], m, nn, k, code, bufs[r], 0, flags, out[r]))
        assert torch.equal(torch.cat(out).view(torch.int16), results[0][0].view(torch.int16))


@pytest.mark.parametrize("m_per,nn,k,layout", [(128, 256, 128, "tn"), (256, 520, 320, "tn"), (384, 256, 512, "nn"), (1024, 1024, 1024, "tn"),
                                               (128, 8, 72, "tn"), (256, 136, 1000, "nn"), (128, 136, 1000, "tn")])
def test_all_gather_gemm_bit_exact(world, bg, m_per, nn, k, layout):
    n = world.n
    m = m_per * n
    code = LAYOUT[layout]
    stage = m * k * 2
    bufs = world.sym(stage + FLAG_BYTES)
    for kind in ("int", "real"):
        g = torch.Generator(device="cpu").manual_seed(300 + m + nn + k)

        def rand(*shape):
            if kind == "int":
                return torch.randint(-8, 9, shape, generator=g).to(torch.bfloat16).cuda()
            return (torch.randn(*shape, generator=g) * 0.5).to(torch.bfloat16).cuda()
        a_loc = [rand(m_per, k) for _ in range(n)]
        a_full = torch.cat(a_loc)
        bw = [rand(nn, k) if code == 0 else rand(k, nn) for _ in range(n)]
        for rep in range(2):        # twice: counters must return to rest and the staging be reusable
            out, out_guard = zip(*[_guarded(m, nn) for _ in range(n)])
            world.run(lambda r, c: c.all_gather_gemm(world.group, a_loc[r], bw[r], out[r], m, nn, k, code, bufs[r], 0, stage,
                                                     world.comm_streams[r]))
            for r in range(n):
                _assert_guard(out_guard[r], "after c, rank %d" % r)
                want = torch.empty(m, nn, device="cuda", dtype=torch.bfloat16)
                bg.gemm_bf16(a_full, bw[r], want, m, nn, k, code)
                torch.cuda.synchronize()
                assert torch.equal(out[r].view(torch.int16), want.view(torch.int16)), "rank %d rep %d" % (r, rep)
                if kind == "int":       # and both equal the correctly rounded exact product (a shared epilogue bug cannot hide)
                    exact = a_full.double() @ (bw[r].double().t() if code == 0 else bw[r].double())
                    assert torch.equal(out[r].view(torch.int16), exact.to(BF).view(torch.int16)), "rank %d rep %d" % (r, rep)
                # the gathered operand sits complete in staging afterwards (the wgrad GEMM reads it there)
                got_a = bufs[r].u8[:stage].view(torch.bfloat16).view(m, k)
                assert torch.equal(got_a.view(torch.int16), a_full.view(torch.int16))
                assert int(bufs[r].u8[stage:].view(torch.int32).abs().sum()) == 0        # counters cleared


def test_fused_reject_m_not_split_into_row_blocks(world, bg):
    """M that is not a multiple of p*128 is refused with BG_EINVAL on every rank by all three fused entries, before anything is
    launched (no entry barrier, no push); the symmetric buffers are large enough that only this check can refuse the call.
    A valid call in the same world afterwards finds the barrier flags and arrival counters at rest."""
    n = world.n
    m, nn, k = n * 128 + 64, 128, 64
    a = [torch.zeros(m, k, device="cuda", dtype=BF) for _ in range(n)]
    b = [torch.zeros(nn, k, device="cuda", dtype=BF) for _ in range(n)]
    c = [torch.zeros(m, nn, device="cuda", dtype=BF) for _ in range(n)]
    region = max(m * nn, m * k) * 2
    bufs = world.sym(2 * region + FLAG_BYTES)
    calls = {
        "bg_gemm_reduce_scatter": lambda r, cm: cm.gemm_reduce_scatter(world.group, a[r], b[r], m, nn, k, 0, bufs[r], 0, 2 * region, c[r]),
        "bg_gemm_all_reduce": lambda r, cm: cm.gemm_all_reduce(world.group, a[r], b[r], m, nn, k, 0, bufs[r], 0, 2 * region, region),
        "bg_all_gather_gemm": lambda r, cm: cm.all_gather_gemm(world.group, a[r], b[r], c[r], m, nn, k, 0, bufs[r], 0, 2 * region,
                                                                world.comm_streams[r]),
    }
    for name, call in calls.items():
        errors = []

        def bad(r, cm):
            with pytest.raises(bg.BgError) as e:
                call(r, cm)
            errors.append(str(e.value))
        before = bg.launch_count()
        world.run(bad)
        assert bg.launch_count() == before, "%s launched %d kernels before refusing" % (name, bg.launch_count() - before)
        want = "bg_galvatron error -1: %s: M=%d must be a multiple of p*128" % (name, m)
        assert errors == [want] * n, errors
    # the same world still runs a valid call
    m = n * 128
    a, b, parts, sums = _operands(n, m, nn, k, "tn", 7, "int")
    out = [torch.full((128, nn), float("nan"), device="cuda", dtype=BF) for _ in range(n)]
    world.run(lambda r, cm: cm.gemm_reduce_scatter(world.group, a[r], b[r], m, nn, k, 0, bufs[r], 0, 2 * region, out[r]))
    for r in range(n):
        rows = slice(r * 128, (r + 1) * 128)
        _check_reduced(out[r], [x[rows] for x in parts], [x[rows] for x in sums], "int", k, "rank %d" % r)

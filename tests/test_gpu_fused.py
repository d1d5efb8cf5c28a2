"""GPU parity of the fused GEMM + collective kernels (through the C ABI), on ONE H100: n virtual ranks (n contexts, n arenas) on
the device, every rank's kernels on its own streams, so the real cross-rank protocol runs -- partial tiles TMA-stored into the
owner's arena, per-tile / per-block arrival counters, the tile reducer's broadcast and exit barrier, the chunk-signalled push
kernel beside the gathering GEMM.  Checked against (a) the plain wgmma GEMM on the same operands and (b) an fp32 torch matmul:

  GEMM + reduce-scatter (C8)   == reduce_scatter(sum_r A_r op B_r): <= 1 bf16 ulp of the fp32 sum, run-to-run bit-identical
  GEMM + all-reduce (C5/C6)    == the same rows on EVERY member, bit-identical across members and runs
  all-gather + GEMM (C7)       == plain GEMM on the concatenated operand, BIT-EXACT (same tiles, same accumulation order)

The same operations at real NVLink scale are exercised by bench.py's path legs and scripts/test_fused_collectives.py (N GPUs)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

FLAG_BYTES = 1 << 16


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


def _operands(n, m, nn, k, layout, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = [(torch.randn(m, k, generator=g) * 0.5).to(torch.bfloat16).cuda() for _ in range(n)]
    if layout == "tn":
        b = [(torch.randn(nn, k, generator=g) * 0.5).to(torch.bfloat16).cuda() for _ in range(n)]
        ref = [x.float() @ w.float().t() for x, w in zip(a, b)]
    else:
        b = [(torch.randn(k, nn, generator=g) * 0.5).to(torch.bfloat16).cuda() for _ in range(n)]
        ref = [x.float() @ w.float() for x, w in zip(a, b)]
    return a, b, ref


def _ulp_close(got, partials32):
    """The fused kernels ship every rank's partial tile as bf16 (half an ulp each: |partial| * 2^-8), sum the p partials in fp32 in
    a fixed order and round once more: |got - exact| <= (sum_r |partial_r| + |sum|) * 2^-8 (+ the fp32 accumulation-order noise
    of a K-long dot product)."""
    want32 = sum(partials32)
    tol = (sum(p.abs() for p in partials32) + want32.abs()) * 2 ** -8 * 1.01 + 1e-2
    err = (got.float() - want32).abs()
    assert bool((err <= tol).all()), float((err - tol).max())


@pytest.mark.parametrize("m_per,nn,k,layout", [(128, 256, 128, "tn"), (256, 512, 320, "tn"), (256, 264, 512, "nn"), (1024, 1024, 1024, "tn")])
def test_gemm_reduce_scatter(world, m_per, nn, k, layout):
    n = world.n
    m = m_per * n
    a, b, ref = _operands(n, m, nn, k, layout, 100 + m + nn)
    bufs = world.sym(m * nn * 2 + FLAG_BYTES)
    code = 0 if layout == "tn" else 1
    outs = []
    for rep in range(2):
        out = [torch.zeros(m_per, nn, device="cuda", dtype=torch.bfloat16) for _ in range(n)]
        world.run(lambda r, c: c.gemm_reduce_scatter(world.group, a[r], b[r], m, nn, k, code, bufs[r], 0, m * nn * 2, out[r]))
        outs.append(out)
    for r in range(n):
        _ulp_close(outs[0][r], [x[r * m_per:(r + 1) * m_per] for x in ref])
        assert torch.equal(outs[0][r].view(torch.int16), outs[1][r].view(torch.int16))      # deterministic


@pytest.mark.parametrize("m_per,nn,k,layout", [(128, 256, 128, "tn"), (256, 512, 320, "tn"), (256, 264, 512, "nn"), (1024, 1024, 1024, "tn")])
def test_gemm_all_reduce(world, m_per, nn, k, layout):
    n = world.n
    m = m_per * n
    a, b, ref = _operands(n, m, nn, k, layout, 200 + m + nn)
    region = m * nn * 2
    bufs = world.sym(2 * region + FLAG_BYTES)       # [partials | result | counters]
    code = 0 if layout == "tn" else 1
    results = []
    for rep in range(2):
        for bf in bufs:
            bf.u8[region:2 * region].zero_()
        world.run(lambda r, c: c.gemm_all_reduce(world.group, a[r], b[r], m, nn, k, code, bufs[r], 0, 2 * region, region))
        results.append([bf.u8[region:2 * region].view(torch.bfloat16).view(m, nn).clone() for bf in bufs])
    _ulp_close(results[0][0], ref)
    for r in range(1, n):      # replicas bit-identical across the group
        assert torch.equal(results[0][r].view(torch.int16), results[0][0].view(torch.int16))
    assert torch.equal(results[1][0].view(torch.int16), results[0][0].view(torch.int16))    # and across runs
    # the fused all-reduce == fused reduce-scatter + exact all-gather: same bits as the reduce-scatter variant
    out = [torch.zeros(m_per, nn, device="cuda", dtype=torch.bfloat16) for _ in range(n)]
    world.run(lambda r, c: c.gemm_reduce_scatter(world.group, a[r], b[r], m, nn, k, code, bufs[r], 0, 2 * region, out[r]))
    assert torch.equal(torch.cat(out).view(torch.int16), results[0][0].view(torch.int16))


@pytest.mark.parametrize("m_per,nn,k,layout", [(128, 256, 128, "tn"), (256, 520, 320, "tn"), (384, 256, 512, "nn"), (1024, 1024, 1024, "tn")])
def test_all_gather_gemm_bit_exact(world, bg, m_per, nn, k, layout):
    n = world.n
    m = m_per * n
    g = torch.Generator(device="cpu").manual_seed(300 + m + nn)
    a_loc = [(torch.randn(m_per, k, generator=g) * 0.5).to(torch.bfloat16).cuda() for _ in range(n)]
    a_full = torch.cat(a_loc)
    code = 0 if layout == "tn" else 1
    bw = [((torch.randn(nn, k, generator=g) if code == 0 else torch.randn(k, nn, generator=g)) * 0.5).to(torch.bfloat16).cuda() for _ in range(n)]
    stage = m * k * 2
    bufs = world.sym(stage + FLAG_BYTES)
    for rep in range(2):        # twice: counters must return to rest and the staging be reusable
        out = [torch.zeros(m, nn, device="cuda", dtype=torch.bfloat16) for _ in range(n)]
        world.run(lambda r, c: c.all_gather_gemm(world.group, a_loc[r], bw[r], out[r], m, nn, k, code, bufs[r], 0, stage,
                                                 world.comm_streams[r]))
        for r in range(n):
            want = torch.empty(m, nn, device="cuda", dtype=torch.bfloat16)
            bg.gemm_bf16(a_full, bw[r], want, m, nn, k, code)
            torch.cuda.synchronize()
            assert torch.equal(out[r].view(torch.int16), want.view(torch.int16)), "rank %d rep %d" % (r, rep)
            # the gathered operand sits complete in staging afterwards (the wgrad GEMM reads it there)
            got_a = bufs[r].u8[:stage].view(torch.bfloat16).view(m, k)
            assert torch.equal(got_a.view(torch.int16), a_full.view(torch.int16))
            assert int(bufs[r].u8[stage:].view(torch.int32).abs().sum()) == 0        # counters cleared

"""GPU parity of the peer-memory collectives (through the C ABI) against oracle/collectives_ref.py.

One H100 is enough: ``BgComm.local_world(n)`` creates n virtual ranks (n contexts, n arenas) on the device and
every rank's kernel runs on its own stream, so the real cross-rank protocol (device barriers, peer loads/stores
through the peer-pointer table) is what executes.  Integer/byte-moving paths are checked bit-exact; reductions
against the fp64 "exact" oracle (fp32 accumulate => 1e-6) and against the reference-order oracle (bf16 rounding).
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


@pytest.fixture(scope="module")
def bg():
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import hetu_galvatron_b200._bg as bg
    bg.lib()
    bg.set_tunable("timeout_ms", 20000)
    bg.set_tunable("comm_ctas", 16)  # 8 virtual ranks x 16 slim CTAs stay co-resident on one device
    return bg


@pytest.fixture(scope="module")
def ref():
    from oracle import collectives_ref
    return collectives_ref


class World:
    def __init__(self, bg, n, arena=512 << 20):
        from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
        self.bg, self.n = bg, n
        self.comms = bg.BgComm.local_world(n, device=0, arena_bytes=arena)
        self.group = CommGroup(list(range(n)))
        self.streams = [torch.cuda.Stream() for _ in range(n)]

    def sym(self, nbytes):
        bufs = [c.sym_alloc(self.group, nbytes) for c in self.comms]
        for c in self.comms:
            c.exchange()
        return bufs

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


@pytest.fixture(scope="module", params=[2, 4, 8])
def world(request, bg):
    w = World(bg, request.param)
    yield w
    w.close()


def test_barrier_and_repeat(world):
    for _ in range(5):
        world.run(lambda r, c: c.barrier(world.group))


@pytest.mark.parametrize("shard", [8, 1000 * 8, 1 << 20])
@pytest.mark.parametrize("src_dtype", [torch.float32, torch.bfloat16])
def test_all_gather_cast_bit_exact(world, ref, shard, src_dtype):
    n = world.n
    g = torch.Generator(device="cpu").manual_seed(1234 + shard)
    shards = [(torch.randn(shard, generator=g) * 3).to(src_dtype) for _ in range(n)]
    want = ref.all_gather_cast(shards)
    dst = world.sym(shard * n * 2)
    dev = [s.cuda() for s in shards]
    for _ in range(2):  # twice: the flags must return to rest and the buffers be reusable
        for b in dst:
            b.view(torch.bfloat16).zero_()
        world.run(lambda r, c: c.all_gather_cast(world.group, dev[r], dst[r]))
        for r in range(n):
            got = dst[r].view(torch.bfloat16, shard * n).cpu()
            assert torch.equal(got.view(torch.int16), want[r].view(torch.int16)), f"rank {r}"


@pytest.mark.parametrize("shard", [8, 1000 * 8, 1 << 19])
@pytest.mark.parametrize("accumulate", [False, True])
def test_reduce_scatter_acc(world, ref, shard, accumulate):
    n = world.n
    g = torch.Generator(device="cpu").manual_seed(99 + shard)
    srcs = [torch.randn(shard * n, generator=g).to(torch.bfloat16) for _ in range(n)]
    prev = [torch.randn(shard, generator=g) for _ in range(n)]
    pre, post = ref.fsdp_divide_factors(n)
    exact = ref.reduce_scatter_acc(srcs, prev, order="exact", accumulate=accumulate)
    refo = ref.reduce_scatter_acc(srcs, prev, order="reference", accumulate=accumulate)
    sym = world.sym(shard * n * 2)
    for r in range(n):
        sym[r].view(torch.bfloat16, shard * n).copy_(srcs[r])
    dst = [p.clone().cuda() for p in prev]
    world.run(lambda r, c: c.reduce_scatter_acc(world.group, sym[r], torch.bfloat16, dst[r], prescale=1.0 / pre,
                                                postscale=1.0 / post, accumulate=accumulate))
    for r in range(n):
        got = dst[r].cpu()
        torch.testing.assert_close(got, exact[r], rtol=2e-6, atol=2e-6)
        # the reference rounds to bf16 after every hop of the sum (<= n roundings of 2^-9 relative each)
        absmax = max(float(s_.abs().max()) for s_ in srcs)
        assert float((got - refo[r]).abs().max()) <= n * 2 ** -8 * absmax
    # sources untouched
    for r in range(n):
        assert torch.equal(sym[r].view(torch.bfloat16, shard * n).cpu().view(torch.int16), srcs[r].view(torch.int16))


def test_reduce_scatter_fp32_and_bf16_out(world, ref):
    n, shard = world.n, 4096
    g = torch.Generator(device="cpu").manual_seed(5)
    srcs32 = [torch.randn(shard * n, generator=g) for _ in range(n)]
    sym = world.sym(shard * n * 4)
    for r in range(n):
        sym[r].view(torch.float32, shard * n).copy_(srcs32[r])
    dst = [torch.zeros(shard, device="cuda") for _ in range(n)]
    world.run(lambda r, c: c.reduce_scatter_acc(world.group, sym[r], torch.float32, dst[r], prescale=0.5, postscale=0.25))
    for r in range(n):
        want = sum(s[r * shard:(r + 1) * shard].double() for s in srcs32) * 0.125
        torch.testing.assert_close(dst[r].cpu().double(), want, rtol=1e-6, atol=1e-6)
    # bf16 -> bf16 (Megatron-SP reduce-scatter of activations, mappings_group.py:105-122)
    srcs = [s.to(torch.bfloat16) for s in srcs32]
    symb = world.sym(shard * n * 2)
    for r in range(n):
        symb[r].view(torch.bfloat16, shard * n).copy_(srcs[r])
    dstb = [torch.zeros(shard, device="cuda", dtype=torch.bfloat16) for _ in range(n)]
    world.run(lambda r, c: c.reduce_scatter_acc(world.group, symb[r], torch.bfloat16, dstb[r]))
    for r in range(n):
        want = sum(s[r * shard:(r + 1) * shard].double() for s in srcs).to(torch.bfloat16)
        torch.testing.assert_close(dstb[r].cpu().float(), want.float(), rtol=2 ** -7, atol=1e-6)


@pytest.mark.parametrize("elems,twoshot", [(8, False), (8 * 1024, False), (8 * 1024 * 8, True), (1 << 21, True)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_all_reduce_sum(world, ref, bg, elems, twoshot, dtype):
    n = world.n
    bg.set_tunable("oneshot_bytes", 1 if twoshot else 1 << 40)
    try:
        g = torch.Generator(device="cpu").manual_seed(7 + elems)
        srcs = [torch.randn(elems, generator=g).to(dtype) for _ in range(n)]
        want = ref.all_reduce(srcs, order="exact")[0]
        sym = world.sym(elems * srcs[0].element_size())
        for r in range(n):
            sym[r].view(dtype, elems).copy_(srcs[r])
        dst = [torch.zeros(elems, device="cuda", dtype=dtype) for _ in range(n)]
        world.run(lambda r, c: c.all_reduce(world.group, sym[r], dst[r]))
        outs = [d.cpu() for d in dst]
        for r in range(1, n):  # replicas must stay bit-identical across the group
            assert torch.equal(outs[r].view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                               outs[0].view(torch.int16 if dtype == torch.bfloat16 else torch.int32))
        if dtype == torch.bfloat16:  # fp32 accumulate, one rounding (<= 1 ulp from the fp64 answer)
            torch.testing.assert_close(outs[0].float(), want.float(), rtol=2 ** -7, atol=1e-6)
            assert float((outs[0].view(torch.int16) != want.view(torch.int16)).float().mean()) < 1e-3
        else:
            torch.testing.assert_close(outs[0], want, rtol=2e-6, atol=2e-6)
    finally:
        bg.set_tunable("oneshot_bytes", 512 * 1024)


def test_all_reduce_max_fp32(world, ref, bg):
    n, elems = world.n, 4096
    g = torch.Generator(device="cpu").manual_seed(3)
    srcs = [torch.randn(elems, generator=g) for _ in range(n)]
    want = ref.all_reduce(srcs, op="max")[0]
    sym = world.sym(elems * 4)
    for r in range(n):
        sym[r].view(torch.float32, elems).copy_(srcs[r])
    dst = [torch.zeros(elems, device="cuda") for _ in range(n)]
    world.run(lambda r, c: c.all_reduce(world.group, sym[r], dst[r], op=bg.MAX))
    for r in range(n):
        assert torch.equal(dst[r].cpu(), want)


@pytest.mark.parametrize("b,s,heads,d", [(1, 64, 8, 16), (2, 128, 16, 64), (1, 256, 8, 128)])
def test_ulysses_all_to_all_bit_exact(world, ref, bg, b, s, heads, d):
    p = world.n
    if heads % p or s % p:
        pytest.skip("heads/seq not divisible")
    g = torch.Generator(device="cpu").manual_seed(11)
    # forward direction: [b, s/p, n, d] -> [b, s, n/p, d], q and k (GQA: half the heads) in ONE launch
    kv_heads = heads if (heads // 2) % p else heads // 2
    qs = [torch.randn(b, s // p, heads, d, generator=g).to(torch.bfloat16) for _ in range(p)]
    ks = [torch.randn(b, s // p, kv_heads, d, generator=g).to(torch.bfloat16) for _ in range(p)]
    want_q, want_k = ref.ulysses_all_to_all(qs, 2, 1), ref.ulysses_all_to_all(ks, 2, 1)
    sq, sk = world.sym(qs[0].numel() * 2), world.sym(ks[0].numel() * 2)
    for r in range(p):
        sq[r].view(torch.bfloat16, qs[r].numel()).copy_(qs[r].flatten())
        sk[r].view(torch.bfloat16, ks[r].numel()).copy_(ks[r].flatten())
    oq = [torch.zeros(b, s, heads // p, d, device="cuda", dtype=torch.bfloat16) for _ in range(p)]
    ok = [torch.zeros(b, s, kv_heads // p, d, device="cuda", dtype=torch.bfloat16) for _ in range(p)]

    def desc_fwd(src, dst, n_heads):
        hp = n_heads // p
        return dict(src=src, dst=dst, batch=b, rows=s // p, row_elems=hp * d, src_bs=(s // p) * n_heads * d, src_rs=n_heads * d,
                    src_me_off=hp * d, dst_bs=s * hp * d, dst_rs=hp * d, dst_peer_off=(s // p) * hp * d)

    world.run(lambda r, c: c.all_to_all_rows(world.group, [desc_fwd(sq[r], oq[r], heads), desc_fwd(sk[r], ok[r], kv_heads)],
                                             torch.bfloat16))
    for r in range(p):
        assert torch.equal(oq[r].cpu().view(torch.int16), want_q[r].view(torch.int16))
        assert torch.equal(ok[r].cpu().view(torch.int16), want_k[r].view(torch.int16))
    # inverse direction: [b, s, n/p, d] -> [b, s/p, n, d]; must undo the forward one (round trip)
    so = world.sym(want_q[0].numel() * 2)
    for r in range(p):
        so[r].view(torch.bfloat16, want_q[r].numel()).copy_(want_q[r].flatten())
    back = [torch.zeros(b, s // p, heads, d, device="cuda", dtype=torch.bfloat16) for _ in range(p)]
    hp = heads // p

    def desc_inv(src, dst):
        return dict(src=src, dst=dst, batch=b, rows=s // p, row_elems=hp * d, src_bs=s * hp * d, src_rs=hp * d,
                    src_me_off=(s // p) * hp * d, dst_bs=(s // p) * heads * d, dst_rs=heads * d, dst_peer_off=hp * d)

    world.run(lambda r, c: c.all_to_all_rows(world.group, [desc_inv(so[r], back[r])], torch.bfloat16))
    want_back = ref.ulysses_all_to_all(want_q, 1, 2)
    for r in range(p):
        assert torch.equal(back[r].cpu().view(torch.int16), want_back[r].view(torch.int16))
        assert torch.equal(back[r].cpu().view(torch.int16), qs[r].view(torch.int16))


def test_p2p_send_wait_release(world, bg):
    if world.n < 2:
        pytest.skip()
    c0, c1 = world.comms[0], world.comms[1]
    nbytes = 1 << 20
    off1, recv = c1.alloc(nbytes)
    msgs = [torch.full((nbytes // 2,), float(i + 1), device="cuda", dtype=torch.bfloat16) for i in range(3)]
    got = []
    for i in range(3):  # same slot three times: the 2nd/3rd send must wait for the receiver's release
        with torch.cuda.stream(world.streams[0]):
            c0.p2p_send(1, off1, msgs[i], flag_id=3)
        with torch.cuda.stream(world.streams[1]):
            c1.p2p_wait(0, flag_id=3)
            got.append(recv.view(torch.bfloat16).clone())
            c1.p2p_release(0, flag_id=3)
    torch.cuda.synchronize()
    for i in range(3):
        assert torch.equal(got[i].cpu(), msgs[i].cpu())


def test_full_size_round_trip_property(bg, ref):
    """BASELINE config (2): one Llama-3-8B layer's flat parameter (218,112,000 elements, SDP=8).  all-gather(cast)
    of fp32 shards followed by reduce-scatter of the gathered bf16 copies returns bf16(shard) exactly
    (8 equal addends, divisions by 4 and 2 are exact): a size-independent check at full size."""
    n, P = 8, 218_112_000
    shard = ref.pad_to_multiple(P, 8 * n) // n
    w = World(bg, n, arena=(shard * n * 2 + (1 << 20)) * 1 + (8 << 20))
    try:
        bg.set_tunable("comm_ctas", 16)
        masters = [torch.randn(shard, device="cuda") for _ in range(n)]
        wbuf = w.sym(shard * n * 2)
        w.run(lambda r, c: c.all_gather_cast(w.group, masters[r], wbuf[r]))
        full0 = wbuf[0].view(torch.bfloat16, shard * n)
        for r in range(1, n):
            assert torch.equal(wbuf[r].view(torch.bfloat16, shard * n), full0)
        out = [torch.empty(shard, device="cuda") for _ in range(n)]
        pre, post = ref.fsdp_divide_factors(n)
        w.run(lambda r, c: c.reduce_scatter_acc(w.group, wbuf[r], torch.bfloat16, out[r], prescale=1 / pre, postscale=1 / post))
        for r in range(n):
            assert torch.equal(out[r], masters[r].to(torch.bfloat16).float())
    finally:
        bg.set_tunable("comm_ctas", 16)
        w.close()


@pytest.mark.parametrize("shard", [8, 4096 * 8 + 8])
def test_reduce_scatter_adamw_epilogue(world, ref, shard):
    """C2 with the AdamW epilogue == exact reduce-scatter followed by torch.optim.AdamW on the fp32 shard (3 steps)."""
    n = world.n
    g = torch.Generator(device="cpu").manual_seed(21 + shard)
    pre, post = ref.fsdp_divide_factors(n)
    params = [torch.randn(shard, generator=g) for _ in range(n)]
    refs = [torch.nn.Parameter(p.clone().double()) for p in params]
    opts = [torch.optim.AdamW([r], lr=1e-2, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.1) for r in refs]
    dev_p = [p.clone().cuda() for p in params]
    dev_m = [torch.zeros(shard, device="cuda") for _ in range(n)]
    dev_v = [torch.zeros(shard, device="cuda") for _ in range(n)]
    sym = world.sym(shard * n * 2)
    for step in range(1, 4):
        srcs = [torch.randn(shard * n, generator=g).to(torch.bfloat16) for _ in range(n)]
        for r in range(n):
            sym[r].view(torch.bfloat16, shard * n).copy_(srcs[r])
        world.run(lambda r, c: c.reduce_scatter_adamw(world.group, sym[r], torch.bfloat16, dev_p[r], dev_m[r], dev_v[r], shard,
                                                      1.0 / pre, 1.0 / post, 1e-2, 0.9, 0.95, 1e-8, 0.1, step))
        exact = ref.reduce_scatter_acc(srcs, None, order="exact", accumulate=False, out_dtype=torch.float64)
        for r in range(n):
            refs[r].grad = exact[r].double()
            opts[r].step()
    for r in range(n):
        torch.testing.assert_close(dev_p[r].cpu().double(), refs[r].detach(), rtol=2e-5, atol=2e-5)

"""Gradient clipping with the fused optimizer on one H100: the norm pass, the fp32 shard with partials and the clipped AdamW
reduce-scatter through the C ABI on p = 1, 2, 4, 8 virtual ranks (as in tests/test_gpu_collectives.py), then whole tiny-Llama runs
through the CUDA path against the torch optimizer clipped the same way.  Every case checks the device error flag."""
import os
import sys
import tempfile

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


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


class World:
    def __init__(self, bg, n, arena=256 << 20):
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


@pytest.fixture(scope="module", params=[1, 2, 4, 8])
def world(request, bg):
    w = World(bg, request.param)
    yield w
    w.close()


def _factors(n):
    from oracle import collectives_ref
    return collectives_ref.fsdp_divide_factors(n)


def _sources(world, shard, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    srcs = [(torch.randn(world.n * shard, generator=g) * 1e-2).to(dtype) for _ in range(world.n)]
    esz = torch.empty((), dtype=dtype).element_size()
    sym = world.sym(world.n * shard * esz)
    for r in range(world.n):
        sym[r].view(dtype, world.n * shard).copy_(srcs[r])
    return srcs, sym


def _exact(srcs, n, shard, r):
    pre, post = _factors(n)
    return sum(s[r * shard:(r + 1) * shard].double() / pre for s in srcs) / post


def _partials(bg, n):
    return [torch.full((4 * max(bg.get_tunable("comm_ctas"), bg.get_tunable("local_ctas")),), float("nan"), device="cuda")
            for _ in range(n)]


SKIP = [(0, 0), (64, 1024), (2048, 2056)]


@pytest.mark.parametrize("skip", [False, True], ids=["all", "skip"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_norm_pass_sum_of_squares(world, bg, dtype, skip):
    n, shard = world.n, 4096 * 8 + 8
    srcs, sym = _sources(world, shard, dtype, 3 + n)
    ranges = [r for r in SKIP if r[1] > r[0]] if skip else []
    pre, post = _factors(n)
    outs = []
    for _ in range(2):
        parts = _partials(bg, n)
        world.run(lambda r, c: c.reduce_scatter_sumsq(world.group, sym[r], dtype, shard, 1.0 / pre, 1.0 / post, parts[r], ranges))
        outs.append(parts)
    for r in range(n):
        want = _exact(srcs, n, shard, r)
        keep = torch.ones(shard, dtype=torch.bool)
        for lo, hi in ranges:
            keep[lo:hi] = False
        want = float(want[keep].pow(2).sum())
        got = float(outs[0][r].double().sum())
        assert abs(got - want) <= 1e-6 * want, (r, got, want)
        assert not torch.isnan(outs[0][r]).any()                      # the whole slot is written (the tail with zeros)
        assert torch.equal(outs[0][r].view(torch.int32), outs[1][r].view(torch.int32))     # deterministic


def test_fp32_shard_with_partials(world, bg):
    n, shard = world.n, 4096 * 8 + 8
    srcs, sym = _sources(world, shard, torch.bfloat16, 7 + n)
    pre, post = _factors(n)
    acc = [torch.zeros(shard, device="cuda") for _ in range(n)]
    with_parts = [torch.full((shard,), float("nan"), device="cuda") for _ in range(n)]
    parts_a, parts_b = _partials(bg, n), _partials(bg, n)
    world.run(lambda r, c: c.reduce_scatter_acc(world.group, sym[r], torch.bfloat16, acc[r], prescale=1.0 / pre, postscale=1.0 / post))
    world.run(lambda r, c: c.reduce_scatter_sumsq(world.group, sym[r], torch.bfloat16, shard, 1.0 / pre, 1.0 / post, parts_a[r],
                                                  SKIP[1:], dst=with_parts[r]))
    world.run(lambda r, c: c.reduce_scatter_sumsq(world.group, sym[r], torch.bfloat16, shard, 1.0 / pre, 1.0 / post, parts_b[r],
                                                  SKIP[1:]))
    for r in range(n):
        assert torch.equal(with_parts[r].view(torch.int32), acc[r].view(torch.int32))
        assert torch.equal(parts_a[r].view(torch.int32), parts_b[r].view(torch.int32))


def _ulps(got, want, floor=0.0):
    """|got - want| in fp32 ulps of max(|want|, floor): ``floor`` is the size of the terms an element is the difference of (an
    element near zero that is the difference of larger terms carries their rounding)."""
    scale = torch.clamp(want.abs(), min=floor) if torch.is_tensor(floor) or floor else want.abs()
    spacing = torch.nextafter(scale, torch.tensor(float("inf"), device=want.device)) - scale
    return float(((got - want).abs() / spacing).max())


def _f32_one_minus(x):
    return float(torch.tensor(1.0) - torch.tensor(x, dtype=torch.float32))


def test_clipped_adamw(world, bg):
    """coefficient 1: bit-identical to the unclipped AdamW reduce-scatter over 3 steps; 0.3: within 4 fp32 ulps per step of a torch
    restatement in the kernel's operation order, g = (sum prescale * x) * (postscale * coef) (the kernel contracts multiply-adds,
    the restatement rounds every operation).  The local clipped step (pooled units) likewise, after one step."""
    n, shard = world.n, 4096 * 8 + 8
    pre, post = _factors(n)
    g = torch.Generator().manual_seed(40 + n)
    params = [torch.randn(shard, generator=g).cuda() for _ in range(n)]
    hyper = (1e-2, 0.9, 0.95, 1e-8, 0.1)
    state = {k: ([p.clone() for p in params], [torch.zeros(shard, device="cuda") for _ in range(n)],
                 [torch.zeros(shard, device="cuda") for _ in range(n)]) for k in ("plain", "one", "clip", "ref")}
    one, coef = torch.ones((), device="cuda"), torch.full((), 0.3, device="cuda")
    m_scale = [torch.zeros(shard, device="cuda") for _ in range(n)]     # the largest term each exp_avg element was formed from
    sym = world.sym(shard * n * 2)
    for step in range(1, 4):
        srcs = [(torch.randn(shard * n, generator=g) * 1e-2).to(torch.bfloat16) for _ in range(n)]
        for r in range(n):
            sym[r].view(torch.bfloat16, shard * n).copy_(srcs[r])
        red = [torch.zeros(shard, device="cuda") for _ in range(n)]
        world.run(lambda r, c: c.reduce_scatter_acc(world.group, sym[r], torch.bfloat16, red[r], prescale=1.0 / pre, postscale=1.0 / post))
        p, m, v = state["plain"]
        world.run(lambda r, c: c.reduce_scatter_adamw(world.group, sym[r], torch.bfloat16, p[r], m[r], v[r], shard, 1.0 / pre, 1.0 / post,
                                                      *hyper, step))
        for key, k in (("one", one), ("clip", coef)):
            p, m, v = state[key]
            world.run(lambda r, c: c.reduce_scatter_adamw_clipped(world.group, sym[r], torch.bfloat16, p[r], m[r], v[r], shard, 1.0 / pre,
                                                                  1.0 / post, *hyper, step, k))
        lr, b1, b2, eps, wd = hyper
        c1, c2 = _f32_one_minus(b1), _f32_one_minus(b2)     # the kernel forms 1 - beta in fp32
        p, m, v = state["ref"]
        for r in range(n):      # postscale is a power of two: red * coef rounds as acc * (postscale * coef)
            gr = red[r] * coef
            m_scale[r] = torch.maximum(m_scale[r], torch.maximum(b1 * m[r].abs(), c1 * gr.abs()))
            m[r].copy_(b1 * m[r] + c1 * gr)
            v[r].copy_(b2 * v[r] + c2 * gr * gr)
            denom = v[r].sqrt() / torch.tensor((1 - b2 ** step) ** 0.5, dtype=torch.float32, device="cuda") + eps
            p[r].copy_(p[r] * (1 - lr * wd) - torch.tensor(lr / (1 - b1 ** step), dtype=torch.float32, device="cuda") * m[r] / denom)
    for r in range(n):
        for i in range(3):
            assert torch.equal(state["one"][i][r].view(torch.int32), state["plain"][i][r].view(torch.int32))
        # param: the difference of p * decay and an update of size ~lr; exp_avg: of b1 * m and (1 - b1) * g; exp_avg_sq: no cancellation
        for i, floor in ((0, hyper[0]), (1, m_scale[r]), (2, 0.0)):
            assert _ulps(state["clip"][i][r], state["ref"][i][r], floor) <= 4 * 3, (i, _ulps(state["clip"][i][r], state["ref"][i][r], floor))
    # the local step of pooled units: the same rule on an fp32 gradient
    p, m, v = [t.clone() for t in params[:1]], [torch.zeros(shard, device="cuda")], [torch.zeros(shard, device="cuda")]
    p2, m2, v2 = [t.clone() for t in params[:1]], [torch.zeros(shard, device="cuda")], [torch.zeros(shard, device="cuda")]
    grad = torch.randn(shard, generator=g).cuda() * 1e-2
    bg.adamw_clipped(p[0], m[0], v[0], grad, *hyper, 1, coef)
    torch.cuda.synchronize()
    gr = grad * coef
    m2[0] = _f32_one_minus(hyper[1]) * gr
    v2[0] = _f32_one_minus(hyper[2]) * gr * gr
    denom = v2[0].sqrt() / torch.tensor((1 - hyper[2]) ** 0.5, device="cuda") + hyper[3]
    p2[0] = p2[0] * (1 - hyper[0] * hyper[4]) - torch.tensor(hyper[0] / (1 - hyper[1]), device="cuda") * m2[0] / denom
    assert _ulps(p[0], p2[0], hyper[0]) <= 4 and _ulps(m[0], m2[0]) <= 4 and _ulps(v[0], v2[0]) <= 4


# ---- whole model through the CUDA path ----------------------------------------------------------------------------------------
_PORT = [32400]


def _launch(world, over, arm):
    from _launch import launch_ranks
    _PORT[0] += 1
    tmp = tempfile.mkdtemp(prefix="hgb_gpu_clip_")
    rep = launch_ranks("_clip_worker", world, dict(over, _arm=arm, _dump=os.path.join(tmp, "m")), _PORT[0] + os.getpid() % 500,
                       timeout=900, backend="cuda")
    ms = []
    for r in range(world):
        path = os.path.join(tmp, "m.rank%d" % r)
        ms.append(torch.load(path, weights_only=True))
        os.remove(path)
    os.rmdir(tmp)
    rep["masters"] = torch.cat([m[k].reshape(-1) for m in ms for k in sorted(m)])
    return rep


def _rel(a, b):
    return float((a - b).norm() / b.norm())


MODEL_CASES = {"world1": (1, {}), "dp2_zero3": (2, dict(sdp=1, embed_sdp=1)),
               "tp2_megatron_sp": (2, dict(global_tp_deg=2, vocab_tp=2, sequence_parallel=True))}


@pytest.mark.parametrize("name", sorted(MODEL_CASES))
def test_model_fused_clip_against_torch_clip(name):
    """Whole-model runs are not bit-reproducible across processes (two runs of the same arm end ~1e-6 apart in the masters; the
    kernels of this feature are, see above), and the fused and torch AdamW round differently, so the clipped pair is held to the
    drift of the unclipped fused-vs-torch pair, which measures its norms with clip_grad_norm(model, inf): the step-0 norms (same
    weights) to 1e-5; the masters after 3 steps, of the pair and of a repeat, at most 2x the unclipped pair's gap.  The norms of
    later steps are single samples of diverging trajectories (measured at step 2: a repeat of the same arm up to 1.1e-4 apart, the
    unclipped pair 4e-5 to 2.3e-4): held to 1e-3, which a norm that miscounts a unit or a coefficient applied twice exceeds."""
    world, over = MODEL_CASES[name]
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    fc, tc = _launch(world, over, "fused_clip"), _launch(world, over, "torch_clip")
    fu, tu = _launch(world, over, "fused_norm"), _launch(world, over, "torch_norm")
    again = _launch(world, over, "fused_clip")
    rel_n = lambda a, b: [abs(x - y) / y for x, y in zip(a, b)]  # noqa: E731
    gap_clip, gap_plain, gap_repeat = _rel(fc["masters"], tc["masters"]), _rel(fu["masters"], tu["masters"]), _rel(fc["masters"], again["masters"])
    print("norms clipped fused %s torch %s | unclipped fused %s torch %s | repeat %s" % (fc["norms"], tc["norms"], fu["norms"], tu["norms"],
                                                                                        again["norms"]))
    print("masters rel-L2: clipped pair %.3g, unclipped pair %.3g, repeat of the clipped fused run %.3g (bit-identical: %s)"
          % (gap_clip, gap_plain, gap_repeat, torch.equal(fc["masters"].view(torch.int32), again["masters"].view(torch.int32))))
    assert tc["norms"][0] > 0.05                         # clipping bites
    d_clip, d_plain = rel_n(fc["norms"], tc["norms"]), rel_n(fu["norms"], tu["norms"])
    assert d_clip[0] <= 1e-5 and d_plain[0] <= 1e-5 and rel_n(again["norms"], fc["norms"])[0] <= 1e-5, (d_clip, d_plain)
    assert max(d_clip[1:]) <= 1e-3, (d_clip, d_plain)
    assert gap_clip <= 2 * gap_plain and gap_repeat <= 2 * gap_plain, (gap_clip, gap_plain, gap_repeat)
    calls = fc["fused_calls"]
    assert calls.get("rs_sumsq", 0) > 0 and calls.get("rs_adamw_clipped", 0) + calls.get("adamw_clipped", 0) > 0, calls
    assert all(needed for _, needed in fc["fp32_grad_units"]), fc["fp32_grad_units"]

"""The peer-memory collectives of csrc/bg_coll.cu against exact float64 references, on virtual ranks.

One H100 is enough: ``BgComm.local_world(n)`` creates n virtual ranks (n contexts, n arenas) on the device and every rank's
kernel runs on its own stream, so the real cross-rank protocol (device barriers, peer loads and stores through the peer-pointer
table) is what executes.

Every reference is computed in float64 from the bf16 / fp32 values the kernel reads:
  - integer data: entries are integers in [-200, 200] times 2^-3, so every fp32 partial sum is exact and the output must be the
    float64 result rounded once to the output type, bit for bit.  Some sums are odd and lie in (256, 512) -- halfway between two
    bf16 neighbours -- and must round to even.  Only with power-of-two scales.
  - real data: the output must be within a bound derived, next to its assertion, from the fp32 operations the kernel evaluates
    (``_fp_check``: half a bf16 ulp plus eps for bf16 outputs, eps plus half an fp32 ulp for fp32 outputs).
  - MAX, all-gather and all-to-all need no bound: they are exact.
Stores are guarded.  Local destinations start as NaN between 4 KiB guards.  Symmetric buffers sit between guard buffers allocated
just before and after them in the arena, and the bytes of a buffer outside the region a call may write hold a sentinel.  Every
guard and every source must come back unchanged, with one documented exception: after a two-shot all-reduce, slice `me` of each
member's source holds that member's reduced slice.  Every call runs twice on the same buffers, the second time onto the first
run's output.  The edge shapes, the real-data reduce-scatter and all-reduce cases and the concurrent-group cases run under
comm_ctas 1, 3 and 16, which must give bit-identical results.  On real data that means no element's summation order depends on
the grid (on integer data every order gives the same bits, so there it only checks coverage and stores).
"""
import contextlib
import os
import sys

import pytest
import torch

# before any CUDA context exists in this process: a kernel waiting for a peer must never falsely order another stream behind it
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from _fp_check import BF, _bits, assert_rounded, assert_within, gamma  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

F32 = torch.float32
GUARD = 4096                 # bytes of every guard region
NAN_BITS = {BF: 0x7FC0, F32: 0x7FC00000}
INT_UNIT = 2.0 ** -3         # integer data are multiples of this
TIE_SUMS = (257, -259, 383, -385)   # odd sums in (256, 512): exact in fp32, halfway between two bf16 neighbours

# Launch geometry of bg_coll.cu, mirrored here to put sizes on the edges of its loops.  kThreads = 128 threads per CTA.  Per loop
# iteration a thread handles V 16-B vectors: kUnroll = 4 in the all-gather push; RsPlan<PMAX, kEpiF32 / kEpiBf16>::V =
# kInFlight / PMAX in the reduce-scatter pull and the two-shot all-reduce (kInFlight = 8; PMAX = 2, 4 or 8, the smallest that
# is >= n); 1 in the one-shot all-reduce; kInFlight = 8 in the all-to-all.  grid = comm_grid(vectors / V + 1) =
# min(ceil((vectors / V + 1) / 128), comm_ctas), with local_ctas in place of comm_ctas for a group of one.
THREADS, K_UNROLL, K_IN_FLIGHT = 128, 4, 8
CTAS = (1, 3, 16)            # 8 ranks x 2 concurrent collectives x 16 slim CTAs stay co-resident on one device


def _pmax(n):
    return 2 if n <= 2 else 4 if n <= 4 else 8


def v_rs(n):
    return K_IN_FLIGHT // _pmax(n)


def v_ar(n, twoshot):
    return K_IN_FLIGHT // _pmax(n) if twoshot else 1


def comm_grid(vectors, v, cap):
    return max(1, min(cap, -(-(vectors // v + 1) // THREADS)))


def edge_counts(n, v, cap=16):
    """Loop vector counts at the edges of a launch capped at `cap` CTAs: one vector, fewer vectors than members, one whole
    iteration of the capped grid (cap * 128 * V) and one vector fewer and more, and 2.5 iterations plus 3 vectors (the grid is
    capped and the loop wraps a non-whole number of times)."""
    full = cap * THREADS * v
    assert comm_grid(full - 1, v, cap) == cap and comm_grid(full, v, cap) == cap
    return sorted({1, max(1, n - 1), full - 1, full, full + 1, 5 * full // 2 + 3})


def _esz(dt):
    return 2 if dt == BF else 4


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
    with tunables(bg, timeout_ms=20000, comm_ctas=16, oneshot_bytes=512 * 1024):
        yield bg


@pytest.fixture(scope="module")
def ref():
    from oracle import collectives_ref
    return collectives_ref


class World:
    def __init__(self, bg, n, arena=512 << 20):
        from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
        self.bg, self.n, self.CommGroup = bg, n, CommGroup
        self.comms = bg.BgComm.local_world(n, device=0, arena_bytes=arena)
        self.group = CommGroup(list(range(n)))
        self.streams = [[torch.cuda.Stream() for _ in range(n)] for _ in range(2)]   # two streams per rank
        self.gen = torch.Generator(device="cuda").manual_seed(1000 + n)

    def sym(self, nbytes, group=None):
        group = self.group if group is None else group
        bufs = [self.comms[r].sym_alloc(group, nbytes) for r in group.ranks]
        for c in self.comms:
            c.exchange()
        return bufs

    def run(self, fn):
        torch.cuda.synchronize()
        for r, c in enumerate(self.comms):
            with torch.cuda.stream(self.streams[0][r]):
                fn(r, c)
        torch.cuda.synchronize()
        for c in self.comms:
            assert c.error_flag() == 0

    def close(self):
        torch.cuda.synchronize()
        for c in self.comms:
            c.close()


@pytest.fixture(scope="module", params=[1, 2, 3, 4, 6, 8])
def world(request, bg):
    w = World(bg, request.param)
    yield w
    w.close()


# ---- data and guarded buffers --------------------------------------------------------------------------------------------------
def sentinel(nbytes, gen):
    return torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda", generator=gen)


def int_units(numel, gen):
    return torch.randint(-200, 201, (numel,), device="cuda", generator=gen, dtype=torch.int64)


def from_units(u, dt):
    return (u.double() * INT_UNIT).to(dt)       # exact: |u| <= 256


def force_ties(units, cols):
    """units: one int tensor per member.  At element cols[j] the members' values sum to TIE_SUMS[j]."""
    n = len(units)
    if n < 2:
        return                     # a single member's value is its own, bf16-exact, sum
    for col, s in zip(cols, TIE_SUMS):
        c = s // n
        for m in range(n):
            units[m][col] = s - (n - 1) * c if m == 0 else c


def real_data(numel, dt, gen):
    return (torch.randn(numel, device="cuda", generator=gen) * 3).to(dt)


def n_ties(exact64):
    """elements of an exactly-fp32 float64 tensor that lie halfway between two bf16 neighbours"""
    b = exact64.float().view(torch.int32)
    return int(((b & 0xFFFF) == 0x8000).sum())


def exact_to(v64, dt):
    """round a float64 tensor that holds exact fp32 values once to dt"""
    f = v64.float()
    assert torch.equal(f.double(), v64), "reference is not exact in fp32"
    return f.to(dt)


class Guarded:
    """A symmetric buffer between two guard buffers allocated just before and after it in every member's arena.  All three hold
    a sentinel; `write` puts data into a region, and `check` asserts that every byte outside the allowed regions is as left."""

    def __init__(self, w, group, nbytes):
        self.lo, self.buf, self.hi = w.sym(GUARD, group), w.sym(nbytes, group), w.sym(GUARD, group)
        for parts in (self.lo, self.buf, self.hi):
            for b in parts:
                b.u8.copy_(sentinel(b.u8.numel(), w.gen))
        self.snap()

    def snap(self):
        self.saved = [[b.u8.clone() for b in parts] for parts in (self.lo, self.buf, self.hi)]

    def region(self, i, off, numel, dt):
        return self.buf[i].u8[off: off + numel * _esz(dt)].view(dt)

    def check(self, i, allow=(), what=""):
        lo, buf, hi = self.lo[i].u8, self.buf[i].u8, self.hi[i].u8
        assert torch.equal(lo, self.saved[0][i]), f"{what}: guard before the symmetric buffer overwritten (member {i})"
        assert torch.equal(hi, self.saved[2][i]), f"{what}: guard after the symmetric buffer overwritten (member {i})"
        keep = torch.ones(buf.numel(), dtype=torch.bool, device="cuda")
        for a, b in allow:
            keep[a:b] = False
        bad = keep & (buf != self.saved[1][i])
        assert not bad.any(), f"{what}: member {i}: {int(bad.sum())} bytes changed outside the written region, first at " \
                              f"{int(bad.nonzero()[0])}"


class LocalOut:
    """A local destination of `numel` elements inside a larger tensor, with 4 KiB sentinel guards on both sides."""

    def __init__(self, numel, dt, gen):
        self.dt, nbytes = dt, numel * _esz(dt)
        self.u8 = sentinel(2 * GUARD + nbytes, gen)
        self.t = self.u8[GUARD: GUARD + nbytes].view(dt)
        self.saved = self.u8.clone()

    def nan(self):
        _bits(self.t).fill_(NAN_BITS[self.dt])

    def check(self, what=""):
        assert torch.equal(self.u8[:GUARD], self.saved[:GUARD]), f"{what}: guard before the destination overwritten"
        end = GUARD + self.t.numel() * _esz(self.dt)
        assert torch.equal(self.u8[end:], self.saved[end:]), f"{what}: guard after the destination overwritten"


def expect_bits(got, want, what):
    g, w = _bits(got), _bits(want)
    bad = g != w
    assert not bad.any(), f"{what}: {int(bad.sum())} / {bad.numel()} elements differ, first at {int(bad.nonzero()[0])}: got " \
                          f"{got.reshape(-1)[bad.nonzero()[0]].item()} want {want.reshape(-1)[bad.nonzero()[0]].item()}"


# ---- one collective call per case: prepare (reference from the inputs), launch (one member), check ------------------------------
class Case:
    lane = None

    def __init__(self, w, ranks, sidx=0):
        self.w, self.ranks = w, list(ranks)
        self.group = w.CommGroup(self.ranks)
        self.n = len(self.ranks)
        self.index = {r: i for i, r in enumerate(self.ranks)}    # rank -> member index (`me`), not the rank in a strided group
        self.sidx, self.run_i = sidx, 0

    def stream(self, r):
        return self.w.streams[self.sidx][r]

    def __repr__(self):
        return f"{type(self).__name__}{self.desc} on {self.ranks}"


class AllGather(Case):
    lane = 0

    def __init__(self, w, ranks, shard, sd, dd, data=None, off=0, **kw):
        super().__init__(w, ranks, **kw)
        self.shard, self.sd, self.dd, self.off = shard, sd, dd, off
        self.desc = (shard, str(sd)[6:], str(dd)[6:], off)
        self.src = data if data is not None else [real_data(shard, sd, w.gen) for _ in range(self.n)]
        self.src_saved = [s.clone() for s in self.src]
        self.nbytes = self.n * shard * _esz(dd)
        self.dst = Guarded(w, self.group, off + self.nbytes)
        self.want = torch.cat([s.cpu().to(dd) for s in self.src]).cuda()     # Tensor.to(): round to nearest even

    def reset(self):
        for i in range(self.n):
            _bits(self.dst.region(i, self.off, self.n * self.shard, self.dd)).fill_(NAN_BITS[self.dd])

    def prepare(self):
        pass

    def launch(self, r, c):
        i = self.index[r]
        c.all_gather_cast(self.group, self.src[i], self.dst.buf[i], shard_elems=self.shard, lane=self.lane, stream=self.stream(r),
                          dst_dtype=self.dd, dst_byte_offset=self.off)

    def check(self, what):
        for i in range(self.n):
            got = self.dst.region(i, self.off, self.n * self.shard, self.dd)
            if self.sd != self.dd:            # a converted NaN keeps its NaN-ness, not its payload
                nan = self.want.isnan()
                assert torch.equal(got.isnan(), nan), f"{what}: NaN positions differ on member {i}"
                expect_bits(got[~nan], self.want[~nan], f"{what} member {i}")
            else:
                expect_bits(got, self.want, f"{what} member {i}")
            self.dst.check(i, [(self.off, self.off + self.nbytes)], what)
            assert torch.equal(_bits(self.src[i]), _bits(self.src_saved[i])), f"{what}: source of member {i} changed"

    def bits(self):
        return torch.cat([_bits(self.dst.region(i, self.off, self.n * self.shard, self.dd)) for i in range(self.n)])


class ReduceScatter(Case):
    lane = 1

    def __init__(self, w, ranks, shard, sd, dd, accumulate, pre, post, integer, off=0, **kw):
        super().__init__(w, ranks, **kw)
        self.shard, self.sd, self.dd, self.acc, self.pre, self.post, self.integer, self.off = \
            shard, sd, dd, accumulate, pre, post, integer, off
        self.desc = (shard, str(sd)[6:], str(dd)[6:], "acc" if accumulate else "", pre, post, "int" if integer else "real", off)
        n, total = self.n, self.n * shard
        if integer:
            units = [int_units(total, w.gen) for _ in range(n)]
            for i in range(n):                                     # ties in every member's shard
                force_ties(units, [i * shard + j for j in range(min(4, shard))])
            self.data = [from_units(u, sd) for u in units]
        else:
            self.data = [real_data(total, sd, w.gen) for _ in range(n)]
        self.src = Guarded(w, self.group, off + total * _esz(sd))
        for i in range(n):
            self.src.region(i, off, total, sd).copy_(self.data[i])
        self.src.snap()
        self.dst = [LocalOut(shard, dd, w.gen) for _ in range(n)]
        self.old = []                      # what an accumulating call first adds to
        for _ in range(n):
            if integer:
                u = int_units(shard, w.gen)
                u[:4] = 0                  # keeps the forced ties
                self.old.append(from_units(u, dd))
            else:
                self.old.append(real_data(shard, dd, w.gen))

    def reset(self):
        for d, old in zip(self.dst, self.old):
            if self.acc:
                d.t.copy_(old)
            else:
                d.nan()
        self.run_i = 0

    def prepare(self):
        # what the kernel evaluates, in fp32: acc = fmaf(x_m, prescale, acc) over the n members, acc * postscale, [+ old], then the
        # cast.  Against the exact (float64) prescale and postscale: n roundings of the fmaf chain, one each for prescale and
        # postscale as fp32 values, one for the product and one for the add of old -- gamma(n + 4 [+ 1]) times the sum of the
        # |terms| (the final rounding to the output type is the _fp_check half ulp).
        self.want, self.eps = [], []
        for i in range(self.n):
            t = torch.stack([d[i * self.shard:(i + 1) * self.shard].double() for d in self.data]) * self.pre
            v = t.sum(0) * self.post
            old = self.dst[i].t.double() if self.acc else torch.zeros_like(v)
            self.want.append(v + old)
            self.eps.append(gamma(self.n + 4 + (1 if self.acc else 0)) * (t.abs().sum(0) * abs(self.post) + old.abs()))

    def launch(self, r, c):
        i = self.index[r]
        c.reduce_scatter_acc(self.group, self.src.buf[i], self.sd, self.dst[i].t, shard_elems=self.shard, prescale=self.pre,
                             postscale=self.post, accumulate=bool(self.acc), lane=self.lane, stream=self.stream(r),
                             src_byte_offset=self.off)

    def check(self, what):
        ties = 0
        for i in range(self.n):
            got, want = self.dst[i].t, self.want[i]
            if self.integer:
                expect_bits(got, exact_to(want, self.dd), f"{what} member {i}")
                ties += n_ties(want)
            elif self.dd == BF:
                assert_rounded(got, want, self.eps[i], f"{what} member {i}")
            else:
                assert_within(got, want, self.eps[i], f"{what} member {i}")
            self.dst[i].check(what)
            self.src.check(i, (), what)
        if self.integer and self.dd == BF and self.n > 1 and self.run_i == 0:
            assert ties > 0, f"{what}: no bf16 ties in the exact results"
        self.run_i += 1

    def bits(self):
        return torch.cat([_bits(d.t) for d in self.dst])


class AllReduce(Case):
    lane = 2

    def __init__(self, w, ranks, elems, dt, op, scale, integer, off=0, **kw):
        super().__init__(w, ranks, **kw)
        self.elems, self.dt, self.op, self.scale, self.integer, self.off = elems, dt, op, scale, integer, off
        self.desc = (elems, str(dt)[6:], "max" if op else "sum", scale, "int" if integer else "real", off)
        if integer:
            units = [int_units(elems, w.gen) for _ in range(self.n)]
            force_ties(units, range(min(4, elems)))
            self.data = [from_units(u, dt) for u in units]
        else:
            self.data = [real_data(elems, dt, w.gen) for _ in range(self.n)]
        self.src = Guarded(w, self.group, off + elems * _esz(dt))
        self.dst = [LocalOut(elems, dt, w.gen) for _ in range(self.n)]
        self.twoshot = None

    def reset(self):
        for d in self.dst:
            d.nan()
        self.run_i = 0
        n, per = self.n, 16 // _esz(self.dt)
        # the dispatch of bg_all_reduce (no multicast-bound buffers here)
        self.twoshot = n > 1 and self.elems * _esz(self.dt) > self.w.bg.get_tunable("oneshot_bytes") and (self.elems // per) % n == 0

    def prepare(self):
        # sources are rewritten before every run: the two-shot kernel leaves its reduced slice in the member's own source
        for i in range(self.n):
            self.src.region(i, self.off, self.elems, self.dt).copy_(self.data[i])
        self.src.snap()
        x = torch.stack([d.double() for d in self.data])
        s32 = float(torch.tensor(self.scale, dtype=F32))
        if self.op == self.w.bg.MAX:   # exact: the fp32 product of the max and fp32(scale), rounded once more to a bf16 output
            self.want = (x.max(0).values * s32).float().to(self.dt)
        else:
            # fp32: n - 1 additions in member order, then * fp32(scale) -- n - 1 roundings, one for the fp32 scale, one for the
            # product: gamma(n + 1) * sum |x| * |scale| (the final rounding to the output type is the _fp_check half ulp)
            self.want = x.sum(0) * self.scale
            self.eps = gamma(self.n + 1) * x.abs().sum(0) * abs(self.scale)

    def launch(self, r, c):
        i = self.index[r]
        c.all_reduce(self.group, self.src.buf[i], self.dst[i].t, elems=self.elems, op=self.op, scale=self.scale, lane=self.lane,
                     stream=self.stream(r), src_byte_offset=self.off)

    def check(self, what):
        what = f"{what} ({'two' if self.twoshot else 'one'}-shot)"
        got0 = self.dst[0].t
        if self.op == self.w.bg.MAX:
            expect_bits(got0, self.want, what)
        elif self.integer:
            expect_bits(got0, exact_to(self.want, self.dt), what)
            if self.dt == BF and self.n > 1 and self.run_i == 0:
                assert n_ties(self.want) > 0, f"{what}: no bf16 ties in the exact results"
        elif self.dt == BF:
            assert_rounded(got0, self.want, self.eps, what)
        else:
            assert_within(got0, self.want, self.eps, what)
        esz = _esz(self.dt)
        slice_b = self.elems * esz // self.n
        for i in range(self.n):
            expect_bits(self.dst[i].t, got0, f"{what}: replica {i} vs replica 0")
            self.dst[i].check(what)
            if self.twoshot:    # the documented write-back: slice i of member i's source holds the reduced slice
                lo = self.off + i * slice_b
                expect_bits(self.src.buf[i].u8[lo: lo + slice_b].view(self.dt), got0[i * slice_b // esz:(i + 1) * slice_b // esz],
                            f"{what}: two-shot write-back of member {i}")
                self.src.check(i, [(lo, lo + slice_b)], what)
            else:
                self.src.check(i, (), what)
        self.run_i += 1

    def bits(self):
        return torch.cat([_bits(d.t) for d in self.dst])


def gather_first_dim(chunk, p):
    """the descriptor of CudaBackend.all_gather_first_dim: rows = 1, zero strides"""
    return dict(batch=1, rows=1, row_elems=chunk, src_bs=0, src_rs=0, src_me_off=0, dst_bs=0, dst_rs=0, dst_peer_off=chunk,
                src_numel=chunk, dst_numel=p * chunk)


def ulysses_fwd(b, s_in, heads, d, p):
    """[b, s/p, heads, d] -> [b, s, heads/p, d] (CudaBackend.ulysses_all_to_all, to_heads)"""
    hp = heads // p
    return dict(batch=b, rows=s_in, row_elems=hp * d, src_bs=s_in * heads * d, src_rs=heads * d, src_me_off=hp * d,
                dst_bs=s_in * p * hp * d, dst_rs=hp * d, dst_peer_off=s_in * hp * d, src_numel=b * s_in * heads * d,
                dst_numel=b * s_in * p * hp * d)


def ulysses_inv(b, s_in, n_in, d, p):
    """[b, s, heads/p, d] -> [b, s/p, heads, d] (the inverse)"""
    sl = s_in // p
    return dict(batch=b, rows=sl, row_elems=n_in * d, src_bs=s_in * n_in * d, src_rs=n_in * d, src_me_off=sl * n_in * d,
                dst_bs=sl * n_in * p * d, dst_rs=n_in * p * d, dst_peer_off=n_in * d, src_numel=b * s_in * n_in * d,
                dst_numel=b * sl * n_in * p * d)


_A2A_KEYS = ("batch", "rows", "row_elems", "src_bs", "src_rs", "src_me_off", "dst_bs", "dst_rs", "dst_peer_off")


class AllToAll(Case):
    lane = 2

    def __init__(self, w, ranks, dt, specs, off=0, **kw):
        super().__init__(w, ranks, **kw)
        self.dt, self.specs, self.off = dt, specs, off
        self.desc = (str(dt)[6:], [(s["batch"], s["rows"], s["row_elems"]) for s in specs], off)
        self.data = [[real_data(s["src_numel"], dt, w.gen) for _ in range(self.n)] for s in specs]
        self.src = [Guarded(w, self.group, off + s["src_numel"] * _esz(dt)) for s in specs]
        for t, s in enumerate(specs):
            for i in range(self.n):
                self.src[t].region(i, off, s["src_numel"], dt).copy_(self.data[t][i])
            self.src[t].snap()
        self.dst = [[LocalOut(s["dst_numel"], dt, w.gen) for _ in range(self.n)] for s in specs]

    def reset(self):
        for outs in self.dst:
            for d in outs:
                d.nan()

    def prepare(self):
        # the header's definition: dst[b*dst_bs + r*dst_rs + q*dst_peer_off + c] = src(peer q)[b*src_bs + r*src_rs + me*src_me_off + c]
        self.want = []
        for t, s in enumerate(self.specs):
            b = torch.arange(s["batch"], device="cuda")[:, None, None]
            r = torch.arange(s["rows"], device="cuda")[None, :, None]
            c = torch.arange(s["row_elems"], device="cuda")[None, None, :]
            outs = []
            for me in range(self.n):
                want = self.dst[t][me].t.clone()
                for q in range(self.n):
                    di = (b * s["dst_bs"] + r * s["dst_rs"] + q * s["dst_peer_off"] + c).reshape(-1)
                    si = (b * s["src_bs"] + r * s["src_rs"] + me * s["src_me_off"] + c).reshape(-1)
                    want[di] = self.data[t][q][si]
                outs.append(want)
            self.want.append(outs)

    def launch(self, r, c):
        i = self.index[r]
        descs = [dict({k: s[k] for k in _A2A_KEYS}, src=self.src[t].buf[i], src_byte_offset=self.off, dst=self.dst[t][i].t)
                 for t, s in enumerate(self.specs)]
        c.all_to_all_rows(self.group, descs, self.dt, lane=self.lane, stream=self.stream(r))

    def check(self, what):
        for t in range(len(self.specs)):
            for i in range(self.n):
                expect_bits(self.dst[t][i].t, self.want[t][i], f"{what} tensor {t} member {i}")
                self.dst[t][i].check(what)
                self.src[t].check(i, (), what)

    def bits(self):
        return torch.cat([_bits(d.t) for outs in self.dst for d in outs])


def drive(w, cases, ctas=CTAS, runs=2, **tun):
    """Run the cases together (every rank launches its part of each, in order) `runs` times per grid size, checking after each
    run; the results must be bit-identical across grid sizes."""
    bg, first = w.bg, None
    for cap in ctas:
        with tunables(bg, comm_ctas=cap, local_ctas=cap, **tun):
            for case in cases:
                case.reset()
            for run in range(runs):
                for case in cases:
                    case.prepare()
                w.run(lambda r, c: [case.launch(r, c) for case in cases if r in case.index])
                for case in cases:
                    case.check(f"{case} ctas={cap} run {run}")
            bits = [case.bits() for case in cases]
        if first is None:
            first = bits
        else:
            for case, a, b in zip(cases, first, bits):
                assert torch.equal(a, b), f"{case}: comm_ctas={cap} changed the result bits"


def group_scales(n):
    """the prescale and postscale FSDP uses for a group of n (1 / predivide, 1 / postdivide)"""
    from oracle import collectives_ref
    pre, post = collectives_ref.fsdp_divide_factors(n)
    return 1.0 / pre, 1.0 / post


AG_PAIRS = [(F32, BF), (BF, BF), (F32, F32)]
RS_CFGS = [(BF, F32), (BF, BF), (F32, F32)]
def _ids(v):
    return {BF: "bf16", F32: "f32"}.get(v, str(v)) if isinstance(v, torch.dtype) else str(v)


# ---- tests -----------------------------------------------------------------------------------------------------------------------
def test_barrier_and_repeat(world):
    for _ in range(5):
        world.run(lambda r, c: c.barrier(world.group))


@pytest.mark.parametrize("shard", [8, 1000 * 8, 1 << 20])
@pytest.mark.parametrize("src_dtype", [torch.float32, torch.bfloat16])
def test_all_gather_cast_bit_exact(world, shard, src_dtype):
    drive(world, [AllGather(world, range(world.n), shard, src_dtype, BF)], ctas=(16,))


@pytest.mark.parametrize("sd,dd", AG_PAIRS, ids=_ids)
def test_all_gather_cast_edges(world, sd, dd):
    per = 4 if dd == F32 else 8
    drive(world, [AllGather(world, range(world.n), v * per, sd, dd) for v in edge_counts(world.n, K_UNROLL)])


@pytest.mark.parametrize("sd,dd", AG_PAIRS, ids=_ids)
def test_all_gather_cast_special_values(world, sd, dd):
    """±0, ±inf, NaN (one whose upper half alone would read as inf), fp32 subnormals, values that round to the bf16 maximum or
    overflow to inf, and exact ties on even and odd bf16 mantissas: the gathered shard is Tensor.to(bf16)."""
    specials = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001, 0xFFC12345,
                0x00000001, 0x80000001, 0x00008000, 0x00018000, 0x007FFFFF, 0x00400000, 0x807F8000,
                0x7F7F0000, 0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF, 0xFF7F8000, 0x7F7E8000,
                0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000, 0x3F80FFFF, 0x3F817FFF, 0x40490FDB, 0x0080C000]
    bits = torch.tensor([v - (1 << 32) if v >= 1 << 31 else v for v in specials], dtype=torch.int32)
    shard = 64
    srcs = []
    for m in range(world.n):
        f = torch.randn(shard, generator=torch.Generator().manual_seed(m)) * 3
        f[:len(specials)] = bits.view(F32)
        f = f.roll(3 * m)                                     # a different layout on every member
        srcs.append((f if sd == F32 else f.to(BF)).cuda())
    case = AllGather(world, range(world.n), shard, sd, dd, data=srcs)
    drive(world, [case], ctas=(16,))


@pytest.mark.parametrize("shard", [8, 1000 * 8, 1 << 19])
@pytest.mark.parametrize("accumulate", [False, True])
def test_reduce_scatter_acc(world, shard, accumulate):
    pre, post = group_scales(world.n)
    drive(world, [ReduceScatter(world, range(world.n), shard, BF, F32, accumulate, pre, post, integer=False)], ctas=(16,))


def test_reduce_scatter_fp32_and_bf16_out(world):
    drive(world, [ReduceScatter(world, range(world.n), 4096, F32, F32, False, 0.5, 0.25, integer=False),
                  ReduceScatter(world, range(world.n), 4096, BF, BF, False, 1.0, 1.0, integer=False)], ctas=(16,))


@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("sd,dd", RS_CFGS, ids=_ids)
def test_reduce_scatter_edges_integer_exact(world, sd, dd, accumulate):
    per = 8 if sd == BF else 4
    drive(world, [ReduceScatter(world, range(world.n), v * per, sd, dd, accumulate, 0.5, 0.25, integer=True)
                  for v in edge_counts(world.n, v_rs(world.n))])


@pytest.mark.parametrize("scales", ["group", "1/3,0.7"])
@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("sd,dd", RS_CFGS, ids=_ids)
def test_reduce_scatter_real(world, sd, dd, accumulate, scales):
    """The group's own FSDP pre/post scales (1/2 and 1/1.5 at n = 3; 1/4 and 1/1.5 at n = 6) and a pair of non-powers of two.
    Real data under every grid size: a summation order that depended on the grid would change the bits (integer data cannot
    show that -- every order of their exact sums gives the same bits)."""
    pre, post = group_scales(world.n) if scales == "group" else (1.0 / 3.0, 0.7)
    per, v = 8 if sd == BF else 4, v_rs(world.n)
    drive(world, [ReduceScatter(world, range(world.n), c * per, sd, dd, accumulate, pre, post, integer=False)
                  for c in (1, 3 * THREADS * v + 5, 16 * THREADS * v + 1, 4099)])


@pytest.mark.parametrize("elems,twoshot", [(8, False), (8 * 1024, False), (8 * 1024 * 8, True), (1 << 21, True)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_all_reduce_sum(world, bg, elems, twoshot, dtype):
    """`elems` is rounded up to a whole number of vectors per member, so that the two-shot cases split evenly and really take
    the two-shot kernel at every group size."""
    n, per = world.n, 16 // _esz(dtype)
    elems = -(-elems // (n * per)) * n * per
    case = AllReduce(world, range(n), elems, dtype, bg.SUM, 1.0, integer=False)
    drive(world, [case], ctas=(16,), oneshot_bytes=1 if twoshot else 1 << 40)
    assert case.twoshot == (twoshot and n > 1)


def test_all_reduce_max_fp32(world, bg):
    drive(world, [AllReduce(world, range(world.n), 4096, F32, bg.MAX, 1.0, integer=False)], ctas=(16,))


AR_INT = [(BF, 0, 1.0), (BF, 0, 0.5), (F32, 0, 0.5), (BF, 1, 1.0 / 3.0), (F32, 1, 1.0)]


@pytest.mark.parametrize("path", ["oneshot", "twoshot"])
@pytest.mark.parametrize("dt,op,scale", AR_INT, ids=_ids)
def test_all_reduce_edges_integer_exact(world, dt, op, scale, path):
    """SUM at power-of-two scales on integer data, bit-exact; MAX at any scale, exact.  One-shot sizes are counted in vectors of
    the whole buffer, two-shot sizes in vectors of one member's slice (the two-shot loop runs over a slice)."""
    n, per = world.n, 16 // _esz(dt)
    if path == "twoshot" and n == 1:
        pytest.skip("a group of one has no two-shot path")
    two = path == "twoshot"
    nvecs = [v * n for v in edge_counts(n, v_ar(n, True))] if two else edge_counts(n, 1)
    cases = [AllReduce(world, range(n), v * per, dt, op, scale, integer=True) for v in nvecs]
    drive(world, cases, oneshot_bytes=1 if two else 1 << 40)
    assert all(c.twoshot == two for c in cases)


@pytest.mark.parametrize("path", ["oneshot", "twoshot"])
@pytest.mark.parametrize("scale", [1.0, 0.5, 1.0 / 3.0])
@pytest.mark.parametrize("dt", [BF, F32], ids=_ids)
def test_all_reduce_real(world, bg, dt, scale, path):
    n, per = world.n, 16 // _esz(dt)
    if path == "twoshot" and n == 1:
        pytest.skip("a group of one has no two-shot path")
    two = path == "twoshot"
    v = v_ar(n, two)          # sizes in vectors per member: a two-shot slice, or 1/n of the one-shot loop
    cases = [AllReduce(world, range(n), c * n * per, dt, op, scale, integer=False)
             for c in (1, 2 * THREADS + 3, 16 * THREADS * v + 1, 1500) for op in (bg.SUM, bg.MAX)]
    drive(world, cases, oneshot_bytes=1 if two else 1 << 40)     # real data under every grid size, as for the reduce-scatter
    assert all(c.twoshot == two for c in cases)


def test_all_reduce_uneven_above_threshold(world, bg):
    """Above oneshot_bytes a buffer whose vectors do not split evenly over the members takes the one-shot kernel: its result must
    be right and its sources must stay untouched (no two-shot write-back)."""
    n = world.n
    if n == 1:
        pytest.skip("needs a group")
    for dt in (BF, F32):
        per = 16 // _esz(dt)
        nvec = (512 * 1024 // 16 // n + 7) * n + 1              # above the default 512 KiB threshold, nvec % n == 1
        cases = [AllReduce(world, range(n), nvec * per, dt, bg.SUM, 0.5, integer=True),
                 AllReduce(world, range(n), (4 * n + 1) * per, dt, bg.SUM, 1.0 / 3.0, integer=False)]
        assert cases[0].elems * _esz(dt) > 512 * 1024
        drive(world, cases[:1], ctas=(16,), oneshot_bytes=512 * 1024)
        drive(world, cases[1:], ctas=(16,), oneshot_bytes=1)
        assert not any(c.twoshot for c in cases)


@pytest.mark.parametrize("dt", [BF, F32], ids=_ids)
def test_all_to_all_rows_edges(world, dt):
    """The exact descriptor CudaBackend.all_gather_first_dim builds at every loop edge, and the Ulysses exchange with batch 2:
    q, a GQA k with half the heads and v in one launch, and the inverse."""
    n, per = world.n, 16 // _esz(dt)
    d = 8 * per
    cases = [AllToAll(world, range(n), dt, [gather_first_dim(v * per, n)]) for v in edge_counts(n, K_IN_FLIGHT)]
    cases.append(AllToAll(world, range(n), dt, [ulysses_fwd(2, 5, 2 * n, d, n), ulysses_fwd(2, 5, n, d, n),
                                                ulysses_fwd(2, 5, n, d, n)]))
    cases.append(AllToAll(world, range(n), dt, [ulysses_inv(2, 3 * n, 2, d, n), ulysses_inv(2, 3 * n, 1, d, n)]))
    drive(world, cases)


OFF = 16 * 37     # bytes: a nonzero 16-B multiple, not a multiple of the 16,000-B slices below


def test_nonzero_byte_offsets(world, bg):
    """Every collective once more with its symmetric buffer entered at a byte offset, as CudaBackend's staging calls do."""
    n, ranks, s = world.n, range(world.n), 1000
    pre, post = group_scales(n)
    drive(world, [AllGather(world, ranks, s * 8, F32, BF, off=OFF), AllGather(world, ranks, s * 4, F32, F32, off=OFF),
                  ReduceScatter(world, ranks, s * 8, BF, BF, 0, 1.0, 1.0, integer=True, off=OFF),
                  ReduceScatter(world, ranks, s * 8, BF, F32, 1, pre, post, integer=False, off=OFF),
                  AllReduce(world, ranks, s * n * 8, BF, bg.SUM, 1.0, integer=True, off=OFF),
                  AllToAll(world, ranks, BF, [gather_first_dim(s * 8, n)], off=OFF)], ctas=(16,), oneshot_bytes=1 << 40)
    if n > 1:
        cases = [AllReduce(world, ranks, s * n * 4, F32, bg.SUM, 0.5, integer=False, off=OFF)]
        drive(world, cases, ctas=(16,), oneshot_bytes=1)
        assert cases[0].twoshot


def _strided_cases(w, bg, ranks):
    n = len(ranks)
    pre, post = group_scales(n)
    return [AllGather(w, ranks, 4099 * 8, F32, BF), ReduceScatter(w, ranks, 3001 * 8, BF, F32, 1, pre, post, integer=False),
            AllReduce(w, ranks, 2050 * n * 8, BF, bg.SUM, 0.5, integer=True),
            AllToAll(w, ranks, BF, [ulysses_fwd(2, 5, 2 * n, 64, n), gather_first_dim(777 * 8, n)])]


def test_oversized_counts_are_refused(world, bg):
    """An element count whose byte size exceeds the arena is refused with BG_EINVAL and no launch -- also when count x element
    size x members would wrap around to a small number (2^63 bf16 elements are 2^64 bytes, 0 modulo 2^64).  On a group of one,
    so that no peer could be left waiting."""
    if world.n != 1:
        pytest.skip("a group of one")
    c, L = world.comms[0], bg.lib()
    buf = world.sym(4096)[0]
    dst = torch.empty(4096, device="cuda")
    gid, sp = c.group_id(world.group), bg._vp(torch.cuda.current_stream().cuda_stream)
    huge = 1 << 63
    calls = [lambda: L.bg_all_gather_cast(c._ctx, gid, 0, bg._ptr(dst), bg.F32, buf.offs(), bg.BF16, huge, sp),
             lambda: L.bg_reduce_scatter_acc(c._ctx, gid, 1, buf.offs(), bg.BF16, bg._ptr(dst), bg.F32, huge, 1.0, 1.0, 0, sp),
             lambda: L.bg_all_reduce(c._ctx, gid, 2, buf.offs(), bg._ptr(dst), huge, bg.BF16, bg.SUM, 1.0, sp)]
    for call in calls:
        before = L.bg_launch_count()
        assert call() == -1
        assert "outside arena" in L.bg_last_error().decode()
        assert L.bg_launch_count() == before
    torch.cuda.synchronize()


def test_strided_groups_concurrent(world, bg):
    """The data-parallel groups of TP = 2 on 8 ranks, [0, 2, 4, 6] and [1, 3, 5, 7] -- where a member's index is not its rank --
    running each collective at the same time on the same lane."""
    if world.n != 8:
        pytest.skip("needs the 8-rank world")
    even, odd = _strided_cases(world, bg, [0, 2, 4, 6]), _strided_cases(world, bg, [1, 3, 5, 7])
    for a, b in zip(even, odd):
        drive(world, [a, b], oneshot_bytes=1)
    assert even[2].twoshot and odd[2].twoshot


def test_tp_all_reduce_beside_dp_reduce_scatter(world, bg):
    """Tensor-parallel all-reduces on [0, 1], [2, 3], ... (LANE_ACT, first stream of each rank) in flight at the same time as the
    data-parallel reduce-scatters on [0, 2, 4, 6] and [1, 3, 5, 7] (LANE_REDUCE, second stream)."""
    if world.n != 8:
        pytest.skip("needs the 8-rank world")
    pre, post = group_scales(4)
    tp = [AllReduce(world, [2 * k, 2 * k + 1], 6000 * 8, BF, bg.SUM, 1.0, integer=False, sidx=0) for k in range(4)]
    tp_small = [AllReduce(world, [2 * k, 2 * k + 1], 100 * 8, F32, bg.SUM, 1.0, integer=True, sidx=0) for k in range(4)]
    dp = [ReduceScatter(world, g, 5000 * 8, BF, F32, 1, pre, post, integer=False, sidx=1) for g in ([0, 2, 4, 6], [1, 3, 5, 7])]
    drive(world, tp + dp, oneshot_bytes=64 * 1024)
    drive(world, tp_small + dp, oneshot_bytes=64 * 1024)
    assert all(c.twoshot for c in tp) and not any(c.twoshot for c in tp_small)


def test_large_2p25_elements_per_rank(bg):
    """About 2^25 elements per rank on 8 ranks: the all-gather's gathered buffer, the reduce-scatter's and the two-shot
    all-reduce's source, and the all-to-all's gathered output."""
    n, big = 8, 1 << 25
    w = World(bg, n, arena=400 << 20)
    try:
        pre, post = group_scales(n)
        ranks = range(n)
        drive(w, [AllGather(w, ranks, big // n, F32, BF)], ctas=(16,))
        drive(w, [ReduceScatter(w, ranks, big // n, BF, F32, 1, pre, post, integer=False)], ctas=(16,))
        case = AllReduce(w, ranks, big, BF, bg.SUM, 1.0 / 3.0, integer=False)
        drive(w, [case], ctas=(16,))
        assert case.twoshot
        drive(w, [AllToAll(w, ranks, BF, [gather_first_dim(big // n, n)])], ctas=(16,))
    finally:
        w.close()


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
    oq = [torch.full((b, s, heads // p, d), float("nan"), device="cuda", dtype=torch.bfloat16) for _ in range(p)]
    ok = [torch.full((b, s, kv_heads // p, d), float("nan"), device="cuda", dtype=torch.bfloat16) for _ in range(p)]

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
    back = [torch.full((b, s // p, heads, d), float("nan"), device="cuda", dtype=torch.bfloat16) for _ in range(p)]
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
        with torch.cuda.stream(world.streams[0][0]):
            c0.p2p_send(1, off1, msgs[i], flag_id=3)
        with torch.cuda.stream(world.streams[0][1]):
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

"""GPU checks of ring context parallelism (``cp_comm="ring"``).

* the LSE merge kernel against its torch fp32 restatement (tests/_cp_ring_ref.py), with and without a query-row offset;
* the ring push and the accumulate-and-forward push with ``BgComm.local_world(c)`` virtual ranks, c = 2, 4, 8: after the hops every
  rank has seen every block bit for bit, and the accumulators equal the fixed-order fp32 sum bit for bit;
* the whole ring schedule of tensor_parallel/transformer.py, forward and backward, for c virtual ranks on one device at
  Llama-3.2-1B head shapes, against ONE flash-attn call on the un-zigzagged sequence;
* the context-parallel strategies of tests/test_cp_ring.py end to end through the CUDA path (skipped below the GPU count they need).

Virtual ranks issue their steps in step-major order on one stream, so every flag a kernel waits for was raised by work queued
before it."""
import os
import sys

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


class Ring:
    """c virtual ranks, each with its ring transport over one symmetric slot buffer"""

    def __init__(self, bg, c, capacity):
        from hetu_galvatron_b200.core.runtime.backend import CudaBackend, _CpRing
        from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
        self.bg, self.c = bg, c
        self.comms = bg.BgComm.local_world(c, device=0, arena_bytes=_CpRing.slot_bytes(capacity) + (64 << 20))
        self.group = CommGroup(list(range(c)))
        bufs = [cm.sym_alloc(self.group, _CpRing.slot_bytes(capacity)) for cm in self.comms]
        for cm in self.comms:
            cm.exchange()
        self.counts = {}
        self.rings = [_CpRing(cm, self.group, buf, capacity, counts=self.counts) for cm, buf in zip(self.comms, bufs)]
        self.be = CudaBackend(comm=self.comms[0])      # (local ops only: attention library calls, merge, casts)

    def check(self):
        torch.cuda.synchronize()
        for cm in self.comms:
            assert cm.error_flag() == 0, cm.error_info()

    def close(self):
        torch.cuda.synchronize()
        for cm in self.comms:
            cm.close()


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


# ---- LSE merge --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row_off,sq_blk", [(0, 256), (128, 128), (0, 128)])
def test_lse_merge_matches_torch(bg, row_off, sq_blk):
    from _cp_ring_ref import lse_merge_ref
    g = torch.Generator(device="cuda").manual_seed(3)
    b, s, n, d = 2, 256, 8, 64
    acc0 = torch.randn(b, s, n, d, device="cuda", generator=g)
    lse0 = torch.randn(b, n, s, device="cuda", generator=g) * 4
    blk = torch.randn(b, sq_blk, n, d, device="cuda", generator=g).bfloat16()
    blse = torch.randn(b, n, sq_blk, device="cuda", generator=g) * 4
    for final in (False, True):
        acc, lse = acc0.clone(), lse0.clone()
        out = torch.empty(b, s, n, d, device="cuda", dtype=torch.bfloat16) if final else None
        bg.lse_merge(blk, blse, acc, lse, out, row_off)
        racc, rlse = acc0.double(), lse0.double()
        lse_merge_ref(blk.double(), blse.double(), racc, rlse, None, row_off)
        torch.cuda.synchronize()
        # a few fp32 ulps (the kernel's expf / logf against correctly rounded fp64)
        assert torch.allclose(acc.double(), racc, rtol=1e-6, atol=1e-6), float((acc.double() - racc).abs().max())
        assert torch.allclose(lse.double(), rlse, rtol=1e-6, atol=1e-6), float((lse.double() - rlse).abs().max())
        if final:       # one rounding of the merged fp32 output, every row (also those the block did not cover)
            assert torch.equal(out, acc.bfloat16())
    # init: the running state becomes the block
    acc, lse = torch.empty(b, s, n, d, device="cuda"), torch.empty(b, n, s, device="cuda")
    blk = torch.randn(b, s, n, d, device="cuda", generator=g).bfloat16()
    blse = torch.randn(b, n, s, device="cuda", generator=g)
    bg.lse_merge(blk, blse, acc, lse, None, 0, init=True)
    assert torch.equal(acc, blk.float()) and torch.equal(lse, blse)


# ---- transport -------------------------------------------------------------------------------------------------------------
def _rows(r, j, half, s):
    from hetu_galvatron_b200.core.runtime.tensor_parallel.transformer import _ring_block
    _, nk, _ = _ring_block(r, j, half)
    return s if nk is None else nk


@pytest.mark.parametrize("c", [2, 4, 8])
def test_ring_push_and_accumulate_bit_exact(bg, c):
    b, s, ng, d = 2, 64, 8, 64
    W = Ring(bg, c, b * s * ng * d)
    try:
        g = torch.Generator(device="cuda").manual_seed(c)
        kv = [(torch.randn(b, s, ng, d, device="cuda", generator=g).bfloat16(),
               torch.randn(b, s, ng, d, device="cuda", generator=g).bfloat16()) for _ in range(c)]
        contrib = [[(torch.randn(b, _rows(r, (r - i) % c, s // 2, s), ng, d, device="cuda", generator=g).bfloat16(),
                     torch.randn(b, _rows(r, (r - i) % c, s // 2, s), ng, d, device="cuda", generator=g).bfloat16())
                    for i in range(c)] for r in range(c)]
        for rep in range(2):                    # twice: the second round waits for the first round's releases
            seen = [[None] * c for _ in range(c)]
            held = [kv[r] for r in range(c)]
            for i in range(c):
                for r, ring in enumerate(W.rings):
                    if i > 0:
                        held[r] = ring.recv_kv(i)
                        seen[r][(r - i) % c] = (held[r][0].clone(), held[r][1].clone())
                    if i < c - 1:
                        ring.send_kv(i, *held[r])
                    acc_in = ring.recv_acc(i) if i > 0 else None
                    dk, dv = contrib[r][i]
                    ring.send_acc(i, acc_in, dk, dv, 0, dk.shape[1])
                    if i > 0:
                        ring.release_acc(i)
                        ring.release_kv(i)
            final = []
            for ring in W.rings:
                final.append(ring.recv_acc(c).clone())
                ring.release_acc(c)
            W.check()
            for r in range(c):
                for j in range(c):
                    if j != r:
                        assert torch.equal(seen[r][j][0], kv[j][0]) and torch.equal(seen[r][j][1], kv[j][1]), (rep, r, j)
            for j in range(c):                  # owner j's block: contributions of ranks j, j+1, ... in that order
                want = torch.zeros(2, b, s, ng, d, device="cuda")
                for i in range(c):
                    dk, dv = contrib[(j + i) % c][i]
                    want[0][:, :dk.shape[1]] += dk.float()
                    want[1][:, :dv.shape[1]] += dv.float()
                assert torch.equal(final[j].view(want.shape), want), (rep, j)
        assert W.counts["cp_ring"] == 2 * ((c - 1) + c) * c
    finally:
        W.close()


# ---- whole ring attention against one flash-attn call ------------------------------------------------------------------------
def _zigzag(x, c, r):
    """rank r's chunks (r, 2c-1-r) of x [b, S, ...] along dim 1"""
    ch = x.shape[1] // (2 * c)
    return torch.cat([x[:, r * ch:(r + 1) * ch], x[:, (2 * c - 1 - r) * ch:(2 * c - r) * ch]], 1).contiguous()


def _unzigzag(parts, c, dim=1):
    ch = parts[0].shape[dim] // 2
    chunks = [None] * (2 * c)
    for r, p in enumerate(parts):
        a, b = p.split(ch, dim)
        chunks[r], chunks[2 * c - 1 - r] = a, b
    return torch.cat(chunks, dim)


@pytest.mark.parametrize("c,S", [(2, 8192), (4, 16384), (8, 32768)])
def test_ring_attention_matches_flash(bg, c, S):
    from flash_attn.flash_attn_interface import _flash_attn_backward, _flash_attn_forward
    from hetu_galvatron_b200.core.runtime.tensor_parallel import transformer as tr
    b, n, ng, d = 1, 32, 8, 64                  # Llama-3.2-1B attention
    scale = d ** -0.5
    W = Ring(bg, c, b * (S // c) * ng * d)
    try:
        g = torch.Generator(device="cuda").manual_seed(11)
        q = torch.randn(b, S, n, d, device="cuda", generator=g).bfloat16()
        k = torch.randn(b, S, ng, d, device="cuda", generator=g).bfloat16()
        v = torch.randn(b, S, ng, d, device="cuda", generator=g).bfloat16()
        dout = torch.randn(b, S, n, d, device="cuda", generator=g).bfloat16()
        out_ref, lse_ref, _, _ = _flash_attn_forward(q, k, v, 0.0, scale, causal=True, window_size_left=-1, window_size_right=-1,
                                                     softcap=0.0, alibi_slopes=None, return_softmax=False)
        dq_ref, dk_ref, dv_ref = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        _flash_attn_backward(dout, q, k, v, out_ref, lse_ref, dq_ref, dk_ref, dv_ref, 0.0, scale, True, -1, -1, 0.0, None, False)
        loc = [[_zigzag(t, c, r) for t in (q, k, v, dout)] for r in range(c)]
        fwd = [tr.ring_attention_fwd(W.be, W.rings[r], *loc[r][:3], scale) for r in range(c)]
        res = _interleave(fwd)
        bwd = [tr.ring_attention_bwd(W.be, W.rings[r], loc[r][3], *loc[r][:3], res[r][0], res[r][1], scale) for r in range(c)]
        grads = _interleave(bwd)
        W.check()
        out = _unzigzag([o for o, _ in res], c)
        lse = _unzigzag([l for _, l in res], c, dim=2)
        dq, dk, dv = [_unzigzag([gr[i] for gr in grads], c) for i in range(3)]
        obs = {"out_rel_l2": _rel(out, out_ref), "lse_max_abs": float((lse - lse_ref).abs().max()), "dq_rel_l2": _rel(dq, dq_ref),
               "dk_rel_l2": _rel(dk, dk_ref), "dv_rel_l2": _rel(dv, dv_ref)}
        print("CP_RING_OBS c=%d S=%d %s" % (c, S, obs), flush=True)
        assert obs["out_rel_l2"] < 1e-2 and obs["lse_max_abs"] < 1e-3, obs
        assert obs["dq_rel_l2"] < 2e-2 and obs["dk_rel_l2"] < 2e-2 and obs["dv_rel_l2"] < 2e-2, obs
    finally:
        W.close()


def _interleave(gens):
    """step-major: step i of every rank before step i + 1 of any"""
    done = [None] * len(gens)
    live = list(range(len(gens)))
    while live:
        for r in list(live):
            try:
                next(gens[r])
            except StopIteration as stop:
                done[r] = stop.value
                live.remove(r)
    return done


# ---- the strategies end to end --------------------------------------------------------------------------------------------
def _cases():
    from test_cp_ring import CASES
    return CASES


@pytest.mark.parametrize("world,name", _cases(), ids=[n for _, n in _cases()])
def test_ring_strategy_cuda(world, name):
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    from test_cp_ring import _CORPUS, launch
    rep = launch(world, dict(_CORPUS[world][name]), backend="cuda")
    assert rep["max_grad_err"] < 3e-2
    assert rep["ring_pushes"] > 0

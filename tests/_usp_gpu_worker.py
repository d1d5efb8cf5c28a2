"""Worker for tests/test_gpu_usp.py: the composed attention of tensor_parallel/transformer.py (``ulysses_cp_attention``: to-heads
all-to-all over the sp group, the cp exchange on those heads, the inverse all-to-all), forward and backward, for sp x cp virtual
ranks (``BgComm.local_world``) on one device, at Llama-3.2-1B head shapes, under both cp exchanges, against ONE flash-attn call on
the natural-order sequence; and the ring's merged LSE on the heads a rank holds after the exchange.  Prints one ``USP_CASE`` JSON
line per case.

Every virtual rank has its own backend, staging, ring slots and stream; rank r's whole forward (then backward) is issued with the
world rank simulated as r before rank r + 1's, so a collective of rank r waits on the device for peers the host issues later.
Nothing the host does in between may therefore wait for the device:
* modules load eagerly (CUDA_MODULE_LOADING=EAGER, set before CUDA starts): the first launch of a lazily loaded kernel waits for
  the device, i.e. for a collective whose peers are not issued yet, until the device-side timeout traps;
* the caching allocator is grown before the ranks run, so no device allocation happens among them.
A fault prints every virtual rank's timeout record (``error_info``)."""
import os

os.environ["CUDA_MODULE_LOADING"] = "EAGER"
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import json  # noqa: E402
import sys  # noqa: E402
import traceback  # noqa: E402

import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_HEADS, N_KV, HEAD_DIM = 32, 8, 64                     # Llama-3.2-1B attention
ATTN_CASES = [(sp, cp, S, comm) for sp, cp, S in ((2, 2, 8192), (2, 4, 16384), (4, 2, 16384)) for comm in ("allgather", "ring")]
LSE_CASES = [(2, 2, 8192), (2, 4, 16384), (4, 2, 16384)]


class UspWorld:
    """sp x cp virtual ranks; rank = cp_rank * sp + sp_rank (the sp-minor order of the tp_sp_cp groups)"""

    def __init__(self, bg, sp, cp, staging_bytes, ring_elems):
        from hetu_galvatron_b200.core.runtime.backend import CudaBackend, _CpRing
        from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
        self.sp, self.cp, self.n = sp, cp, sp * cp
        arena = 6 * staging_bytes + _CpRing.slot_bytes(ring_elems) + (64 << 20)
        self.comms = bg.BgComm.local_world(self.n, device=0, arena_bytes=arena)
        self.bes, self.sp_groups, self.cp_groups = [], [], []
        for r, cm in enumerate(self.comms):
            be = CudaBackend(comm=cm)
            spg = CommGroup([(r // sp) * sp + j for j in range(sp)])
            cpg = CommGroup([i * sp + r % sp for i in range(cp)])
            be.reserve_staging(spg, staging_bytes)
            be.reserve_staging(cpg, staging_bytes)
            be.reserve_cp_ring(cpg, ring_elems)
            self.bes.append(be)
            self.sp_groups.append(spg)
            self.cp_groups.append(cpg)
        for cm in self.comms:
            cm.exchange()
        self.streams = [torch.cuda.Stream() for _ in range(self.n)]

    def run(self, fn):
        """fn(r) for every rank, each on its own stream with its backend and world rank; -> the results"""
        from hetu_galvatron_b200.core.runtime import world as _world
        from hetu_galvatron_b200.core.runtime.backend import set_backend
        torch.cuda.synchronize()
        out = []
        for r in range(self.n):
            set_backend(self.bes[r])
            with _world.simulated(r, self.n), torch.cuda.stream(self.streams[r]):
                out.append(fn(r))
        torch.cuda.synchronize()
        for cm in self.comms:
            assert cm.error_flag() == 0, cm.error_info()
        return out

    def error_infos(self):
        out = []
        for cm in self.comms:
            try:
                out.append(cm.error_info())
            except Exception as e:  # noqa: BLE001 -- a faulted context may refuse
                out.append(repr(e))
        return out

    def close(self):
        from hetu_galvatron_b200.core.runtime.backend import set_backend
        torch.cuda.synchronize()
        set_backend(None)
        for cm in self.comms:
            cm.close()


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def _grow_allocator(gib):
    """one large cached segment (later large tensors are carved from it) and a stock of small-pool segments"""
    big = torch.empty(int(gib * (1 << 30)), dtype=torch.uint8, device="cuda")
    small = [torch.empty(1 << 20, dtype=torch.uint8, device="cuda") for _ in range(256)]
    del big, small


def _inputs(S, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(1, S, h, HEAD_DIM, device="cuda", generator=g).bfloat16() for h in (N_HEADS, N_KV, N_KV, N_HEADS)]


def _sizes(sp, cp, S):
    kv_heads = (N_KV if N_KV % sp == 0 else N_HEADS) // sp
    # staging: q + k + v of one exchange, or a gathered cp K/V (whole sequence, kv_heads) -- with slack
    staging = max(3 * (S // cp) * N_HEADS * HEAD_DIM * 2, 2 * S * kv_heads * HEAD_DIM * 2) + (1 << 20)
    return staging, (S // cp) * kv_heads * HEAD_DIM


def attn_case(bg, sp, cp, S, comm):
    from flash_attn.flash_attn_interface import _flash_attn_backward, _flash_attn_forward
    from hetu_galvatron_b200.core.runtime.redistribute import local_positions
    from hetu_galvatron_b200.core.runtime.tensor_parallel import transformer as tr
    scale = HEAD_DIM ** -0.5
    q, k, v, dout = _inputs(S, 11)
    out_ref, lse_ref, _, _ = _flash_attn_forward(q, k, v, 0.0, scale, causal=True, window_size_left=-1, window_size_right=-1,
                                                 softcap=0.0, alibi_slopes=None, return_softmax=False)
    dq_ref, dk_ref, dv_ref = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    _flash_attn_backward(dout, q, k, v, out_ref, lse_ref, dq_ref, dk_ref, dv_ref, 0.0, scale, True, -1, -1, 0.0, None, False)
    W = UspWorld(bg, sp, cp, *_sizes(sp, cp, S))
    try:
        pos = [local_positions(S, cp, r // sp, sp, r % sp).cuda() for r in range(W.n)]
        loc = [[t[:, pos[r]].contiguous().requires_grad_(True) for t in (q, k, v)] for r in range(W.n)]
        dloc = [dout[:, pos[r]].contiguous() for r in range(W.n)]
        _grow_allocator(4)
        outs = W.run(lambda r: tr.ulysses_cp_attention(*loc[r], W.sp_groups[r], W.cp_groups[r], scale, comm))
        W.run(lambda r: outs[r].backward(dloc[r]))
        got = {name: torch.zeros_like(ref) for name, ref in (("out", out_ref), ("dq", dq_ref), ("dk", dk_ref), ("dv", dv_ref))}
        for r in range(W.n):
            got["out"][:, pos[r]] = outs[r].detach()
            for name, t in zip(("dq", "dk", "dv"), loc[r]):
                got[name][:, pos[r]] = t.grad
        rec = {"kind": "attention", "sp": sp, "cp": cp, "S": S, "comm": comm, "out_rel_l2": _rel(got["out"], out_ref),
               "dq_rel_l2": _rel(got["dq"], dq_ref), "dk_rel_l2": _rel(got["dk"], dk_ref), "dv_rel_l2": _rel(got["dv"], dv_ref),
               "ring_pushes": sum(be.n_fused.get("cp_ring", 0) for be in W.bes)}
    except Exception:
        print("USP_ERROR_INFO " + json.dumps(W.error_infos()), flush=True)
        raise
    W.close()
    return rec


def lse_case(bg, sp, cp, S):
    from flash_attn.flash_attn_interface import _flash_attn_forward
    from hetu_galvatron_b200.core.runtime.redistribute import local_positions
    from hetu_galvatron_b200.core.runtime.tensor_parallel import transformer as tr
    scale = HEAD_DIM ** -0.5
    q, k, v, _ = _inputs(S, 5)
    _, lse_ref, _, _ = _flash_attn_forward(q, k, v, 0.0, scale, causal=True, window_size_left=-1, window_size_right=-1,
                                           softcap=0.0, alibi_slopes=None, return_softmax=False)
    W = UspWorld(bg, sp, cp, *_sizes(sp, cp, S))
    try:
        pos = [local_positions(S, cp, r // sp, sp, r % sp).cuda() for r in range(W.n)]
        loc = [[t[:, pos[r]].contiguous() for t in (q, k, v)] for r in range(W.n)]
        _grow_allocator(4)
        heads = W.run(lambda r: tr._ulysses_to_heads(*loc[r], W.sp_groups[r]))
        res = W.run(lambda r: tr.run_steps(tr.ring_attention_fwd(W.bes[r], W.bes[r].cp_ring(W.cp_groups[r]), *heads[r], scale)))
        worst = 0.0
        for r in range(W.n):
            rows = local_positions(S, cp, r // sp).cuda()                 # the cp rank's s/c zigzag rows, all of them
            hs = slice((r % sp) * N_HEADS // sp, (r % sp + 1) * N_HEADS // sp)   # the sp rank's heads
            worst = max(worst, float((res[r][1] - lse_ref[:, hs][:, :, rows]).abs().max()))
        rec = {"kind": "lse", "sp": sp, "cp": cp, "S": S, "comm": "ring", "lse_max_abs": worst}
    except Exception:
        print("USP_ERROR_INFO " + json.dumps(W.error_infos()), flush=True)
        raise
    W.close()
    return rec


def main():
    import hetu_galvatron_b200._bg as bg
    assert torch.cuda.is_available(), "needs a GPU"
    bg.lib()
    bg.set_tunable("timeout_ms", 20000)
    bg.set_tunable("comm_ctas", 16)  # 8 virtual ranks x 16 slim CTAs stay co-resident on one device
    for sp, cp, S, comm in ATTN_CASES:
        print("USP_CASE " + json.dumps(attn_case(bg, sp, cp, S, comm)), flush=True)
        torch.cuda.empty_cache()
    for sp, cp, S in LSE_CASES:
        print("USP_CASE " + json.dumps(lse_case(bg, sp, cp, S)), flush=True)
        torch.cuda.empty_cache()
    print("USP_DONE", flush=True)


if __name__ == "__main__":
    try:
        main()
    except Exception:
        traceback.print_exc()
        sys.exit(1)

"""Restatement of ring context parallelism on the CPU (TEST INFRASTRUCTURE ONLY).

* ``lse_merge_ref``: the log-sum-exp merge of include/bg_galvatron.h (bg_lse_merge) in torch fp32.
* ``CpRingOracleBackend``: the CPU (gloo) backend plus what the ring schedule of tensor_parallel/transformer.py asks of a backend:
  block attention with flash-attn's (out, LSE) interface and its backward from the merged out / LSE, the merge, and a ring
  transport whose hop is a gloo all-gather that keeps the previous member's block.  The schedule itself is the product's.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.gloo_backend import OracleBackend  # noqa: E402


def lse_merge_ref(blk_out, blk_lse, acc_out, acc_lse, final_out=None, row_off=0, init=False):
    """In place on acc_out [b, s, n, d] / acc_lse [b, n, s] (fp32); the block covers query rows row_off .. row_off + sq_blk - 1."""
    sq = blk_out.shape[1]
    ob, lb = blk_out.float(), blk_lse.float()
    if init:
        acc_out.copy_(ob)
        acc_lse.copy_(lb)
    else:
        oa, la = acc_out[:, row_off:row_off + sq], acc_lse[:, :, row_off:row_off + sq]
        m = torch.maximum(la, lb)
        lse = m + torch.log(torch.exp(la - m) + torch.exp(lb - m))
        wa, wb = torch.exp(la - lse), torch.exp(lb - lse)                  # [b, n, sq]
        oa.copy_(oa * wa.transpose(1, 2)[..., None] + ob * wb.transpose(1, 2)[..., None])
        la.copy_(lse)
    if final_out is not None:
        final_out.copy_(acc_out.to(final_out.dtype))


class _GlooRing:
    """One hop = an all-gather over the cp group from which every member keeps its previous member's block."""

    def __init__(self, be, group):
        self.be, self.group = be, group
        self.size, self.rank = group.size, group.rank_in_group(be.rank)
        self._kv, self._acc, self.shape = {}, {}, None

    def _from_prev(self, t):
        allt = self.be.all_gather_first_dim(t.contiguous().unsqueeze(0), self.group)
        return allt[(self.rank - 1) % self.size].clone()

    def _count(self):
        self.be.n_fused["cp_ring"] = self.be.n_fused.get("cp_ring", 0) + 1

    def send_kv(self, step, k, v):
        self.shape = tuple(k.shape)
        self._kv[step + 1] = (self._from_prev(k), self._from_prev(v))
        self._count()

    def recv_kv(self, step):
        return self._kv.pop(step)

    def release_kv(self, step):
        pass

    def send_acc(self, step, acc_in, dk, dv, c_row0, c_rows):
        nxt = torch.zeros((2,) + self.shape, dtype=torch.float32) if acc_in is None else acc_in.view((2,) + self.shape).clone()
        nxt[0][:, c_row0:c_row0 + c_rows] += dk.float()
        nxt[1][:, c_row0:c_row0 + c_rows] += dv.float()
        self._acc[step + 1] = self._from_prev(nxt).reshape(-1)
        self._count()

    def recv_acc(self, step):
        return self._acc.pop(step)

    def release_acc(self, step):
        pass


class CpRingOracleBackend(OracleBackend):
    """The gloo backend with the ring's backend methods of ``CudaBackend`` restated on the CPU."""

    def __init__(self):
        super().__init__()
        self.n_fused = {"cp_ring": 0}
        self._rings = {}

    def reserve_cp_ring(self, group, elems):
        pass

    def cp_ring(self, group):
        key = tuple(group.ranks)
        if key not in self._rings:
            self._rings[key] = _GlooRing(self, group)
        return self._rings[key]

    def lse_merge(self, blk_out, blk_lse, acc_out, acc_lse, final_out=None, row_off=0, init=False):
        lse_merge_ref(blk_out, blk_lse, acc_out, acc_lse, final_out, row_off, init)

    @staticmethod
    def _scores(q, k, causal, softmax_scale, key_mask):
        rep = q.shape[2] // k.shape[2]
        qf, kf = q.float().transpose(1, 2), k.float().repeat_interleave(rep, 2).transpose(1, 2)
        scores = qf @ kf.transpose(-1, -2) * softmax_scale                               # [b, n, sq, sk]
        if key_mask is not None:
            scores = scores.masked_fill(~key_mask.bool()[:, None, None, :], float("-inf"))
        if causal:      # bottom-right aligned, as flash-attn
            sq, sk = scores.shape[-2:]
            scores = scores.masked_fill(torch.arange(sk)[None, :] > torch.arange(sq)[:, None] + (sk - sq), float("-inf"))
        return scores

    # flash-attn's interface: (out, LSE [b, n, sq] fp32, rng); the backward takes the (possibly merged) out and LSE
    def attention_fwd(self, q, k, v, causal, softmax_scale, key_mask=None):
        rep = q.shape[2] // k.shape[2]
        scores = self._scores(q, k, causal, softmax_scale, key_mask)
        lse = torch.logsumexp(scores, -1)
        p = torch.exp(scores - lse[..., None])
        out = (p @ v.float().repeat_interleave(rep, 2).transpose(1, 2)).transpose(1, 2).contiguous().to(q.dtype)
        return out, lse.contiguous(), None

    def attention_bwd(self, dout, q, k, v, out, lse, causal, softmax_scale, rng):
        rep = q.shape[2] // k.shape[2]
        b, sk, ng, d = k.shape
        p = torch.exp(self._scores(q, k, causal, softmax_scale, None) - lse.float()[..., None])
        qf, kf, vf = q.float(), k.float().repeat_interleave(rep, 2), v.float().repeat_interleave(rep, 2)
        qf, kf, vf, do = [t.transpose(1, 2) for t in (qf, kf, vf, dout.float())]
        delta = (dout.float() * out.float()).sum(-1).transpose(1, 2)                       # [b, n, sq]
        dv = p.transpose(-1, -2) @ do
        ds = p * (do @ vf.transpose(-1, -2) - delta[..., None]) * softmax_scale
        dq = (ds @ kf).transpose(1, 2)
        dk = (ds.transpose(-1, -2) @ qf).transpose(1, 2).reshape(b, sk, ng, rep, d).sum(3)
        dv = dv.transpose(1, 2).reshape(b, sk, ng, rep, d).sum(3)
        return dq.contiguous().to(q.dtype), dk.contiguous().to(k.dtype), dv.contiguous().to(v.dtype)

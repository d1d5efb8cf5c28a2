"""The CPU (gloo) backend with the T5 method pair of ``CudaBackend`` restated in torch (TEST INFRASTRUCTURE ONLY).

``T5OracleBackend`` extends oracle/gloo_backend.OracleBackend with bg_cross_attn_qkv_fwd / bg_cross_attn_qkv_bwd of
include/bg_galvatron.h: the two projections' SBH outputs + bias (fp32 add, one rounding) -> q [b, s_q, heads, hn] and k, v
[b, s_k, heads, hn] (per head k | v in kv_mixed), and back, with the bias gradients as fp32 column sums.  The GPU tests compare the
kernels against these functions bit for bit (the dbias sums, whose order differs, within fp32 summation error)."""
import torch

from oracle.gloo_backend import OracleBackend


def cross_attn_qkv_fwd(q_mixed, q_bias, kv_mixed, kv_bias, heads, hn):
    s_q, b, s_k = q_mixed.shape[0], q_mixed.shape[1], kv_mixed.shape[0]
    q, kv = q_mixed, kv_mixed
    if q_bias is not None:
        q = (q.float() + q_bias.float()).to(q_mixed.dtype)
    if kv_bias is not None:
        kv = (kv.float() + kv_bias.float()).to(kv_mixed.dtype)
    q = q.reshape(s_q, b, heads, hn).transpose(0, 1).contiguous()
    kv = kv.reshape(s_k, b, heads, 2, hn).transpose(0, 1)
    return q, kv[:, :, :, 0].contiguous(), kv[:, :, :, 1].contiguous()


def cross_attn_qkv_bwd(dq, dk, dv):
    b, s_q, heads, hn = dq.shape
    s_k = dk.shape[1]
    dqm = dq.transpose(0, 1).reshape(s_q, b, heads * hn).contiguous()
    dkvm = torch.stack([dk, dv], dim=3).transpose(0, 1).reshape(s_k, b, heads * 2 * hn).contiguous()
    return dqm, dkvm, dqm.float().reshape(-1, heads * hn).sum(0), dkvm.float().reshape(-1, heads * 2 * hn).sum(0)


class T5OracleBackend(OracleBackend):
    def cross_attn_qkv_fwd(self, q_mixed, q_bias, kv_mixed, kv_bias, heads, hn):
        return cross_attn_qkv_fwd(q_mixed, q_bias, kv_mixed, kv_bias, heads, hn)

    def cross_attn_qkv_bwd(self, dq, dk, dv):
        return cross_attn_qkv_bwd(dq, dk, dv)

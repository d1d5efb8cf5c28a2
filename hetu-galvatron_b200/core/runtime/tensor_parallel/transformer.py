"""Transformer-layer math around the per-layer collectives: ``ParallelMLP`` / ``ParallelAttention`` with explicit
``tp_group / sp_group / cp_group`` (``galvatron/core/runtime/tensor_parallel/transformer.py``: ParallelMLP :82-166,
ParallelAttention :512-900, Ulysses ``_SeqAllToAll`` / ``DistributedAttention`` :1990-2177) and the fused RMSNorm the
Llama family uses (``flash_attn.ops.rms_norm.RMSNorm``, LlamaModel_tensor_parallel.py:2,48).

Data flow of one attention block (SBH activations, flash layout inside):
    hidden [s,b,h] -> ColumnParallelLinear (wgmma GEMM, TP/SP comm in staging)            -> mixed [s,b,ng*(r+2)*hn]
    -> ONE kernel: QKV split + RoPE + SBH->BSND relayout (K/V stay un-expanded for GQA)        -> q,k,v
    -> [Ulysses: ONE pull all-to-all for q,k,v with the head/seq transpose folded in]
    -> attention LIBRARY call (cuDNN SDPA; the reference calls flash-attn) -> [Ulysses: inverse all-to-all] -> context [s,b,np*hn]
    -> RowParallelLinear (GEMM into staging -> all-reduce | reduce-scatter over NVLink)      -> out [s,b,h]
The reference runs split, repeat_interleave, 2x rope, 3x rearrange().contiguous() and, per Ulysses tensor, a permute
copy + NCCL all_to_all + a second permute copy (transformer.py:731-767,842-867,1934-1962).
"""
import enum
import math

import torch
import torch.nn as nn

from ..backend import get_backend
from .layers import ColumnParallelLinear, RowParallelLinear
from .random import check_probability, get_rng_tracker, model_parallel_seed


class AttnType(enum.Enum):
    self_attn = 1
    cross_attn = 2


class AttnMaskType(enum.Enum):
    padding = 1
    causal = 2


def _size(group):
    return 1 if group is None else group.size


# ---------------------------------------------------------------------------------------------------------------
# fused elementwise autograd ops
# ---------------------------------------------------------------------------------------------------------------
class _RMSNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, eps):
        y, rstd = get_backend().rmsnorm_fwd(x.contiguous(), weight, eps)
        ctx.save_for_backward(x, weight, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, rstd = ctx.saved_tensors
        dx, dw = get_backend().rmsnorm_bwd(dy.contiguous(), x.contiguous(), weight, rstd)
        return dx, dw, None


class RMSNorm(nn.Module):
    """y = x * rsqrt(mean(x^2) + eps) * weight, fp32 math, one rounding (flash_attn.ops.rms_norm semantics)."""

    def __init__(self, hidden_size, eps=1e-5, params_dtype=torch.float32, device=None, sequence_parallel=False):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.empty(hidden_size, dtype=params_dtype, device=device))
        # under Megatron-SP the norm sees only the local sequence slice: its grad is summed over the TP group on the
        # last microbatch (sp_grad_reduce.py:104-123)
        self._sequence_parallel = bool(sequence_parallel)
        setattr(self.weight, "sequence_parallel", self._sequence_parallel)
        if self.weight.device.type != "meta":
            self.reset_parameters()

    def reset_parameters(self):
        nn.init.ones_(self.weight)
        # (re)tag: materialising from the meta device replaces the Parameter object and drops custom attributes
        setattr(self.weight, "sequence_parallel", self._sequence_parallel)

    def forward(self, x):
        return _RMSNormFn.apply(x, self.weight, self.eps)


class _SwigluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gate_up):
        gate_up = gate_up.contiguous()
        ctx.save_for_backward(gate_up)
        return get_backend().swiglu_fwd(gate_up)

    @staticmethod
    def backward(ctx, dy):
        (gate_up,) = ctx.saved_tensors
        return get_backend().swiglu_bwd(dy.contiguous(), gate_up)


class _QkvRopeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mixed, cos, sin, ng, r, hn, stage_group):
        ctx.save_for_backward(cos, sin)
        ctx.dims = (ng, r, hn)
        q, k, v = get_backend().qkv_rope_fwd(mixed.contiguous(), cos, sin, ng, r, hn, stage_group)
        return q, k, v

    @staticmethod
    def backward(ctx, dq, dk, dv):
        cos, sin = ctx.saved_tensors
        ng, r, hn = ctx.dims
        return get_backend().qkv_rope_bwd(dq, dk, dv, cos, sin, ng, r, hn), None, None, None, None, None, None


class _CrossQkvFn(torch.autograd.Function):
    """Cross-attention relayout: the query projection's output (+ bias) and the key_value projection's output (+ bias) -> q, k, v in
    one kernel; backward gives both projections' dgrad inputs and both biases' gradients in one kernel."""

    @staticmethod
    def forward(ctx, q_mixed, q_bias, kv_mixed, kv_bias, heads, hn):
        ctx.bias_dtypes = (None if q_bias is None else q_bias.dtype, None if kv_bias is None else kv_bias.dtype)
        return get_backend().cross_attn_qkv_fwd(q_mixed, q_bias, kv_mixed, kv_bias, heads, hn)

    @staticmethod
    def backward(ctx, dq, dk, dv):
        dqm, dkvm, dqb, dkvb = get_backend().cross_attn_qkv_bwd(dq, dk, dv)
        qdt, kvdt = ctx.bias_dtypes
        return dqm, (None if qdt is None else dqb.to(qdt)), dkvm, (None if kvdt is None else dkvb.to(kvdt)), None, None


class _CrossKvFn(torch.autograd.Function):
    """The key_value projection of a cross-attention layer on the encoder output, which also returns the encoder output itself: a
    decoder layer passes it on to the next one.  Backward sums the gradient of that pass-through into the projection's dgrad -- as the
    dgrad GEMM's addend when no collective follows it (tensor-parallel degree 1), else once after the all-reduce / Megatron-SP
    reduce-scatter -- instead of autograd's separate add (and buffer) per decoder layer."""

    @staticmethod
    def forward(ctx, encoder_output, weight, sequence_parallel, tp_group):
        ctx.set_materialize_grads(False)
        from .layers import LinearWithGradAccumulationAndAsyncCommunication as Linear
        out = Linear.forward(ctx, encoder_output, weight, sequence_parallel, not sequence_parallel, False, tp_group)
        return out, encoder_output

    @staticmethod
    def backward(ctx, grad_kv, grad_passthrough):
        if grad_kv is None:
            return grad_passthrough, None, None, None
        from .layers import LinearWithGradAccumulationAndAsyncCommunication as Linear
        ctx.dgrad_addend = grad_passthrough
        grads = Linear.backward(ctx, grad_kv)
        return grads[0], grads[1], None, None


class _UlyssesFn(torch.autograd.Function):
    """All tensors of one exchange in one launch; backward is the inverse exchange (transformer.py:2040-2062)."""

    @staticmethod
    def forward(ctx, group, to_heads, *tensors):
        ctx.group, ctx.to_heads = group, to_heads
        return tuple(get_backend().ulysses_all_to_all(list(tensors), group, to_heads))

    @staticmethod
    def backward(ctx, *grads):
        back = get_backend().ulysses_all_to_all([g.contiguous() for g in grads], ctx.group, not ctx.to_heads)
        return (None, None) + tuple(back)


class _FlashAttnFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, causal, softmax_scale, key_mask=None, dropout_p=0.0):
        drop = {"dropout_p": dropout_p} if dropout_p > 0.0 else {}      # (the backend draws the mask; its backward replays it)
        if key_mask is None:
            out, lse, rng = get_backend().attention_fwd(q, k, v, causal, softmax_scale, **drop)
        else:
            out, lse, rng = get_backend().attention_fwd(q, k, v, causal, softmax_scale, key_mask, **drop)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.causal, ctx.scale, ctx.rng, ctx.drop = causal, softmax_scale, rng, drop
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse = ctx.saved_tensors
        dq, dk, dv = get_backend().attention_bwd(dout, q, k, v, out, lse, ctx.causal, ctx.scale, ctx.rng, **ctx.drop)
        return dq, dk, dv, None, None, None, None


class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps):
        y, mean, rstd = get_backend().layernorm_fwd(x.contiguous(), weight, bias, eps)
        ctx.save_for_backward(x, weight, mean, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, mean, rstd = ctx.saved_tensors
        dx, dw, db = get_backend().layernorm_bwd(dy.contiguous(), x.contiguous(), weight, mean, rstd)
        return dx, dw, db, None


class LayerNorm(nn.Module):
    """``torch.nn.LayerNorm`` of the GPT / BERT families (gpt_hf/GPTModel_tensor_parallel.py:34, bert_hf/BertModel_tensor_parallel.py)
    as one fused row kernel forward and one backward: y = (x - mean) * rstd * weight + bias, fp32 math, one rounding."""

    def __init__(self, hidden_size, eps=1e-5, params_dtype=torch.float32, device=None, sequence_parallel=False):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.empty(hidden_size, dtype=params_dtype, device=device))
        self.bias = nn.Parameter(torch.empty(hidden_size, dtype=params_dtype, device=device))
        self._sequence_parallel = bool(sequence_parallel)
        if self.weight.device.type != "meta":
            self.reset_parameters()

    def reset_parameters(self):
        nn.init.ones_(self.weight)
        nn.init.zeros_(self.bias)
        # under Megatron-SP the norm sees only the local sequence slice: its grads are summed over the TP group on the last
        # microbatch (sp_grad_reduce.py:104-123); (re)tag here, materialising from meta makes new Parameter objects
        setattr(self.weight, "sequence_parallel", self._sequence_parallel)
        setattr(self.bias, "sequence_parallel", self._sequence_parallel)

    def forward(self, x):
        return _LayerNormFn.apply(x, self.weight, self.bias, self.eps)


class _BiasGeluFn(torch.autograd.Function):
    """gelu(x + bias) of the GPT / BERT MLP in one pass (transformer.py:150-160 ``bias_gelu_impl``); dbias = column sums of dx."""

    @staticmethod
    def forward(ctx, x, bias, tanh_form):
        x = x.contiguous()
        ctx.save_for_backward(x, bias)
        ctx.tanh_form = tanh_form
        return get_backend().bias_gelu_fwd(x, bias, tanh_form)

    @staticmethod
    def backward(ctx, dy):
        x, bias = ctx.saved_tensors
        dx = get_backend().bias_gelu_bwd(dy.contiguous(), x, bias, ctx.tanh_form)
        db = None if bias is None else dx.reshape(-1, dx.shape[-1]).float().sum(0).to(bias.dtype)
        return dx, db, None


class _CpGatherKvFn(torch.autograd.Function):
    """Context parallelism, K or V: this rank's two zigzag chunks [b, s/c, ng, d] -> the whole sequence in natural token order
    [b, s, ng, d] (all-gather over the cp group + un-zigzag); backward re-applies the zigzag order and reduce-scatters the
    gradient (the reference's ring passes the same bytes around hop by hop, transformer.py:2252-2680)."""

    @staticmethod
    def forward(ctx, x, group):
        from ..redistribute import _reverse_zigzag_transformation
        b, s_loc, ng, d = x.shape
        ctx.group, ctx.dims = group, (b, s_loc, ng, d)
        rows = x.transpose(0, 1).contiguous().reshape(s_loc, b * ng * d)
        full = get_backend().all_gather_first_dim(rows, group)                       # rank-major chunk order
        full = _reverse_zigzag_transformation(full, group.size)
        return full.reshape(group.size * s_loc, b, ng, d).transpose(0, 1).contiguous()

    @staticmethod
    def backward(ctx, grad):
        from ..redistribute import _zigzag_transformation
        b, s_loc, ng, d = ctx.dims
        c = ctx.group.size
        rows = grad.transpose(0, 1).contiguous().reshape(c * s_loc, b * ng * d)
        rows = _zigzag_transformation(rows, c)
        out = get_backend().reduce_scatter_first_dim(rows, ctx.group)
        return out.reshape(s_loc, b, ng, d).transpose(0, 1).contiguous(), None


def _cp_attention(q, k, v, group, scale):
    """Causal self-attention under zigzag context parallelism: the rank holds token chunks (r, 2c-1-r); each chunk attends
    the gathered keys/values up to its own end."""
    be = get_backend()
    c, r = group.size, group.rank_in_group()
    k_full, v_full = _CpGatherKvFn.apply(k, group), _CpGatherKvFn.apply(v, group)
    half = q.shape[1] // 2
    outs = []
    for q_blk, chunk in ((q[:, :half], r), (q[:, half:], 2 * c - 1 - r)):
        end = (chunk + 1) * half
        outs.append(be.attention_prefix(q_blk, k_full[:, :end], v_full[:, :end], scale))
    return torch.cat(outs, 1)


CP_COMM_MODES = ("allgather", "ring")


def cp_comm_mode():
    """``args.cp_comm``: how a context-parallel layer exchanges keys/values (``"allgather"``, the default, or ``"ring"``)."""
    try:
        from ..arguments import get_args
        mode = getattr(get_args(), "cp_comm", "allgather")
    except RuntimeError:
        mode = "allgather"
    if mode not in CP_COMM_MODES:
        raise ValueError("cp_comm must be one of %s, not %r" % (", ".join(CP_COMM_MODES), mode))
    return mode


# ---- ring context parallelism (the reference's zigzag ring, transformer.py:2209-2551) ----------------------------------------
# Rank r of c holds queries and keys of the zigzag chunks (r, 2c-1-r), s_loc/2 rows each.  Step i works on the K/V block of rank
# j = (r - i) mod c, which reaches r after i hops: step 0 is local q x local K/V, causal; for j < r every query sees the block's
# first chunk (chunk j) and nothing of its second; for j > r only the second query chunk (2c-1-r) sees the block, all of it.
# The step functions below are generators that yield after every step: a model runs one rank's steps back to back, a test with
# several ranks on one device interleaves them.  The transport (``ring``: send/recv/release of K/V and of the dK/dV accumulators)
# is the only part that differs between backends.
def _ring_block(r, j, half):
    """-> (first query row, K/V rows used or None for all, causal) of the step that holds rank j's block"""
    if j == r:
        return 0, None, True
    if j < r:
        return 0, half, False
    return half, None, False


def run_steps(gen):
    """drive a step generator to its end; -> its return value"""
    while True:
        try:
            next(gen)
        except StopIteration as stop:
            return stop.value


def ring_attention_fwd(be, ring, q, k, v, scale):
    """-> (out [b, s_loc, n, d] bf16, lse [b, n, s_loc] fp32) of causal attention of the local queries over the whole sequence"""
    c, r = ring.size, ring.rank
    b, s, n, d = q.shape
    half = s // 2
    acc_out = torch.empty(b, s, n, d, dtype=torch.float32, device=q.device)
    acc_lse = torch.empty(b, n, s, dtype=torch.float32, device=q.device)
    out = torch.empty_like(q)
    kv = (k, v)
    for i in range(c):
        if i > 0:
            kv = ring.recv_kv(i)
        if i < c - 1:
            ring.send_kv(i, *kv)           # the next step's block travels while this step's attention runs
        q0, nk, causal = _ring_block(r, (r - i) % c, half)
        kb, vb = kv if nk is None else (kv[0][:, :nk], kv[1][:, :nk])
        o, lse, _ = be.attention_fwd(q[:, q0:], kb, vb, causal, scale)
        be.lse_merge(o, lse, acc_out, acc_lse, out if i == c - 1 else None, q0, init=i == 0)
        if i > 0:
            ring.release_kv(i)
        yield
    return out, acc_lse


def ring_attention_bwd(be, ring, dout, q, k, v, out, lse, scale):
    """-> (dq, dk, dv) bf16: the block backward of every step with the merged out / LSE; dq accumulates in fp32 here, dK/dV in the
    fp32 accumulators that travel with the blocks and are back at their owner after the c-th hop"""
    c, r = ring.size, ring.rank
    b, s, n, d = q.shape
    half = s // 2
    dq_acc = torch.empty(b, s, n, d, dtype=torch.float32, device=q.device)
    kv = (k, v)
    for i in range(c):
        if i > 0:
            kv = ring.recv_kv(i)
        if i < c - 1:
            ring.send_kv(i, *kv)
        q0, nk, causal = _ring_block(r, (r - i) % c, half)
        kb, vb = kv if nk is None else (kv[0][:, :nk], kv[1][:, :nk])
        lse_b = lse if q0 == 0 else lse[:, :, q0:].contiguous()
        dq, dk, dv = be.attention_bwd(dout[:, q0:], q[:, q0:], kb, vb, out[:, q0:], lse_b, causal, scale, None)
        if q0 == 0:
            be.cast(dq, dq_acc, accumulate=i > 0)
        else:
            for bi in range(b):            # (rows q0.. of one sample are contiguous)
                be.cast(dq[bi], dq_acc[bi, q0:], accumulate=True)
        acc_in = ring.recv_acc(i) if i > 0 else None
        ring.send_acc(i, acc_in, dk, dv, 0, s if nk is None else nk)
        if i > 0:
            ring.release_acc(i)
            ring.release_kv(i)
        yield
    acc = ring.recv_acc(c)
    dk_out, dv_out = torch.empty_like(k), torch.empty_like(v)
    be.cast(acc[:k.numel()].view(k.shape), dk_out)
    be.cast(acc[k.numel():].view(v.shape), dv_out)
    ring.release_acc(c)
    dq_out = torch.empty_like(q)
    be.cast(dq_acc, dq_out)
    return dq_out, dk_out, dv_out


class _CpRingAttnFn(torch.autograd.Function):
    """Causal self-attention under zigzag context parallelism over the ring: only this rank's K/V (s/c rows) is kept for
    backward; the other blocks pass through the receive slots hop by hop, in the forward and again in the backward."""

    @staticmethod
    def forward(ctx, q, k, v, group, scale):
        be = get_backend()
        ring = be.cp_ring(group)
        out, lse = run_steps(ring_attention_fwd(be, ring, q, k, v, scale))
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.group, ctx.scale = group, scale
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse = ctx.saved_tensors
        be = get_backend()
        dq, dk, dv = run_steps(ring_attention_bwd(be, be.cp_ring(ctx.group), dout.contiguous(), q, k, v, out, lse, ctx.scale))
        return dq, dk, dv, None, None


def cp_attention(q, k, v, group, scale, comm):
    """Causal attention of a cp rank's zigzag rows [b, s/c, n, d] over the whole sequence, by the exchange ``comm`` names
    (``cp_comm``: "allgather" or "ring")."""
    if comm == "ring" and _size(group) > 1:
        return _CpRingAttnFn.apply(q, k, v, group, scale)
    return _cp_attention(q, k, v, group, scale)


def _ulysses_to_heads(q, k, v, sp_group):
    """[b, s/p, n, d] -> [b, s, n/p, d] in one exchange; K/V with fewer heads than p are first expanded to the query heads, as the
    reference does (transformer.py:842-848)"""
    p = sp_group.size
    if k.shape[2] % p:
        rep = q.shape[2] // k.shape[2]
        k, v = k.repeat_interleave(rep, dim=2), v.repeat_interleave(rep, dim=2)
    return _UlyssesFn.apply(sp_group, True, q, k, v)


def ulysses_cp_attention(q, k, v, sp_group, cp_group, scale, comm):
    """Ulysses and zigzag context parallelism on one layer (the reference wraps its zigzag ring in DistributedAttention,
    transformer.py:641-654): this rank's rows [b, s/(c*p), n, d] -> the to-heads exchange over the sp group gives the cp rank's s/c
    zigzag rows of n/p heads (the sp ranks hold contiguous slices of them, redistribute.local_positions), the cp exchange
    attends them over the whole sequence, the inverse exchange returns [b, s/(c*p), n, d].  Only the existing kernels run."""
    q, k, v = _ulysses_to_heads(q, k, v, sp_group)                      # [b, s/c, n/p, d]
    ctxt = cp_attention(q, k, v, cp_group, scale, comm)
    return _UlyssesFn.apply(sp_group, False, ctxt)[0]


def _check_ulysses_cp(p, c, kv_row_bytes):
    """Construction-time limits of a layer with both Ulysses (degree p) and context parallelism (degree c), beyond Ulysses' own
    n_heads % p: the sequence splits into 2c zigzag chunks whose concatenated pairs split p ways, and every K/V row the exchanges
    move is whole 16-byte vectors."""
    try:
        from ..arguments import get_args
        seq = getattr(get_args(), "seq_length", None)
    except RuntimeError:
        seq = None
    if seq is not None and seq % (2 * c * p):
        raise ValueError("sequence length %d must be a multiple of 2 x cp x sp = %d when context parallelism (cp %d) and Ulysses "
                         "(sp %d) share a layer" % (seq, 2 * c * p, c, p))
    if kv_row_bytes % 16:
        raise ValueError("a K/V row of %d bytes per token after the Ulysses exchange is not a multiple of 16 bytes" % kv_row_bytes)


def _recompute_activations():
    try:
        from ..arguments import get_args
        return bool(getattr(get_args(), "recompute_activations", False))
    except RuntimeError:
        return False


def _attention(q, k, v, causal, scale, key_mask=None, dropout_p=0.0):
    be = get_backend()
    fn = getattr(be, "attention", None)
    drop = {"dropout_p": dropout_p} if dropout_p > 0.0 else {}
    if fn is None:
        out = None
    elif key_mask is None:
        out = fn(q, k, v, causal, scale, **drop)                    # differentiable library call (cuDNN SDPA)
    else:
        out = fn(q, k, v, causal, scale, key_mask, **drop)
    return out if out is not None else _FlashAttnFn.apply(q, k, v, causal, scale, key_mask, dropout_p)


# ---------------------------------------------------------------------------------------------------------------
# layer modules
# ---------------------------------------------------------------------------------------------------------------
class ParallelMLP(nn.Module):
    """h -> 4h (column-parallel) -> activation -> h (row-parallel) (transformer.py:82-166).
    Llama: gated (gate|up, swiglu), no biases.  GPT / BERT (``add_bias_linear``, not gated): bias + GeLU in one fused pass
    (``bias_gelu_impl``, :150-160), the output bias is returned for the caller to add (``skip_bias_add``, :162-166)."""

    def __init__(self, config, is_expert=False, tp_group=None, params_dtype=torch.float32, device=None):
        super().__init__()
        self.tp_group = tp_group
        ffn = config.ffn_hidden_size
        self.gated = getattr(config, "gated_linear_unit", True)
        self.add_bias = bool(getattr(config, "add_bias_linear", False))
        self.gelu_tanh = bool(getattr(config, "gelu_tanh", True))
        self.dense_h_to_4h = ColumnParallelLinear(config.hidden_size, ffn * 2 if self.gated else ffn, config=config, bias=self.add_bias,
                                                  gather_output=False, skip_bias_add=True, tp_group=tp_group,
                                                  params_dtype=params_dtype, device=device)
        self.dense_4h_to_h = RowParallelLinear(ffn, config.hidden_size, config=config, bias=self.add_bias, input_is_parallel=True,
                                               skip_bias_add=True, tp_group=tp_group, params_dtype=params_dtype, device=device)

    def forward(self, hidden_states, input_recipe=None, residual=None):
        """``residual`` (optional): the block's residual, added to the output inside the last GEMM's epilogue."""
        gate_up, bias = self.dense_h_to_4h(hidden_states, recompute=input_recipe)
        if self.gated:
            if bias is not None:
                gate_up = gate_up + bias
            inter = _SwigluFn.apply(gate_up)
            # --recompute_activations: the 4h->h GEMM keeps gate_up (which SwiGLU's own backward holds anyway) instead of the
            # SwiGLU output and redoes the elementwise pass in backward
            recipe = ("swiglu", gate_up) if _recompute_activations() else None
            return self.dense_4h_to_h(inter, recompute=recipe, residual=residual)
        inter = _BiasGeluFn.apply(gate_up, bias, self.gelu_tanh)
        return self.dense_4h_to_h(inter, residual=residual)


class ParallelAttention(nn.Module):
    """Self-attention with TP heads or Ulysses sequence parallelism, and zigzag context parallelism on its own or inside the Ulysses
    exchange (transformer.py:512-900, :641-654).

    ``AttnType.cross_attn`` (T5's decoder, transformer.py:585-620, 755-790): ``query`` on the hidden states and ``key_value`` on the
    encoder output (per head k | v), both column-parallel, no GQA; non-causal attention of the s_q queries over the s_k keys.  Its
    forward returns (out, bias, encoder_output): the encoder output comes back as the pass-through whose gradient the key_value
    dgrad absorbs (``_CrossKvFn``).  Tensor parallelism and Megatron-SP only: Ulysses and context parallelism are refused."""

    def __init__(self, config, layer_number, attention_type=AttnType.self_attn, attn_mask_type=AttnMaskType.padding,
                 tp_group=None, sp_group=None, cp_group=None, cp_ranks=None, use_ulysses=False, use_zigzag_cp=False,
                 params_dtype=torch.float32, device=None):
        super().__init__()
        if attention_type not in (AttnType.self_attn, AttnType.cross_attn):
            raise NotImplementedError("attention type %r is not supported" % (attention_type,))
        self.attention_type = attention_type
        if attention_type == AttnType.cross_attn:
            self._init_cross(config, layer_number, tp_group, sp_group, cp_group, use_ulysses, use_zigzag_cp, params_dtype, device)
            return
        self.use_cp = bool(use_zigzag_cp) or _size(cp_group) > 1
        self.cp_comm = cp_comm_mode()
        self.layer_number = max(1, layer_number)
        self.attn_mask_type = attn_mask_type
        self.tp_group, self.sp_group, self.cp_group = tp_group, sp_group, cp_group
        self.use_ulysses = use_ulysses and _size(sp_group) > 1
        world = _size(tp_group)
        self.hn = getattr(config, "kv_channels", None) or config.hidden_size // config.num_attention_heads
        n_heads = config.num_attention_heads
        n_groups = getattr(config, "num_query_groups", None) or n_heads
        assert n_heads % world == 0 and n_groups % world == 0, \
            "num_attention_heads / num_query_groups must be divisible by the tensor parallel size"   # :577-581
        if self.use_ulysses:
            assert n_heads % sp_group.size == 0, "num_attention_heads must be divisible by the Ulysses degree"  # :642
        self.np_local, self.ng_local = n_heads // world, n_groups // world
        self.r = self.np_local // self.ng_local
        # K/V heads of one rank at the attention call: after the Ulysses exchange ng/p, or n/p when K/V are replicated first
        self.kv_heads_attn = self.ng_local
        if self.use_ulysses:
            p = sp_group.size
            self.kv_heads_attn = (self.ng_local if self.ng_local % p == 0 else self.np_local) // p
        if self.use_ulysses and self.use_cp:
            _check_ulysses_cp(sp_group.size, _size(cp_group), self.kv_heads_attn * self.hn * 2)
        add_bias = bool(getattr(config, "add_bias_linear", False))       # GPT / BERT: biases on both projections (:600-640)
        self.query_key_value = ColumnParallelLinear(config.hidden_size, (n_heads + 2 * n_groups) * self.hn, config=config,
                                                    bias=add_bias, gather_output=False, tp_group=tp_group,
                                                    params_dtype=params_dtype, device=device)
        self.dense = RowParallelLinear(n_heads * self.hn, config.hidden_size, config=config, bias=add_bias, skip_bias_add=True,
                                       input_is_parallel=True, tp_group=tp_group, params_dtype=params_dtype, device=device)
        self.softmax_scale = 1.0 / math.sqrt(self.hn)
        self._identity_rope = {}
        # dropout on the attention probabilities (GPT / BERT: transformer.py:443-503), in training only, drawn by the attention library
        # under this layer's model-parallel RNG stream (random.py)
        self.attention_dropout = check_probability(getattr(config, "attention_dropout", 0.0), "attention_dropout")
        if self.attention_dropout > 0.0:
            if self.use_cp:
                raise NotImplementedError("attention-probability dropout with context parallelism is not supported")
            try:
                from ..arguments import get_args
                seed = int(getattr(get_args(), "seed", 0))
            except RuntimeError:
                seed = 0
            tp_rank = tp_group.rank_in_group() if _size(tp_group) > 1 else 0
            sp_rank = sp_group.rank_in_group() if self.use_ulysses else 0
            self._rng_name = ("attention", layer_number, tp_rank, sp_rank)
            self._rng_seed = model_parallel_seed(seed, layer_number, tp_rank, sp_rank)

    def _init_cross(self, config, layer_number, tp_group, sp_group, cp_group, use_ulysses, use_zigzag_cp, params_dtype, device):
        if use_ulysses and _size(sp_group) > 1:
            raise NotImplementedError("cross-attention under Ulysses sequence parallelism is not supported")
        if use_zigzag_cp or _size(cp_group) > 1:
            raise NotImplementedError("cross-attention under context parallelism is not supported")
        n_heads = config.num_attention_heads
        n_groups = getattr(config, "num_query_groups", None) or n_heads
        if n_groups != n_heads:
            raise NotImplementedError("cross-attention with grouped-query attention (num_query_groups %d != heads %d) is not supported"
                                      % (n_groups, n_heads))
        world = _size(tp_group)
        assert n_heads % world == 0, "num_attention_heads must be divisible by the tensor parallel size"
        self.use_cp, self.use_ulysses, self.cp_comm = False, False, "allgather"
        self.layer_number = max(1, layer_number)
        self.attn_mask_type = AttnMaskType.padding
        self.tp_group, self.sp_group, self.cp_group = tp_group, None, None
        self.hn = getattr(config, "kv_channels", None) or config.hidden_size // n_heads
        self.np_local = self.ng_local = self.kv_heads_attn = n_heads // world
        self.r = 1
        add_bias = bool(getattr(config, "add_bias_linear", False))
        self.query = ColumnParallelLinear(config.hidden_size, n_heads * self.hn, config=config, bias=add_bias, gather_output=False,
                                          skip_bias_add=True, tp_group=tp_group, params_dtype=params_dtype, device=device)
        self.key_value = ColumnParallelLinear(config.hidden_size, 2 * n_heads * self.hn, config=config, bias=add_bias, gather_output=False,
                                              skip_bias_add=True, tp_group=tp_group, params_dtype=params_dtype, device=device)
        self.dense = RowParallelLinear(n_heads * self.hn, config.hidden_size, config=config, bias=add_bias, skip_bias_add=True,
                                       input_is_parallel=True, tp_group=tp_group, params_dtype=params_dtype, device=device)
        self.softmax_scale = 1.0 / math.sqrt(self.hn)
        self.attention_dropout = check_probability(getattr(config, "attention_dropout", 0.0), "attention_dropout")
        if self.attention_dropout > 0.0:
            raise NotImplementedError("attention-probability dropout in cross-attention is not supported")

    def _cross_forward(self, hidden_states, encoder_output, residual):
        """-> (out, bias, encoder_output pass-through) of cross-attention: queries from ``hidden_states`` [s_q(/t), b, h], keys and
        values from ``encoder_output`` [s_k(/t), b, h] (Megatron-SP: both sequence-split)."""
        if encoder_output is None:
            raise ValueError("cross-attention needs encoder_output")
        q_mixed, q_bias = self.query(hidden_states)                                        # [s_q, b, np * hn]
        kv_mixed, enc_out = _CrossKvFn.apply(encoder_output, self.key_value.weight, self.key_value.sequence_parallel, self.tp_group)
        q, k, v = _CrossQkvFn.apply(q_mixed, q_bias, kv_mixed, self.key_value.bias, self.np_local, self.hn)
        ctxt = _attention(q, k, v, False, self.softmax_scale)                              # [b, s_q, np, hn]
        b, s = ctxt.shape[0], ctxt.shape[1]
        ctxt = ctxt.reshape(b, s, -1).transpose(0, 1).contiguous()
        out, bias = self.dense(ctxt, residual=residual)
        return out, bias, enc_out

    def _core_attention(self, q, k, v, causal, key_mask):
        if not (self.attention_dropout > 0.0 and self.training):
            return _attention(q, k, v, causal, self.softmax_scale, key_mask)
        with get_rng_tracker().fork(self._rng_name, self._rng_seed, q.device):
            return _attention(q, k, v, causal, self.softmax_scale, key_mask, self.attention_dropout)

    def _no_rope(self, seq, device):
        """Families with learned absolute positions (GPT, BERT) run the same split + relayout kernel with cos = 1, sin = 0."""
        key = (seq, str(device))
        if key not in self._identity_rope:
            self._identity_rope[key] = (torch.ones(seq, self.hn // 2, dtype=torch.float32, device=device),
                                        torch.zeros(seq, self.hn // 2, dtype=torch.float32, device=device))
        return self._identity_rope[key]

    def forward(self, hidden_states, attention_mask=None, encoder_output=None, inference_params=None, rotary_pos_emb=None,
                input_recipe=None, residual=None):
        # hidden_states [sq, b, h]; rotary_pos_emb = (cos, sin) fp32 tables [sq_local, hn/2] for this rank's positions
        if self.attention_type == AttnType.cross_attn:
            return self._cross_forward(hidden_states, encoder_output, residual)
        mixed, _ = self.query_key_value(hidden_states, recompute=input_recipe)   # [s, b, ng*(r+2)*hn]
        cos, sin = rotary_pos_emb if rotary_pos_emb is not None else self._no_rope(mixed.shape[0], mixed.device)
        stage_group = self.sp_group if self.use_ulysses else None
        q, k, v = _QkvRopeFn.apply(mixed, cos, sin, self.ng_local, self.r, self.hn, stage_group)
        causal = self.attn_mask_type == AttnMaskType.causal
        # padding mask (BERT): [b, s] bool over the keys, True = attend (the reference builds the extended [b,1,1,s] additive
        # mask in bert_hf/BertModel_sequential.py and hands it to every layer)
        key_mask = attention_mask if (not causal and attention_mask is not None) else None
        if self.use_cp:
            assert causal, "context parallelism is implemented for causal self-attention"
        if self.use_ulysses and self.use_cp:
            ctxt = ulysses_cp_attention(q, k, v, self.sp_group, self.cp_group, self.softmax_scale, self.cp_comm)   # [b, s/(c*p), n, hn]
        elif self.use_ulysses:
            q, k, v = _ulysses_to_heads(q, k, v, self.sp_group)              # [b, s, n/p, hn]
            ctxt = self._core_attention(q, k, v, causal, key_mask)
            (ctxt,) = _UlyssesFn.apply(self.sp_group, False, ctxt)         # [b, s/p, n, hn]
        elif self.use_cp:
            ctxt = cp_attention(q, k, v, self.cp_group, self.softmax_scale, self.cp_comm)   # [b, s/c, np, hn]
        else:
            ctxt = self._core_attention(q, k, v, causal, key_mask)          # [b, s, np, hn]
        b, s = ctxt.shape[0], ctxt.shape[1]
        ctxt = ctxt.reshape(b, s, -1).transpose(0, 1).contiguous()          # "b s h d -> s b (h d)"
        return self.dense(ctxt, residual=residual)

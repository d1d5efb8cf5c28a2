"""CPU backend for the host runtime: torch ops + torch.distributed(gloo) collectives (TEST INFRASTRUCTURE ONLY).

Installed with ``hetu_galvatron_b200.core.runtime.backend.set_backend(OracleBackend())`` by tests/ (host-logic tests of the
schedules, sharded units, TP/SP/Ulysses layers at world_size 1-4 over gloo) and by bench.py's reference arm (the CPU
restatement of the reference path, BASELINE.md section 3).  The product never imports this module.

Each method restates the reference semantics of the op it stands for, with the reference's rounding points:
  * unit_reduce   : torch/distributed/fsdp/_runtime_utils.py:852-924 (prediv in reduce dtype, reduce-scatter, postdiv, cast, +=)
  * unit_unshard  : torch/distributed/fsdp/_flat_param.py:1477 (all-gather of the param-dtype shard)
  * all_reduce... : megatron/core/tensor_parallel/mappings_group.py:11-122
  * ulysses       : galvatron/core/runtime/tensor_parallel/transformer.py:1928-1987
  * math          : oracle/llama_ref.py conventions (fp32 compute, one rounding to the storage dtype)
"""
import math

import torch
import torch.distributed as dist
import torch.nn.functional as F


class _Buf:
    def __init__(self, nbytes):
        self.nbytes = (int(nbytes) + 255) // 256 * 256
        self.u8 = torch.zeros(self.nbytes, dtype=torch.uint8)
        self.offsets = None

    def view(self, dtype, numel=None):
        t = self.u8.view(dtype)
        return t if numel is None else t[:numel]


class _Link:
    """Blocking gloo send/recv between neighbouring stages (pipeline.py:1095-1127 semantics)."""

    def __init__(self, peer):
        self.peer = peer
        self._inflight = []

    def send(self, tensors):
        # non-blocking, like the product's side-stream peer copy: a blocking send here would deadlock 1F1B
        # (the reference pairs send/recv in one batch_isend_irecv for the same reason, pipeline.py:1095-1127)
        self._inflight = [(r, t) for r, t in self._inflight if not r.is_completed()]
        for t in tensors:
            t = t.detach().contiguous()
            self._inflight.append((dist.isend(t, dst=self.peer), t))

    def recv(self, shapes, dtypes, requires_grad):
        outs = []
        for shape, dtype in zip(shapes, dtypes):
            t = torch.empty(*shape, dtype=dtype)
            dist.recv(t, src=self.peer)
            if requires_grad and t.is_floating_point():
                t.requires_grad_(True)
            outs.append(t)
        return outs


class OracleBackend:
    name = "oracle-cpu-gloo"
    is_cuda = False

    def __init__(self):
        self.device = torch.device("cpu")
        self.rank = dist.get_rank() if dist.is_initialized() else 0
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self._pgs = {}
        self._staging = {}
        self.world_group = None
        if self.world > 1:
            # every arithmetic-progression subgroup, created in the same order on all ranks (new_group is collective)
            for stride in range(1, self.world):
                for size in range(2, self.world + 1):
                    for first in range(0, self.world - (size - 1) * stride):
                        ranks = tuple(range(first, first + size * stride, stride))
                        self._pgs[ranks] = dist.new_group(list(ranks), backend="gloo")
        self.launches = 0

    def close(self):
        pass

    def _pg(self, group):
        return self._pgs[tuple(group.ranks)]

    # ---- memory ---------------------------------------------------------------------------------------------------------
    def sym_alloc(self, group, nbytes):
        return _Buf(nbytes)

    def exchange(self):
        pass

    def reserve_staging(self, group, nbytes):
        return None

    # ---- sharded units ---------------------------------------------------------------------------------------------------
    def begin_step(self):
        pass

    def finish_reductions(self):
        pass

    def reserve_checkpoint_gather(self, group, nbytes):
        pass

    supports_tied_embedding_exchange = True     # all_reduce works over any rank list (the embedding group: first + last stage)

    def gather_master(self, unit):
        if unit.dp_type == "ddp" or unit.group.size == 1:
            return unit.flat_param.data
        full = torch.empty(unit.padded, dtype=torch.float32)
        dist.all_gather_into_tensor(full, unit.flat_param.data.contiguous(), group=self._pg(unit.group))
        return full

    def barrier_all(self):
        if dist.is_initialized():
            dist.barrier()

    def record_event(self):
        return None

    def reduce_done_event(self):
        return None

    def wait_event(self, ev):
        pass

    def unit_unshard(self, unit):
        shard = unit.flat_param.data.to(unit.param_dtype)
        if unit.dp_type == "ddp" or unit.group.size == 1:
            unit.w_flat.copy_(shard)
        else:
            dist.all_gather_into_tensor(unit.w_flat, shard.contiguous(), group=self._pg(unit.group))

    def unit_wait_unshard(self, unit):
        pass

    def unit_reduce(self, unit, accumulate):
        g = unit.g_flat
        n = unit.group.size
        g = (g / unit.prediv).to(unit.reduce_dtype)                       # _runtime_utils.py:852
        if n > 1:
            g = g.clone()
            dist.all_reduce(g, group=self._pg(unit.group))               # :858 (reduce-scatter == all-reduce + own slice)
            if unit.dp_type != "ddp":
                r = unit.group.rank_in_group(self.rank)
                g = g[r * unit.shard_elems:(r + 1) * unit.shard_elems]
        g = (g / unit.postdiv).to(unit.reduce_dtype).float()             # :879, :917 cast to the param (master) dtype
        if accumulate:
            unit.master_grad.add_(g)                                     # :924
        else:
            unit.master_grad.copy_(g)

    def unit_reduce_adamw(self, unit, opt):
        """reduce (reference rounding points) then torch.optim.AdamW's update rule on the fp32 shard."""
        self.unit_reduce(unit, accumulate=False)
        lr, b1, b2, eps, wd, step = opt.hyper()
        g, p = unit.master_grad, unit.flat_param.data
        p.mul_(1 - lr * wd)
        unit.exp_avg.mul_(b1).add_(g, alpha=1 - b1)
        unit.exp_avg_sq.mul_(b2).addcmul_(g, g, value=1 - b2)
        denom = (unit.exp_avg_sq.sqrt() / math.sqrt(1 - b2 ** step)).add_(eps)
        p.addcdiv_(unit.exp_avg, denom, value=-lr / (1 - b1 ** step))

    def make_stage_link(self, my_rank, peer_rank, max_bytes, send_flag_base, recv_flag_base):
        return _Link(peer_rank)

    # ---- activation collectives -----------------------------------------------------------------------------------------------
    def all_reduce(self, x, group, op="sum"):
        if group is None or group.size == 1:
            return x
        out = x.contiguous().clone()
        dist.all_reduce(out, op=dist.ReduceOp.MAX if op == "max" else dist.ReduceOp.SUM, group=self._pg(group))
        return out

    def all_gather_first_dim(self, x, group):
        if group is None or group.size == 1:
            return x
        x = x.contiguous()
        out = torch.empty((group.size * x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype)
        dist.all_gather_into_tensor(out, x, group=self._pg(group))
        return out

    all_gather_into_staging = all_gather_first_dim

    def reduce_scatter_first_dim(self, x, group):
        if group is None or group.size == 1:
            return x
        full = self.all_reduce(x, group)
        n, r = group.size, group.rank_in_group(self.rank)
        loc = x.shape[0] // n
        return full[r * loc:(r + 1) * loc].contiguous()

    def all_gather_last_dim(self, x, group):
        if group is None or group.size == 1:
            return x
        g = self.all_gather_first_dim(x.contiguous().unsqueeze(0), group)
        return torch.cat([g[i] for i in range(group.size)], dim=-1).contiguous()

    def ulysses_all_to_all(self, tensors, group, to_heads):
        p = group.size
        if p == 1:
            return list(tensors)
        r = group.rank_in_group(self.rank)
        outs = []
        for t in tensors:
            allt = self.all_gather_first_dim(t.contiguous().unsqueeze(0), group)      # [p, b, s, n, d]
            if to_heads:   # [b, s/p, n, d] -> [b, s, n/p, d]: my head slice of every rank's sequence slice
                hp = t.shape[2] // p
                outs.append(torch.cat([allt[q][:, :, r * hp:(r + 1) * hp] for q in range(p)], dim=1).contiguous())
            else:          # [b, s, n/p, d] -> [b, s/p, n, d]: my sequence slice of every rank's head slice
                sl = t.shape[1] // p
                outs.append(torch.cat([allt[q][:, r * sl:(r + 1) * sl] for q in range(p)], dim=2).contiguous())
        return outs

    # ---- GEMM + collective: the GEMM, then the collective (megatron/core/tensor_parallel/layers.py:399-417, :462, :488-494) ---------
    def fuses(self, kind, m, n, k, group):
        return False

    def gemm_reduce_scatter(self, a, b, layout, group):
        return self.reduce_scatter_first_dim(self.gemm(a, b, layout), group)

    def gemm_all_reduce(self, a, b, layout, group):
        return self.all_reduce(self.gemm(a, b, layout), group)

    def all_gather_gemm(self, a_local, b, layout, group):
        gathered = self.all_gather_first_dim(a_local, group)
        return self.gemm(gathered, b, layout), gathered

    # ---- math -------------------------------------------------------------------------------------------------------------------
    def gemm(self, a, b, layout, out=None, accumulate=False, addend=None):
        self.launches += 1
        af = a.float().t() if layout == "nt" else a.float()
        bf = b.float().t() if layout == "tn" else b.float()
        res = af @ bf
        if addend is not None:      # the residual add in the GEMM epilogue: fp32 accumulator + addend, one rounding
            res = res + addend.float().reshape(res.shape)
        if out is None:
            return res.to(a.dtype)
        out.copy_((res + out.float()).to(out.dtype) if accumulate else res.to(out.dtype))
        return out

    def rmsnorm_fwd(self, x, weight, eps):
        xf = x.float()
        rstd = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
        return (xf * rstd * weight.float()).to(x.dtype), rstd.reshape(-1)

    def rmsnorm_bwd(self, dy, x, weight, rstd):
        xf, g = x.float(), dy.float()
        r = rstd.view(*x.shape[:-1], 1)
        xh = xf * r
        gw = g * weight.float()
        dx = r * (gw - xh * (gw * xh).mean(-1, keepdim=True))
        dw = (g * xh).reshape(-1, x.shape[-1]).sum(0)
        return dx.to(x.dtype), dw.to(weight.dtype)

    def layernorm_fwd(self, x, weight, bias, eps):
        xf = x.float()
        mean = xf.mean(-1, keepdim=True)
        rstd = torch.rsqrt((xf - mean).pow(2).mean(-1, keepdim=True) + eps)
        return ((xf - mean) * rstd * weight.float() + bias.float()).to(x.dtype), mean.reshape(-1), rstd.reshape(-1)

    def layernorm_bwd(self, dy, x, weight, mean, rstd):
        xf, g = x.float(), dy.float()
        m, r = mean.view(*x.shape[:-1], 1), rstd.view(*x.shape[:-1], 1)
        xh = (xf - m) * r
        gw = g * weight.float()
        dx = r * (gw - gw.mean(-1, keepdim=True) - xh * (gw * xh).mean(-1, keepdim=True))
        return dx.to(x.dtype), (g * xh).reshape(-1, x.shape[-1]).sum(0).to(weight.dtype), g.reshape(-1, x.shape[-1]).sum(0).to(weight.dtype)

    @staticmethod
    def _gelu(v, tanh_form):
        return F.gelu(v, approximate="tanh" if tanh_form else "none")

    def bias_gelu_fwd(self, x, bias, tanh_form=True):
        v = x.float() if bias is None else x.float() + bias.float()
        return self._gelu(v, tanh_form).to(x.dtype)

    def bias_gelu_bwd(self, dy, x, bias, tanh_form=True):
        v = (x.float() if bias is None else x.float() + bias.float()).detach().requires_grad_(True)
        with torch.enable_grad():
            y = self._gelu(v, tanh_form)
        (dv,) = torch.autograd.grad(y, v, dy.float())
        return dv.to(x.dtype)

    def swiglu_fwd(self, gate_up):
        g, u = torch.chunk(gate_up.float(), 2, dim=-1)
        return (F.silu(g) * u).to(gate_up.dtype)

    def swiglu_bwd(self, dy, gate_up):
        g, u = torch.chunk(gate_up.float(), 2, dim=-1)
        d = dy.float()
        sg = torch.sigmoid(g)
        return torch.cat([d * u * sg * (1 + g * (1 - sg)), d * g * sg], dim=-1).to(gate_up.dtype)

    def rope_tables(self, seq_len, head_dim, base, offset, dtype, device):
        inv_freq = 1.0 / (base ** (torch.arange(0, head_dim, 2, dtype=torch.float32) / head_dim))
        freqs = torch.outer(torch.arange(seq_len, dtype=torch.float32) + offset, inv_freq)
        return torch.cos(freqs).to(dtype).float().contiguous(), torch.sin(freqs).to(dtype).float().contiguous()

    @staticmethod
    def _rot(x, cos, sin, inverse):
        half = x.shape[-1] // 2
        lo, hi = x[..., :half].float(), x[..., half:].float()
        c, s = cos[:, None, None, :], (-sin if inverse else sin)[:, None, None, :]
        return torch.cat([lo * c - hi * s, hi * c + lo * s], dim=-1)

    def qkv_rope_fwd(self, mixed, cos, sin, ng, r, hn, stage_group=None):
        s, b = mixed.shape[:2]
        m = mixed.view(s, b, ng, (r + 2) * hn)
        q, k, v = torch.split(m, [r * hn, hn, hn], dim=3)
        q = self._rot(q.reshape(s, b, ng * r, hn), cos, sin, False).to(mixed.dtype)
        k = self._rot(k, cos, sin, False).to(mixed.dtype)
        return [t.permute(1, 0, 2, 3).contiguous() for t in (q, k, v)]

    def qkv_rope_bwd(self, dq, dk, dv, cos, sin, ng, r, hn):
        b, s = dq.shape[:2]
        dq, dk, dv = [t.permute(1, 0, 2, 3) for t in (dq, dk, dv)]                       # [s, b, heads, hn]
        dq = self._rot(dq, cos, sin, True).reshape(s, b, ng, r * hn)
        dk = self._rot(dk, cos, sin, True)
        return torch.cat([dq, dk, dv.float()], dim=3).reshape(s, b, ng * (r + 2) * hn).to(dv.dtype)

    def attention_prefix(self, q, k, v, softmax_scale):
        """query i attends keys j <= i + (sk - sq) (bottom-right aligned causal mask); plain differentiable torch math."""
        rep = q.shape[2] // k.shape[2]
        qf, kf, vf = q.float(), k.float().repeat_interleave(rep, 2), v.float().repeat_interleave(rep, 2)
        qf, kf, vf = [t.transpose(1, 2) for t in (qf, kf, vf)]
        sq, sk = qf.shape[-2], kf.shape[-2]
        scores = qf @ kf.transpose(-1, -2) * softmax_scale
        mask = torch.arange(sk)[None, :] > (torch.arange(sq)[:, None] + (sk - sq))
        p = torch.softmax(scores.masked_fill(mask, float("-inf")), -1)
        return (p @ vf).transpose(1, 2).contiguous().to(q.dtype)

    def attention_fwd(self, q, k, v, causal, softmax_scale, key_mask=None):
        rep = q.shape[2] // k.shape[2]
        qf, kf, vf = q.float(), k.float().repeat_interleave(rep, 2), v.float().repeat_interleave(rep, 2)
        qf, kf, vf = [t.transpose(1, 2) for t in (qf, kf, vf)]                          # [b, n, s, d]
        scores = qf @ kf.transpose(-1, -2) * softmax_scale
        if key_mask is not None:      # padding mask: key j of sample b is visible iff key_mask[b, j]
            scores = scores.masked_fill(~key_mask.bool()[:, None, None, :], float("-inf"))
        if causal:
            s = scores.shape[-1]
            scores = scores.masked_fill(torch.triu(torch.ones(s, s, dtype=torch.bool), 1), float("-inf"))
        p = torch.softmax(scores, -1)
        return (p @ vf).transpose(1, 2).contiguous().to(q.dtype), p, None

    def attention_bwd(self, dout, q, k, v, out, p, causal, softmax_scale, rng):
        rep = q.shape[2] // k.shape[2]
        b, s, ng, d = k.shape
        qf, kf, vf = q.float(), k.float().repeat_interleave(rep, 2), v.float().repeat_interleave(rep, 2)
        qf, kf, vf, do = [t.transpose(1, 2) for t in (qf, kf, vf, dout.float())]
        dv = p.transpose(-1, -2) @ do
        dp = do @ vf.transpose(-1, -2)
        ds = p * (dp - (dp * p).sum(-1, keepdim=True)) * softmax_scale
        dq = (ds @ kf).transpose(1, 2)
        dk = (ds.transpose(-1, -2) @ qf).transpose(1, 2).reshape(b, s, ng, rep, d).sum(3)
        dv = dv.transpose(1, 2).reshape(b, s, ng, rep, d).sum(3)
        return dq.contiguous().to(q.dtype), dk.contiguous().to(k.dtype), dv.contiguous().to(v.dtype)

    def ce_fwd(self, logits2d, target, vocab_start, tp_group):
        lf = logits2d.float()
        vl = lf.shape[1]
        rowmax = self.all_reduce(lf.max(-1).values, tp_group, op="max")
        ex = torch.exp(lf - rowmax[:, None])
        t = target - vocab_start
        inside = (t >= 0) & (t < vl)
        pred = torch.where(inside, lf.gather(1, t.clamp(0, vl - 1)[:, None]).squeeze(1) - rowmax, torch.zeros_like(rowmax))
        out2 = self.all_reduce(torch.stack([ex.sum(-1), pred], dim=1).contiguous(), tp_group)
        return torch.log(out2[:, 0]) - out2[:, 1], rowmax, out2

    def ce_bwd(self, logits2d, target, rowmax, sum2, grad_loss, vocab_start):
        lf = logits2d.float()
        vl = lf.shape[1]
        p = torch.exp(lf - rowmax[:, None]) / sum2[:, :1]
        t = target - vocab_start
        inside = (t >= 0) & (t < vl)
        onehot = torch.zeros_like(p)
        onehot[inside, t[inside]] = 1.0
        logits2d.copy_(((p - onehot) * grad_loss[:, None]).to(logits2d.dtype))
        return logits2d

    def cast(self, src, dst, scale=1.0, accumulate=False):
        v = src.float() * scale
        dst.copy_((dst.float() + v).to(dst.dtype) if accumulate else v.to(dst.dtype))

    def launch_count(self):
        return 0

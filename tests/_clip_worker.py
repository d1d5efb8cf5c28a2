"""Worker for tests/test_clip_fused.py and tests/test_gpu_clip.py: one rank of a tiny-Llama job that trains a few steps with
gradient clipping by the global norm.

``_arm`` picks the optimizer:
  "fused_clip"  FusedShardedAdamW with ``clip_grad`` (deferred update) + ``clip_grad_norm(model, _max_norm)`` every step
  "torch_clip"  torch.optim.AdamW over the fp32 gradients + the same ``clip_grad_norm`` calls
  "fused_defer" FusedShardedAdamW with ``clip_grad`` but no ``clip_grad_norm`` call (an unclipped deferred update)
  "fused"       FusedShardedAdamW without ``clip_grad`` (the update inside the reduce-scatter)
  "torch"       torch.optim.AdamW, no clipping
  "fused_norm" / "torch_norm"  the unclipped pair that still measures the norm: "fused_defer" / "torch" + clip_grad_norm(model, inf)
Every rank writes its fp32 master shards after the last step to ``<_dump>.rank<r>``; rank 0 reports the per-step norms, the losses,
the single-process oracle's step-0 norm (clipping arms), the units still holding an fp32 gradient buffer, and the fused-kernel
counters (CUDA).  On the CPU the gloo oracle backend gets the deferred-clipping methods from ``ClipOracleBackend`` below."""
import json
import math
import os
import sys
import traceback

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.gloo_backend import OracleBackend  # noqa: E402


class ClipOracleBackend(OracleBackend):
    """The CPU restatement of deferred clipping's backend methods: the reduction with the reference's rounding points (as
    ``OracleBackend.unit_reduce``), the squares summed in fp32 as ``clip_grad_norm`` sums them, and torch.optim.AdamW's operation
    order -- so that the deferred arm and the torch arm differ only by the order of the final sum of squares.  (Clipped to a small
    norm, Adam normalises per-element gradients of ~1e-4: one fp32 ulp in a master flips bf16 weights and the runs drift apart.)"""

    def __init__(self):
        super().__init__()
        self.n_fused = {}

    def _count(self, key):
        self.n_fused[key] = self.n_fused.get(key, 0) + 1

    def _reduced(self, unit):
        g = (unit.g_flat / unit.prediv).to(unit.reduce_dtype)
        if unit.group.size > 1:
            g = g.clone()
            dist.all_reduce(g, group=self._pg(unit.group))
            if unit.dp_type != "ddp":
                r = unit.group.rank_in_group(self.rank)
                g = g[r * unit.shard_elems:(r + 1) * unit.shard_elems]
        return (g / unit.postdiv).to(unit.reduce_dtype).float()

    def _adamw(self, unit, opt, g, clip_coef):
        lr, b1, b2, eps, wd, step = opt.hyper()
        g = g * clip_coef
        p = unit.flat_param.data
        p.mul_(1 - lr * wd)
        unit.exp_avg.lerp_(g, 1 - b1)
        unit.exp_avg_sq.mul_(b2).addcmul_(g, g, value=1 - b2)
        denom = (unit.exp_avg_sq.sqrt() / math.sqrt(1 - b2 ** step)).add_(eps)
        p.addcdiv_(unit.exp_avg, denom, value=-lr / (1 - b1 ** step))

    def clip_partials(self, n_units):
        return torch.zeros(n_units, 1)

    def unit_reduce_sumsq(self, unit, partials, skip, into_master=False):
        g = self._reduced(unit)
        sq = g.pow(2).sum()
        for lo, hi in skip:
            sq = sq - g[lo:hi].pow(2).sum()
        partials.zero_()
        partials[0] = sq
        if into_master:
            unit.master_grad.copy_(g)
        self._count("rs_sumsq")

    def unit_reduce_adamw(self, unit, opt, clip_coef=None):
        self._adamw(unit, opt, self._reduced(unit), 1.0 if clip_coef is None else clip_coef)
        if clip_coef is not None:
            self._count("rs_adamw_clipped")

    def unit_adamw_clipped(self, unit, opt, clip_coef):
        self._adamw(unit, opt, unit.master_grad, clip_coef)
        self._count("adamw_clipped")


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    over = json.loads(os.environ["HOST_TEST_CONFIG"])
    arm, max_norm, steps, dump = over.pop("_arm"), over.pop("_max_norm", 0.05), over.pop("_steps", 3), over.pop("_dump")
    use_cuda = os.environ.get("HOST_TEST_BACKEND", "oracle") == "cuda"
    from oracle import llama_ref
    import smoke_model as sm
    from _host_worker import assemble_full
    from hetu_galvatron_b200.core.runtime.backend import get_backend, set_backend
    from hetu_galvatron_b200.core.runtime.utils import clip_grad_norm, get_optimizer_and_param_scheduler
    if use_cuda:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", torch.cuda.current_device()))
        os.environ.setdefault("HGB_ARENA_BYTES", str(256 << 20))
        be = get_backend()
        be.bg.set_tunable("timeout_ms", 30000)
        dev = be.device
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.set_num_threads(1 if world >= 4 else 2)
        be = set_backend(ClipOracleBackend())
        dev = torch.device("cpu")
    clipping = arm in ("fused_clip", "torch_clip", "fused_norm", "torch_norm")
    if arm.endswith("_norm"):
        max_norm = float("inf")            # coefficient min(1, inf) = 1: the norm is measured, the update is not clipped
    over["fused_optimizer"] = arm.startswith("fused")
    if arm in ("fused_clip", "fused_defer", "fused_norm"):
        over["clip_grad"] = 1.0 if arm == "fused_norm" else max_norm
    args = sm.tiny_args(**over)
    config, model = sm.build(args)
    opt, _ = get_optimizer_and_param_scheduler(model, args)
    w = assemble_full(model, config, world, rank, lambda u: u.read_full_params()) if clipping else None
    gbs, seq = args.global_train_batch_size, config.max_position_embeddings
    dp_group = model.vtp_data_group
    dp_idx, dp = dp_group.rank_in_group(rank), dp_group.size
    g = torch.Generator().manual_seed(11)
    report = {"norms": [], "losses": []}
    for it in range(steps):
        x = torch.randint(0, config.vocab_size, (gbs, seq + 1), generator=g)
        tokens, labels = x[:, :-1].contiguous(), x[:, 1:].contiguous()
        lo, hi = dp_idx * gbs // dp, (dp_idx + 1) * gbs // dp
        loss = model.forward_backward([tokens[lo:hi].to(dev)], it, None, loss_func=None, attention_mask=None,
                                      labels=labels[lo:hi].to(dev))
        if clipping:
            report["norms"].append(clip_grad_norm(model, max_norm))
            if it == 0:   # the un-parallelised model's gradient norm on the global batch
                cfg = sm.oracle_cfg(config, args)
                leaves = [w["embed"], w["norm"], w["lm_head"]] + [t for lw in w["layers"] for t in lw.values()]
                for t in leaves:
                    t.requires_grad_(True)
                _, ref_loss = llama_ref.forward_loss(w, tokens, labels, cfg, dtype=torch.bfloat16)
                ref_loss.backward()
                report["oracle_norm0"] = float(torch.sqrt(sum(t.grad.float().pow(2).sum() for t in leaves)))
        lt = torch.tensor([loss if loss is not None else 0.0, 1.0 if loss is not None else 0.0], dtype=torch.float64, device=dev)
        dist.all_reduce(lt)
        report["losses"].append(float(lt[0] / lt[1]))
        opt.step()
        opt.zero_grad()
        if use_cuda:
            torch.cuda.synchronize()
            assert be.comm.error_flag() == 0
    torch.save({u.name: u.flat_param.data.detach().cpu().clone() for u in model.model.units}, "%s.rank%d" % (dump, rank))
    # units holding an fp32 gradient buffer, and whether each is one that has to (pooled zero3 / replicated DDP layers)
    mine = [[u.name, u.g_pool is not None or not u.uses_fused_optimizer()] for u in model.model.units if u._master_grad is not None]
    held = [None] * world
    dist.all_gather_object(held, mine)
    report["fp32_grad_units"] = [rec for per_rank in held for rec in per_rank]
    report["fused_calls"] = dict(getattr(be, "n_fused", {}))
    if rank == 0:
        print("HOST_TEST_REPORT " + json.dumps(report), flush=True)
    dist.barrier()
    if use_cuda:
        from hetu_galvatron_b200.core.runtime.backend import reset_backend
        reset_backend()
    dist.destroy_process_group()
    return report


if __name__ == "__main__":
    try:
        main()
    except Exception:
        traceback.print_exc()
        sys.exit(1)

"""The flagship workload (bench.py's model, strategy and synthetic batches: Llama-3.2-1B shapes, seq 8192, one GPU) trained with and
without gradient clipping by the global norm, three arms alternated in one call, each run in a fresh process:
  fused       the fused optimizer, no clipping (bench.py's headline configuration)
  fused_clip  the fused optimizer built with clip_grad = 1.0 + clip_grad_norm(model, 1.0) every step (deferred update)
  torch_clip  torch.optim.AdamW(fused=True) over fp32 gradient shards + clip_grad_norm(model, 1.0) every step
Prints one JSON line per run (tokens/s, ms per step, torch.cuda.max_memory_allocated, the norms) and the card's name, power limit
and max SM clock.  Usage: python scripts/bench_clip.py [--steps K] [--warmup W] [--runs R]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARMS = ("fused", "fused_clip", "torch_clip")


def child(arm, steps, warmup):
    os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")
    import types
    import torch
    sys.path.insert(0, ROOT)
    import bench
    from hetu_galvatron_b200.core.runtime.backend import get_backend
    from hetu_galvatron_b200.core.runtime.utils import clip_grad_norm, get_optimizer_and_param_scheduler
    opts = types.SimpleNamespace(model=bench.MODEL, seq=bench.SEQ, layers=0, checkpoint_layers=-1,
                                 optimizer="torch" if arm == "torch_clip" else "fused")
    _, strategy = bench.strategy_for(1, opts.model, None)
    args, config, model = bench.build_model(opts, strategy)
    if arm == "fused_clip":
        args.clip_grad = 1.0
    opt, _ = get_optimizer_and_param_scheduler(model, args)
    batches = bench.synthetic_batches(args, config, warmup + steps, 0, 1, pin=True)
    dev = torch.device("cuda", torch.cuda.current_device())
    norms = []

    def step(it):
        tokens, labels = batches[it]
        model.forward_backward([tokens.to(dev, non_blocking=True)], it, None, loss_func=None, attention_mask=None,
                               labels=labels.to(dev, non_blocking=True))
        if arm != "fused":
            norms.append(clip_grad_norm(model, 1.0))
        opt.step()
        opt.zero_grad()

    for it in range(warmup):
        step(it)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for it in range(warmup, warmup + steps):
        step(it)
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / steps
    tokens = args.global_train_batch_size * config.max_position_embeddings
    print("CLIP_BENCH " + json.dumps({"arm": arm, "tokens_per_s": round(tokens / dt, 1), "ms_per_step": round(dt * 1e3, 2),
                                      "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                                      "norms": [round(n, 5) for n in norms], "fused_calls": dict(get_backend().n_fused)}), flush=True)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=4)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--runs", type=int, default=3)
    p.add_argument("--arm", default=None, help="internal: run one arm in this process")
    a = p.parse_args()
    if a.arm:
        return child(a.arm, a.steps, a.warmup)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"nvidia_smi": q.stdout.strip()}), flush=True)
    results = {arm: [] for arm in ARMS}
    for _ in range(a.runs):
        for arm in ARMS:
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--arm", arm, "--steps", str(a.steps), "--warmup", str(a.warmup)],
                                 capture_output=True, text=True, cwd=ROOT)
            lines = [ln for ln in out.stdout.splitlines() if ln.startswith("CLIP_BENCH ")]
            if out.returncode != 0 or not lines:
                print(json.dumps({"arm": arm, "error": (out.stdout + out.stderr)[-2000:]}), flush=True)
                continue
            rec = json.loads(lines[-1][len("CLIP_BENCH "):])
            results[arm].append(rec)
            print(json.dumps(rec), flush=True)
    summary = {arm: {"tokens_per_s": sorted(r["tokens_per_s"] for r in recs), "max_memory_allocated_gib": sorted(r["max_memory_allocated_gib"] for r in recs)}
               for arm, recs in results.items()}
    print(json.dumps({"summary": summary}), flush=True)


if __name__ == "__main__":
    main()

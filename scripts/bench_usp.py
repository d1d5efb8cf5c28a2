"""Ulysses x context parallelism on one layer, per rank, on one GPU: Llama-3.2-1B attention shapes (32 heads, 8 KV heads of 64),
microbatch 1, S in {32k, 128k}, (sp, cp) in {(8, 1), (4, 2), (2, 4), (1, 8)} -- the four ways to split the sequence 8 ways.

For each point, JSON lines with:
* the attention forward + backward time of ONE rank on the heads and rows it holds after the Ulysses exchange (n/sp heads, S/cp
  rows): at cp 1 one causal flash-attn call; at cp > 1 the ring schedule of tensor_parallel/transformer.py (2cp-1 block calls, LSE
  merges, fp32 accumulation casts) and the all-gather path's two prefix calls on the gathered sequence.  Transport is excluded
  (the ring moves nothing; the gather is not timed), as in ``scripts/bench_kernels.py cp``.  Median of 3 interleaved windows.
* the K/V bytes one layer keeps for backward on a rank, per cp exchange;
* the all-to-all and cp-exchange bytes a rank sends per layer (forward + backward), from the shapes.
NVLink time and multi-GPU step time are not measured here.
Usage: python scripts/bench_usp.py  -> JSON lines on stdout."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

N_HEADS, N_KV, HEAD_DIM, BATCH = 32, 8, 64, 1
POINTS = [(8, 1), (4, 2), (2, 4), (1, 8)]


def bytes_per_rank(S, sp, cp, n=N_HEADS, ng=N_KV, d=HEAD_DIM, b=BATCH, esz=2):
    """-> dict of per-layer byte counts for one rank (forward + backward)"""
    kv_pre = ng if ng % sp == 0 else n                 # K/V heads entering the exchange (replicated when ng % sp != 0)
    kvh = kv_pre // sp                                 # ... and after it
    rows_in = S // (cp * sp)
    # to-heads exchange of q, k, v and the inverse one of the context, each sending (sp-1)/sp of its input; backward: the same again
    a2a = 2 * (sp - 1) / sp * rows_in * d * esz * (n + 2 * kv_pre + n) * b
    blk = b * (S // cp) * kvh * d                      # elements of one rank's K (or V) block
    ring = (cp - 1) * 2 * blk * esz + (cp - 1) * 2 * blk * esz + cp * 2 * blk * 4 if cp > 1 else 0   # fwd K/V, bwd K/V, bwd dK/dV fp32
    gather = 2 * (cp - 1) * 2 * blk * esz if cp > 1 else 0       # K/V all-gather forward, dK/dV reduce-scatter backward (bf16)
    return {"all_to_all_bytes": int(a2a), "ring_bytes": int(ring), "allgather_bytes": int(gather),
            "kv_kept_for_backward_ring": 2 * blk * esz, "kv_kept_for_backward_allgather": 2 * b * S * kvh * d * esz if cp > 1 else None,
            "kv_kept_for_backward_cp1": 2 * blk * esz if cp == 1 else None, "kv_heads_per_rank": kvh}


def main():
    from bench_kernels import _LocalRing, timeit
    from flash_attn import flash_attn_func
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend
    from hetu_galvatron_b200.core.runtime.tensor_parallel import transformer as tr
    if not torch.cuda.is_available():
        raise SystemExit("bench_usp.py measures on a GPU; there is none")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"nvidia_smi": q.stdout.strip()}), flush=True)
    be = CudaBackend(arena_bytes=1 << 24)
    BF = torch.bfloat16
    d, b = HEAD_DIM, BATCH
    scale = d ** -0.5
    for S in (32768, 131072):
        for sp, cp in POINTS:
            info = bytes_per_rank(S, sp, cp)
            nh, kvh, s = N_HEADS // sp, info["kv_heads_per_rank"], S // cp
            qq = torch.randn(b, s, nh, d, device="cuda").to(BF)
            k, v = [torch.randn(b, s, kvh, d, device="cuda").to(BF) for _ in range(2)]
            do = torch.randn(b, s, nh, d, device="cuda").to(BF)
            arms = {}
            if cp == 1:
                qg, kg, vg = [t.detach().clone().requires_grad_(True) for t in (qq, k, v)]
                arms["flash_ms"] = lambda: flash_attn_func(qg, kg, vg, softmax_scale=scale, causal=True).backward(do)
            else:
                ring = _LocalRing(cp, k, v)

                def ring_fb():
                    out, lse = tr.run_steps(tr.ring_attention_fwd(be, ring, qq, k, v, scale))
                    tr.run_steps(tr.ring_attention_bwd(be, ring, do, qq, k, v, out, lse, scale))
                kf, vf = [torch.randn(b, S, kvh, d, device="cuda").to(BF).requires_grad_(True) for _ in range(2)]
                qg = qq.detach().clone().requires_grad_(True)
                half = s // 2

                def gather_fb():
                    outs = [flash_attn_func(qg[:, q0:q0 + half], kf[:, :(ch + 1) * half], vf[:, :(ch + 1) * half], softmax_scale=scale,
                                            causal=True) for q0, ch in ((0, 0), (half, 2 * cp - 1))]      # cp rank 0's two chunks
                    torch.cat(outs, 1).backward(do)
                arms["ring_ms"], arms["allgather_ms"] = ring_fb, gather_fb
            iters = 3 if S > 32768 else 10
            times = {name: [] for name in arms}
            for _ in range(3):                           # interleaved windows
                for name, fn in arms.items():
                    times[name].append(timeit(fn, iters=iters, warm=1))
            allt = [t for ts in times.values() for t in ts]
            rec = {"bench": "usp_attention_fwd_bwd_per_rank", "S": S, "sp": sp, "cp": cp, "heads_per_rank": nh,
                   "rows_per_rank_at_attention": s, "transport": "excluded", "nvlink_time": "not measured",
                   "spread_pct": round(100 * (max(allt) - min(allt)) / min(allt), 1)}
            rec.update({name: round(sorted(ts)[1], 3) for name, ts in times.items()})
            rec.update({key: (round(val / 2 ** 20, 1) if isinstance(val, int) and key != "kv_heads_per_rank" else val)
                        for key, val in info.items()})
            rec["bytes_unit"] = "MiB"
            print(json.dumps(rec), flush=True)
            del qq, k, v, do, arms
            torch.cuda.empty_cache()
    be.close()


if __name__ == "__main__":
    main()

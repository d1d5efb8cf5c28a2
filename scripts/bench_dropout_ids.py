"""The dropout row kernels at an explicit sample map (bg_dropout_add_fwd_ids / bg_dropout_bwd_ids) against the sample_base ones
(bg_dropout_add_fwd / bg_dropout_bwd) on one GPU, at the rows of a gathered microbatch: GPT-2.7B (h 2560, seq 2048) and BERT-large
(h 1024, seq 512), two data-parallel ranks' microbatches of 4 and 16 samples.  The map is the two-run one a relocation produces with
chunks > 1.  The four arms alternate window by window on two input sets of > 50 MB each; CUDA events, median of the rounds.
Algorithmic bytes: forward reads x and the residual and writes y (6 B / element), backward reads dy and writes dx (4 B / element).
Usage: python scripts/bench_dropout_ids.py  -> JSON lines on stdout (the first one names the card and its power limit)."""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BF = torch.bfloat16


def main(rounds=7, iters=20, p=0.1):
    from hetu_galvatron_b200.core.runtime import world
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}), flush=True)
    world.get_rank()
    be = CudaBackend(arena_bytes=1 << 24)
    for name, s, mb, h in (("gpt_2.7b", 2048, 4, 2560), ("bert_large", 512, 16, 1024)):
        b = 2 * mb
        ids = torch.tensor([mb + i for i in range(mb)] + [3 * mb + i for i in range(mb)], dtype=torch.int32, device="cuda")
        base = 0
        sets = [tuple(torch.randn(s, b, h, device="cuda").to(BF) for _ in range(3)) + (torch.randn(h, device="cuda").to(BF),)
                for _ in range(2)]
        n = s * b * h
        arms = {
            "contiguous_fwd": lambda st: be.dropout_add_fwd(st[0], st[3], st[1], p, 1234, 7, 5, 0, base),
            "mapped_fwd": lambda st: be.dropout_add_fwd_ids(st[0], st[3], st[1], p, 1234, 7, 5, 0, ids),
            "contiguous_bwd": lambda st: be.dropout_bwd(st[2], p, 1234, 7, 5, 0, base, with_bias=True),
            "mapped_bwd": lambda st: be.dropout_bwd_ids(st[2], p, 1234, 7, 5, 0, ids, with_bias=True),
        }

        def window(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(iters):
                fn(sets[i % 2])
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / iters

        for fn in arms.values():
            window(fn)
        times = {k: [] for k in arms}
        for _ in range(rounds):
            for k, fn in arms.items():
                times[k].append(window(fn))
        rec = {"bench": "dropout_ids", "shape": name, "s": s, "b": b, "h": h, "p": p, "ids": "two runs"}
        for k, ts in times.items():
            t = sorted(ts)[rounds // 2]
            nbytes = (6 if k.endswith("fwd") else 4) * n
            rec[k + "_ms"] = round(t, 4)
            rec[k + "_GBps_algorithmic"] = round(nbytes / t / 1e6, 1)
            rec[k + "_spread_pct"] = round(100 * (max(ts) - min(ts)) / t, 1)
        for d in ("fwd", "bwd"):
            rec[d + "_mapped_over_contiguous"] = round(rec["mapped_%s_ms" % d] / rec["contiguous_%s_ms" % d], 3)
        print(json.dumps(rec), flush=True)
        del sets
        torch.cuda.empty_cache()
    be.close()


if __name__ == "__main__":
    main()

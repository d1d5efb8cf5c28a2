"""Micro-benchmarks of the C-ABI kernels on one GPU (CUDA events, warm-up, L2-exceeding inputs).
Usage: python scripts/bench_kernels.py [gemm] [cast] [ops] [attn] [dropout] [cp] [clip] [tied]  -> JSON lines on stdout.
       cp's head shape and sequence lengths: --cp-heads N --cp-kv-heads N --cp-head-dim N --cp-seqs S1,S2 (defaults: Llama-3.2-1B)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hetu_galvatron_b200 import _bg as bg  # noqa: E402

BF = torch.bfloat16


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


# The 15 GEMMs of one microbatch of the flagship workload (Llama-3.2-1B shapes, seq 8192): (layout, M, N, K, epilogue).
# epilogue: None, "addend" (the residual add of the row-parallel projections) or "acc" (wgrad of microbatches 2..8).
FLAGSHIP_GEMMS = [
    (0, 8192, 3072, 2048, None), (0, 8192, 2048, 2048, "addend"), (0, 8192, 16384, 2048, None),
    (0, 8192, 2048, 8192, "addend"), (0, 8192, 128256, 2048, None),
    (1, 8192, 2048, 3072, None), (1, 8192, 2048, 2048, None), (1, 8192, 2048, 16384, None), (1, 8192, 8192, 2048, None),
    (1, 8192, 2048, 128256, None),
    (2, 3072, 2048, 8192, "acc"), (2, 2048, 2048, 8192, "acc"), (2, 16384, 2048, 8192, "acc"), (2, 2048, 8192, 8192, "acc"),
    (2, 128256, 2048, 8192, "acc"),
]


def gemm():
    """The flagship GEMMs, ours and cuBLAS (torch) interleaved round by round, on input sets rotated so that their sum exceeds
    the 50 MB L2.  operand_TBps = the A and B bytes the CTAs load from L2 into shared memory (tiles x k-blocks x (128 + tile
    width) x 64 x 2 B: 32 KiB for a 128-wide tile, 48 KiB for a 256-wide one) over the kernel time."""
    import math
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"nvidia_smi": q.stdout.strip()}), flush=True)
    rounds = 5
    for layout, m, n, k, epi in FLAGSHIP_GEMMS:
        set_bytes = 2 * (m * k + n * k + (2 if epi == "addend" else 1) * m * n)
        sets = []
        for _ in range(max(1, math.ceil(200e6 / set_bytes))):
            a = torch.randn((k, m) if layout == 2 else (m, k), device="cuda").to(BF)
            b = torch.randn((n, k) if layout == 0 else (k, n), device="cuda").to(BF)
            c = torch.randn(m, n, device="cuda").to(BF)
            add = torch.randn(m, n, device="cuda").to(BF) if epi == "addend" else None
            sets.append((a, b, c, add))
        fl = 2.0 * m * n * k
        iters = max(4, math.ceil(0.1 * 4e14 / fl))      # ~100 ms per timed window

        def ours(s):
            a, b, c, add = s
            if epi == "addend":
                bg.gemm_bf16_add(a, b, c, add, m, n, k, layout)
            else:
                bg.gemm_bf16(a, b, c, m, n, k, layout, accumulate=epi == "acc")

        def cublas(s):
            a, b, c, add = s
            at, bt = (a.t() if layout == 2 else a), (b.t() if layout == 0 else b)
            if epi == "addend":
                torch.addmm(add, at, bt, out=c)
            elif epi == "acc":
                c.addmm_(at, bt)
            else:
                torch.matmul(at, bt, out=c)

        def window(fn):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for i in range(iters):
                fn(sets[i % len(sets)])
            e.record()
            torch.cuda.synchronize()
            return s.elapsed_time(e) / iters

        arms = {"cublas": cublas, "ours": ours}
        times = {name: [] for name in arms}
        for fn in arms.values():        # warm-up: module load, cuBLAS heuristics
            window(fn)
        for _ in range(rounds):
            for name, fn in arms.items():
                times[name].append(window(fn))
        rec = {"bench": "gemm", "layout": "TN NN NT".split()[layout], "m": m, "n": n, "k": k, "epilogue": epi}
        for name, ts in times.items():
            t = sorted(ts)[rounds // 2]
            rec[name + "_ms"] = round(t, 4)
            rec[name + "_tflops"] = round(fl / t / 1e9, 1)
            rec[name + "_spread_pct"] = round(100 * (max(ts) - min(ts)) / t, 1)
        bn = 256 if n > 128 else 128    # the plain GEMM's tile width for this N (gemm_launch in bg_gemm.cu)
        tiles_kblocks = -(-m // 128) * -(-n // bn) * -(-k // 64)
        rec["ours_tile_n"] = bn
        rec["ours_operand_TBps"] = round(tiles_kblocks * (128 + bn) * 64 * 2 / rec["ours_ms"] / 1e9, 2)
        print(json.dumps(rec), flush=True)
        del sets
        torch.cuda.empty_cache()


def cast():
    n = 1 << 30
    src = torch.randn(n, device="cuda")
    dst = torch.empty(n, device="cuda", dtype=BF)
    t = timeit(lambda: bg.cast(src, dst))
    print(json.dumps({"bench": "cast_f32_bf16", "elems": n, "ms": round(t, 4), "GBps": round(n * 6 / t / 1e6, 1)}), flush=True)
    t = timeit(lambda: dst.copy_(src))
    print(json.dumps({"bench": "torch_copy_cast", "elems": n, "ms": round(t, 4), "GBps": round(n * 6 / t / 1e6, 1)}), flush=True)
    # the n=1 degenerate all-gather+cast / reduce-scatter+acc (what a 1-GPU step runs per layer)
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    P = 218_112_000
    comm = bg.BgComm(0, 1, 0, (P * 2 + (1 << 20)) * 2)
    grp = CommGroup([0])
    w, g = comm.sym_alloc(grp, P * 2), comm.sym_alloc(grp, P * 2)
    master, mg = torch.randn(P, device="cuda"), torch.zeros(P, device="cuda")
    t = timeit(lambda: comm.all_gather_cast(grp, master, w))
    print(json.dumps({"bench": "all_gather_cast_n1", "elems": P, "ms": round(t, 4), "GBps": round(P * 6 / t / 1e6, 1)}), flush=True)
    t = timeit(lambda: comm.reduce_scatter_acc(grp, g, BF, mg, accumulate=True))
    print(json.dumps({"bench": "reduce_scatter_acc_n1", "elems": P, "ms": round(t, 4), "GBps": round(P * 10 / t / 1e6, 1)}), flush=True)
    comm.close()


def ops():
    """the row kernels at the Llama-3-8B shapes of one microbatch (seq 8192): achieved HBM GB/s = algorithmic bytes / time"""
    import ctypes
    L = bg.lib()
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    S = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)  # noqa: E731
    rows, h, ffn = 8192, 4096, 14336
    x, dy, w = torch.randn(rows, h, device="cuda").to(BF), torch.randn(rows, h, device="cuda").to(BF), torch.randn(h, device="cuda").to(BF)
    y, dx, rstd = torch.empty_like(x), torch.empty_like(x), torch.empty(rows, device="cuda")
    npart = 3 * torch.cuda.get_device_properties(0).multi_processor_count      # as backend.norm_partials
    dwp = torch.empty(npart, h, device="cuda")
    gu, dact = torch.randn(rows, 2 * ffn, device="cuda").to(BF), torch.randn(rows, ffn, device="cuda").to(BF)
    act, dgu = torch.empty(rows, ffn, device="cuda", dtype=BF), torch.empty(rows, 2 * ffn, device="cuda", dtype=BF)
    ng, r, hn = 8, 4, 128
    mixed = torch.randn(rows, 1, ng * (r + 2) * hn, device="cuda").to(BF)
    q, k, v = (torch.empty(1, rows, ng * r, hn, device="cuda", dtype=BF), torch.empty(1, rows, ng, hn, device="cuda", dtype=BF),
               torch.empty(1, rows, ng, hn, device="cuda", dtype=BF))
    cos, sin = torch.rand(rows, hn // 2, device="cuda"), torch.rand(rows, hn // 2, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")      # > 50 MB L2: written between timed launches

    def timed(fn, iters=20):
        ts = []
        for _ in range(iters + 3):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(); fn(); e.record()
            torch.cuda.synchronize()
            ts.append(s.elapsed_time(e))
        return sorted(ts[3:])[len(ts[3:]) // 2]
    cases = [
        ("rmsnorm_fwd", lambda: L.bg_rmsnorm_fwd(P(x), P(w), P(y), P(rstd), rows, h, 1e-5, S()), 2 * x.numel() * 2),
        ("rmsnorm_bwd", lambda: L.bg_rmsnorm_bwd(P(dy), P(x), P(w), P(rstd), P(dx), P(dwp), rows, h, npart, S()), 3 * x.numel() * 2),
        ("swiglu_fwd", lambda: L.bg_swiglu_fwd(P(gu), P(act), rows, ffn, S()), 3 * act.numel() * 2),
        ("swiglu_bwd", lambda: L.bg_swiglu_bwd(P(dact), P(gu), P(dgu), rows, ffn, S()), 5 * act.numel() * 2),
        ("qkv_rope_fwd", lambda: L.bg_qkv_rope(P(mixed), P(q), P(k), P(v), P(cos), P(sin), rows, 1, ng, r, hn, 0, S()), 2 * mixed.numel() * 2),
        ("qkv_rope_bwd", lambda: L.bg_qkv_rope(P(mixed), P(q), P(k), P(v), P(cos), P(sin), rows, 1, ng, r, hn, 1, S()), 2 * mixed.numel() * 2),
    ]
    for name, fn, nbytes in cases:
        bg.check(fn())
        t = timed(fn)
        print(json.dumps({"bench": name, "rows": rows, "ms": round(t, 4), "algorithmic_MB": round(nbytes / 1e6, 1),
                          "GBps": round(nbytes / t / 1e6, 1), "frac_of_hbm_peak_6567": round(nbytes / t / 1e6 / 6566.7, 3),
                          "timing": "median of 20 single launches, L2 flushed (256 MiB memset) before each"}), flush=True)


def attn():
    """K3 is a library call in the reference (flash-attn 2); compare the attention libraries present in the image."""
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel
    b, s, n, ng, d = 1, 8192, 32, 8, 128
    q = torch.randn(b, s, n, d, device="cuda", dtype=BF, requires_grad=True)
    k = torch.randn(b, s, ng, d, device="cuda", dtype=BF, requires_grad=True)
    v = torch.randn(b, s, ng, d, device="cuda", dtype=BF, requires_grad=True)
    do = torch.randn(b, s, n, d, device="cuda", dtype=BF)
    fl_f = 4.0 * b * s * s * n * d / 2
    results = {}

    def run(name, fwd):
        try:
            out = fwd()
            t_f = timeit(fwd)
            def fb():
                o = fwd()
                o.backward(do, retain_graph=False)
                q.grad = k.grad = v.grad = None
            t_fb = timeit(fb)
            results[name] = out.detach()
            print(json.dumps({"bench": "attention", "impl": name, "fwd_ms": round(t_f, 3), "fwd_tflops": round(fl_f / t_f / 1e9, 1),
                              "fwd_bwd_ms": round(t_fb, 3), "fwd_bwd_tflops": round(3.5 * fl_f / t_fb / 1e9, 1)}), flush=True)
        except Exception as e:  # noqa: BLE001
            print(json.dumps({"bench": "attention", "impl": name, "error": str(e)[:300]}), flush=True)

    from flash_attn import flash_attn_func
    run("flash_attn2", lambda: flash_attn_func(q, k, v, causal=True))
    for be_name, be in (("sdpa_cudnn", SDPBackend.CUDNN_ATTENTION), ("sdpa_flash", SDPBackend.FLASH_ATTENTION)):
        def f(be=be):
            with sdpa_kernel(be):
                return F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=True,
                                                      enable_gqa=True).transpose(1, 2)
        run(be_name, f)
    if "flash_attn2" in results:
        for name, o in results.items():
            print(json.dumps({"bench": "attention_parity", "impl": name,
                              "max_abs_diff_vs_flash_attn2": float((o.float() - results["flash_attn2"].float()).abs().max())}), flush=True)


def dropout():
    """The bias + dropout + residual row kernels at the GPT-3 6.7B leg shape (h 4096, seq 2048) and the BERT-large leg shape
    (h 1024, seq 8192), microbatch 4, against torch's eager ``F.dropout(x + b) + r`` and its backward (``native_dropout_backward``
    on the stored mask + the bias-gradient column sum), interleaved round by round on two input sets of > 50 MB each.
    Algorithmic bytes: forward reads x and the residual and writes y (6 B / element; torch also writes and reads a 1-B mask and
    the x + b temporary), backward reads dy and writes dx (4 B / element; ours regenerates the mask).  Also probes which SDPA
    backends accept dropout on the attention probabilities at those shapes."""
    import subprocess
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"nvidia_smi": q.stdout.strip()}), flush=True)
    be = CudaBackend(arena_bytes=1 << 24)
    p, rounds = 0.1, 5
    for name, s, h in (("gpt3_6.7b", 2048, 4096), ("bert_large", 8192, 1024)):
        b = 4
        sets = [tuple(torch.randn(s, b, h, device="cuda").to(BF) for _ in range(3)) + (torch.randn(h, device="cuda").to(BF),) for _ in range(2)]
        masks = [torch.rand(s, b, h, device="cuda") >= p for _ in range(2)]
        n = s * b * h
        iters = 20

        arms = {
            "ours_fwd": lambda st, m: be.dropout_add_fwd(st[0], st[3], st[1], p, 1234, 7, 5, 0, 0),
            "torch_fwd": lambda st, m: F.dropout(st[0] + st[3], p) + st[1],
            "ours_bwd": lambda st, m: be.dropout_bwd(st[2], p, 1234, 7, 5, 0, 0, with_bias=True),
            "torch_bwd": lambda st, m: (lambda dx: (dx, dx.sum((0, 1))))(torch.ops.aten.native_dropout_backward(st[2], m, 1.0 / (1.0 - p))),
        }

        def window(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(iters):
                fn(sets[i % 2], masks[i % 2])
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / iters

        times = {k: [] for k in arms}
        for fn in arms.values():
            window(fn)
        for _ in range(rounds):
            for k, fn in arms.items():
                times[k].append(window(fn))
        rec = {"bench": "dropout", "shape": name, "s": s, "b": b, "h": h, "p": p}
        for k, ts in times.items():
            t = sorted(ts)[rounds // 2]
            nbytes = (6 if k.endswith("fwd") else 4) * n
            rec[k + "_ms"] = round(t, 4)
            rec[k + "_GBps_algorithmic"] = round(nbytes / t / 1e6, 1)
            rec[k + "_pct_of_3350GBps"] = round(100 * nbytes / t / 1e6 / 3350, 1)
            rec[k + "_spread_pct"] = round(100 * (max(ts) - min(ts)) / t, 1)
        print(json.dumps(rec), flush=True)
        # which SDPA kernels take dropout_p at this shape (32 heads of 128 for GPT, 16 of 64 for BERT; causal for GPT)
        heads, hd = (32, 128) if name.startswith("gpt") else (16, 64)
        qkv = [torch.randn(1, heads, min(s, 4096), hd, device="cuda", dtype=BF, requires_grad=True) for _ in range(3)]
        ok = {}
        for bk in (SDPBackend.CUDNN_ATTENTION, SDPBackend.FLASH_ATTENTION, SDPBackend.EFFICIENT_ATTENTION):
            try:
                with sdpa_kernel([bk]):
                    o = F.scaled_dot_product_attention(*qkv, dropout_p=0.1, is_causal=name.startswith("gpt"))
                    o.sum().backward()
                torch.cuda.synchronize()
                ok[bk.name] = True
            except RuntimeError as e:
                ok[bk.name] = "refused: " + str(e).splitlines()[0][:120]
        print(json.dumps({"bench": "sdpa_dropout_backends", "shape": name, "accepts_dropout": ok}), flush=True)
        del sets, masks
        torch.cuda.empty_cache()
    be.close()


class _LocalRing:
    """Stand-in ring transport that moves nothing: every block is the rank's own (same shapes as the real hops), so the ring
    schedule of tensor_parallel/transformer.py runs its attention, merge and cast work with the transport excluded."""

    def __init__(self, c, k, v):
        self.size, self.rank, self.kv = c, 0, (k, v)
        self.acc = torch.zeros(2 * k.numel(), device=k.device)

    def send_kv(self, step, k, v):
        pass

    def recv_kv(self, step):
        return self.kv

    def release_kv(self, step):
        pass

    def send_acc(self, step, acc_in, dk, dv, c_row0, c_rows):
        pass

    def recv_acc(self, step):
        return self.acc

    def release_acc(self, step):
        pass


def cp(n=32, ng=8, d=64, seqs=(32768, 131072)):
    """Ring context parallelism at Llama-3.2-1B attention shapes (32 heads, 8 KV heads of 64) by default, or the given heads / KV heads /
    head dim (``--cp-heads 32 --cp-kv-heads 32 --cp-head-dim 128``: GPT-3 6.7B), microbatch 1, sequence S in {32k, 128k} (``--cp-seqs``),
    cp degree c in {2, 4, 8}.  Per rank: attention forward + backward of the ring schedule (2c-1 flash-attn block calls, the LSE
    merges and the fp32 accumulation casts; transport excluded) against the all-gather path's two prefix calls on the gathered
    sequence (gather excluded); the merge and the two push kernels in GB/s over algorithmic bytes -- the pushes between two virtual
    ranks on this one device, i.e. through local HBM, not NVLink; and the K/V bytes each path keeps for backward per layer."""
    import subprocess
    from flash_attn import flash_attn_func
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend, _CpRing
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    from hetu_galvatron_b200.core.runtime.tensor_parallel import transformer as tr
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"nvidia_smi": q.stdout.strip()}), flush=True)
    b = 1
    shape = {} if (n, ng, d) == (32, 8, 64) else {"heads": n, "kv_heads": ng, "head_dim": d}
    scale = d ** -0.5
    be = CudaBackend(arena_bytes=1 << 24)
    for S in seqs:
        for c in (2, 4, 8):
            s = S // c
            qq = torch.randn(b, s, n, d, device="cuda").to(BF)
            k, v = [torch.randn(b, s, ng, d, device="cuda").to(BF) for _ in range(2)]
            do = torch.randn(b, s, n, d, device="cuda").to(BF)
            ring = _LocalRing(c, k, v)

            def ring_fb():
                out, lse = tr.run_steps(tr.ring_attention_fwd(be, ring, qq, k, v, scale))
                tr.run_steps(tr.ring_attention_bwd(be, ring, do, qq, k, v, out, lse, scale))
            kf, vf = [torch.randn(b, S, ng, d, device="cuda").to(BF).requires_grad_(True) for _ in range(2)]
            qg = qq.detach().clone().requires_grad_(True)
            half = s // 2

            def gather_fb():
                outs = [flash_attn_func(qg[:, :half], kf[:, :(ch + 1) * half], vf[:, :(ch + 1) * half], softmax_scale=scale, causal=True)
                        for ch in (0, 2 * c - 1)]     # rank 0's chunks
                torch.cat(outs, 1).backward(do)
            iters = 3 if S > 32768 else 10
            t_ring, t_gather = [], []
            for _ in range(3):                       # interleaved rounds
                t_ring.append(timeit(ring_fb, iters=iters, warm=1))
                t_gather.append(timeit(gather_fb, iters=iters, warm=1))
            kv_ring, kv_gather = 2 * b * s * ng * d * 2, 2 * b * S * ng * d * 2
            print(json.dumps({"bench": "cp_attention_fwd_bwd_per_rank", **shape, "S": S, "c": c, "ring_ms": round(sorted(t_ring)[1], 3),
                              "gather_ms": round(sorted(t_gather)[1], 3), "ring_over_gather": round(sorted(t_ring)[1] / sorted(t_gather)[1], 3),
                              "spread_pct": round(100 * (max(t_ring + t_gather) - min(t_ring + t_gather)) / min(t_ring + t_gather), 1),
                              "transport": "excluded (both paths)", "kv_kept_for_backward_MiB_ring": round(kv_ring / 2 ** 20, 1),
                              "kv_kept_for_backward_MiB_gather": round(kv_gather / 2 ** 20, 1)}), flush=True)
            # the merge: a full-rows step (read block out bf16 + block LSE, read/write running out + LSE fp32)
            acc_out, acc_lse = torch.randn(b, s, n, d, device="cuda"), torch.randn(b, n, s, device="cuda")
            blk_lse = torch.randn(b, n, s, device="cuda")
            t = timeit(lambda: bg.lse_merge(qq, blk_lse, acc_out, acc_lse), iters=20)
            nbytes = b * s * n * d * (2 + 8) + b * n * s * 12
            print(json.dumps({"bench": "cp_lse_merge", "S": S, "c": c, "ms": round(t, 4), "GBps_algorithmic": round(nbytes / t / 1e6, 1),
                              "pct_of_3350GBps": round(100 * nbytes / t / 1e6 / 3350, 1)}), flush=True)
            del qq, do, kf, vf, qg, acc_out, acc_lse, ring
            # the pushes, between two virtual ranks on this device
            elems = b * s * ng * d
            comms = bg.BgComm.local_world(2, device=0, arena_bytes=_CpRing.slot_bytes(elems) + (16 << 20))
            group = CommGroup([0, 1])
            bufs = [cm.sym_alloc(group, _CpRing.slot_bytes(elems)) for cm in comms]
            for cm in comms:
                cm.exchange()
            rings = [_CpRing(cm, group, buf, elems) for cm, buf in zip(comms, bufs)]
            dk, dv = [torch.randn(b, s, ng, d, device="cuda").to(BF) for _ in range(2)]

            def hop_kv():
                rings[0].send_kv(0, k, v)
                rings[1].recv_kv(1)
                rings[1].release_kv(1)

            def hop_acc():
                rings[0].send_acc(0, None, dk, dv, 0, s)
                rings[1].recv_acc(1)
                rings[1].release_acc(1)
            rings[1].shape = tuple(k.shape)
            for name, fn, nb in (("kv_push", hop_kv, 2 * elems * 2), ("acc_push", hop_acc, 2 * elems * (2 + 4))):
                t = timeit(fn, iters=20)
                print(json.dumps({"bench": "cp_ring_" + name, "S": S, "c": c, "ms_per_hop": round(t, 4),
                                  "GBps_algorithmic": round(nb / t / 1e6, 1), "path": "local HBM (two virtual ranks on one device), not NVLink",
                                  "bytes": "kv: K+V bf16 payload; acc: bf16 contribution read + fp32 accumulator written"}), flush=True)
            torch.cuda.synchronize()
            for cm in comms:
                assert cm.error_flag() == 0
                cm.close()
            del k, v, dk, dv
            torch.cuda.empty_cache()
    be.close()


def clip():
    """Gradient clipping with the fused optimizer at the flagship units' shard sizes (Llama-3.2-1B, one GPU, p = 1): the norm pass,
    the clipped step pass and today's unclipped AdamW reduce-scatter, beside what the torch optimizer runs after the backward to
    clip (pow().sum(), mul_, fused AdamW over the fp32 gradient shard).  GB/s over the algorithmic bytes: norm pass P*gsz, step pass
    P*gsz + 24*P (read and write param, exp_avg, exp_avg_sq), pow-sum 4P, mul_ 8P, torch fused AdamW 28P."""
    import subprocess
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"nvidia_smi": q.stdout.strip()}), flush=True)
    hyper = (1e-4, 0.9, 0.95, 1e-8, 0.01)
    for unit, P in (("decoder_layer", 60_821_504), ("embed_or_head", 262_668_288)):
        comm = bg.BgComm(0, 1, 0, P * 2 + (1 << 24))
        grp = CommGroup([0])
        g = comm.sym_alloc(grp, P * 2)
        comm.exchange()
        g.view(BF, P).copy_(torch.randn(P, device="cuda").to(BF) * 1e-3)
        p, m, v = torch.randn(P, device="cuda"), torch.zeros(P, device="cuda"), torch.zeros(P, device="cuda")
        parts = torch.zeros(4 * max(bg.get_tunable("comm_ctas"), bg.get_tunable("local_ctas")), device="cuda")
        coef = torch.full((), 0.5, device="cuda")
        runs = {
            "norm_pass": (lambda: comm.reduce_scatter_sumsq(grp, g, BF, P, 1.0, 1.0, parts), 2 * P),
            "step_pass_clipped": (lambda: comm.reduce_scatter_adamw_clipped(grp, g, BF, p, m, v, P, 1.0, 1.0, *hyper, 1, coef), 26 * P),
            "reduce_scatter_adamw": (lambda: comm.reduce_scatter_adamw(grp, g, BF, p, m, v, P, 1.0, 1.0, *hyper, 1), 26 * P),
        }
        for name, (fn, nbytes) in runs.items():
            t = timeit(fn)
            print(json.dumps({"bench": "clip_" + name, "unit": unit, "elems": P, "ms": round(t, 4),
                              "GBps_algorithmic": round(nbytes / t / 1e6, 1)}), flush=True)
        comm.close()
        del g
        grad = torch.randn(P, device="cuda") * 1e-3
        step = torch.ones((), device="cuda")
        torch_runs = {
            "torch_pow_sum": (lambda: grad.pow(2).sum(), 4 * P),
            "torch_mul": (lambda: grad.mul_(coef), 8 * P),
            "torch_fused_adamw": (lambda: torch._fused_adamw_([p], [grad], [m], [v], [], [step], lr=hyper[0], beta1=hyper[1], beta2=hyper[2],
                                                              weight_decay=hyper[4], eps=hyper[3], amsgrad=False, maximize=False), 28 * P),
        }
        total = 0.0
        for name, (fn, nbytes) in torch_runs.items():
            t = timeit(fn)
            total += t
            print(json.dumps({"bench": "clip_" + name, "unit": unit, "elems": P, "ms": round(t, 4),
                              "GBps_algorithmic": round(nbytes / t / 1e6, 1)}), flush=True)
        print(json.dumps({"bench": "clip_torch_tail_total", "unit": unit, "ms": round(total, 4)}), flush=True)
        del p, m, v, grad
        torch.cuda.empty_cache()


def tied(vocab=50257, hidden=4096):
    """Tied word embeddings across two pipeline stages (C14) at the GPT-3 6.7B embedding (50257 x 4096), vocab-tp 1 and 2, bf16 and
    fp32 gradients: ``bg_pair_sum_inplace`` on the two copies' gradient ranges against what an all-reduce needs (copy into a staging
    buffer, ``bg_all_reduce`` into a temporary, copy back), both for two virtual ranks on this one device -- so every peer access is
    local HBM, not NVLink.  GB/s per member over the algorithmic bytes of the in-place sum: a member reads E/2 elements of its own
    copy and E/2 of the peer's, and writes as many into each (4 x E/2 x element size); both members run at once on the device."""
    import subprocess
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"nvidia_smi": q.stdout.strip()}), flush=True)
    group = CommGroup([0, 1])
    for t in (1, 2):
        elems = vocab * hidden // t // 8 * 8
        for dt in (BF, torch.float32):
            nbytes = elems * torch.empty((), dtype=dt).element_size()
            comms = bg.BgComm.local_world(2, device=0, arena_bytes=2 * nbytes + (16 << 20))
            grads = [c.alloc(nbytes) for c in comms]
            regs = [c.sym_register(group, off, nbytes) for c, (off, _) in zip(comms, grads)]
            stage = [c.sym_alloc(group, nbytes) for c in comms]
            for c in comms:
                c.exchange()
            for _, g in grads:
                g.view(dt).copy_(torch.randn(elems, device="cuda").to(dt) * 1e-3)
            tmp = [torch.empty(elems, dtype=dt, device="cuda") for _ in comms]
            streams = [torch.cuda.Stream() for _ in comms]

            def both(fn):
                cur = torch.cuda.current_stream()
                for s in streams:
                    s.wait_stream(cur)
                for r in range(2):
                    with torch.cuda.stream(streams[r]):
                        fn(r)
                for s in streams:
                    cur.wait_stream(s)

            def pair(r):
                comms[r].pair_sum_inplace(group, regs[r], dt, scale=0.5)

            def staged(r):
                stage[r].u8.copy_(grads[r][1])
                comms[r].all_reduce(group, stage[r], tmp[r], scale=0.5, lane=bg.LANE_REDUCE)
                grads[r][1].view(dt).copy_(tmp[r])
            res = {"pair": [], "staged": []}
            for _ in range(3):                       # interleaved rounds
                res["pair"].append(timeit(lambda: both(pair), iters=10))
                res["staged"].append(timeit(lambda: both(staged), iters=10))
            torch.cuda.synchronize()
            for c in comms:
                assert c.error_flag() == 0
            alg = 4 * (elems // 2) * (nbytes // elems)
            med = {k: sorted(v)[1] for k, v in res.items()}
            for k in ("pair", "staged"):
                print(json.dumps({"bench": "tied_" + k, "vocab_tp": t, "dtype": str(dt).split(".")[-1], "elems": elems, "ms": round(med[k], 4),
                                  "GBps_algorithmic_per_member": round(alg / med[k] / 1e6, 1),
                                  "spread_pct": round(100 * (max(res[k]) - min(res[k])) / min(res[k]), 1),
                                  "extra_arena_bytes_per_member": 0 if k == "pair" else nbytes,
                                  "path": "local HBM (two virtual ranks on one device), not NVLink"}), flush=True)
            print(json.dumps({"bench": "tied_staged_over_pair", "vocab_tp": t, "dtype": str(dt).split(".")[-1],
                              "ratio": round(med["staged"] / med["pair"], 3)}), flush=True)
            for c in comms:
                c.close()
            del grads, regs, stage, tmp
            torch.cuda.empty_cache()


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser(description="kernel micro-benchmarks; JSON lines on stdout")
    ap.add_argument("which", nargs="*", default=["gemm", "cast"])
    ap.add_argument("--cp-heads", type=int, default=32, help="cp: query heads")
    ap.add_argument("--cp-kv-heads", type=int, default=8, help="cp: key/value heads")
    ap.add_argument("--cp-head-dim", type=int, default=64, help="cp: head dimension")
    ap.add_argument("--cp-seqs", default="32768,131072", help="cp: comma-separated sequence lengths")
    opts = ap.parse_args()
    print(json.dumps({"device": torch.cuda.get_device_name(0)}))
    for w in opts.which:
        if w == "cp":
            cp(opts.cp_heads, opts.cp_kv_heads, opts.cp_head_dim, tuple(int(x) for x in opts.cp_seqs.split(",")))
        else:
            globals()[w]()

"""Multi-GPU parity + timing of the three fused GEMM + collective operations at the Llama-3-8B tensor-parallel shapes, against
(our GEMM -> our stand-alone collective) and (cuBLAS -> NCCL), torchrun one process per GPU.  JSON lines on rank 0.

  gemm_reduce_scatter   C8  row-parallel forward under Megatron-SP / SP dgrad       (layers.py:1061-1109, :462,488-494)
  gemm_all_reduce       C5  row-parallel forward, C6 column-parallel dgrad          (layers.py:1110-1114, mappings_group.py:139)
  all_gather_gemm       C7  column-parallel forward under SP, row-parallel dgrad    (layers.py:399-417, mappings_group.py:243-258)

Roofline of a fused op: the slower of FLOPs / GEMM peak and NVLink bytes / 450 GB/s (H100 SXM data-sheet figures).
    torchrun --nproc-per-node N --master-addr 127.0.0.1 scripts/test_fused_collectives.py
"""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hetu_galvatron_b200.core.runtime.arguments import initialize_galvatron  # noqa: E402
from hetu_galvatron_b200.core.runtime.backend import get_backend, reset_backend  # noqa: E402
from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup  # noqa: E402

BF = torch.bfloat16
GEMM_PEAK_TFLOPS, NVLINK_GBS = 989.0, 450.0       # H100 SXM data sheet: dense bf16, NVLink 4 per direction


def timed(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / iters], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t[0])


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    # the fused operations are timed at K below the runtime's thresholds too
    os.environ["HGB_FUSE_GEMM_RS"] = os.environ["HGB_FUSE_GEMM_AR"] = "force"
    initialize_galvatron(arena_bytes=2 << 30)
    be = get_backend()
    be.bg.set_tunable("timeout_ms", 20000)
    grp = CommGroup(list(range(world)))
    p = world
    M = 8192                       # seq 8192 x microbatch 1
    be.reserve_staging(grp, M * 14336 // p * 2 + M * 4096 * 2)
    be.exchange()
    ok_all = True
    warm = torch.randn(256, 256, device="cuda").to(BF)
    torch.matmul(warm, warm)
    dist.all_reduce(torch.zeros(8, device="cuda"))
    torch.cuda.synchronize()

    def emit(rec):
        if rank == 0:
            print(json.dumps(rec), flush=True)
    emit({"p": p, "nvls": bool(getattr(be, "nvls", False)), "nvls_regions": len(getattr(be, "nvls_regions", {}) or {}), "M": M})

    def bound_ms(flops, nvlink_bytes):
        return max(flops / (GEMM_PEAK_TFLOPS * 1e12), nvlink_bytes / (NVLINK_GBS * 1e9)) * 1e3

    # ---- GEMM + reduce-scatter / GEMM + all-reduce: row-parallel forward (down-proj K = ffn/p, o-proj K = h/p) and SP dgrad --------
    for op in ("gemm_reduce_scatter", "gemm_all_reduce"):
        for layout, K, N in (("tn", 14336 // p, 4096), ("tn", 4096 // p, 4096), ("nn", 6144 // p, 4096)):
            torch.manual_seed(7 + rank)
            a = (torch.randn(M, K, device="cuda") * 0.5).to(BF)
            b = (torch.randn((N, K) if layout == "tn" else (K, N), device="cuda") * 0.5).to(BF)
            fused = (lambda: be.gemm_reduce_scatter(a, b, layout, grp)) if op == "gemm_reduce_scatter" else (lambda: be.gemm_all_reduce(a, b, layout, grp))
            out = fused()
            torch.cuda.synchronize()
            full = torch.matmul(a, b.t() if layout == "tn" else b)
            if op == "gemm_reduce_scatter":
                ref = torch.empty(M // p, N, device="cuda", dtype=BF)
                dist.reduce_scatter_tensor(ref, full)
            else:
                ref = full.clone()
                dist.all_reduce(ref)
            torch.cuda.synchronize()
            err = float((out.float() - ref.float()).abs().max() / (ref.float().abs().max() + 1e-6))
            out2 = None
            for _ in range(3):   # repeated use: counters must reset, buffers must be reusable
                out2 = fused()
            torch.cuda.synchronize()
            same = bool(torch.equal(out.view(torch.int16), out2.view(torch.int16)))
            if op == "gemm_all_reduce":      # replicas bit-identical across the group
                chk = out.view(torch.int16).double().sum().reshape(1)
                lo, hi = chk.clone(), chk.clone()
                dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
                same = same and bool(lo == hi)
            fused_ms = timed(fused)

            def unfused():
                staged, _ = be.staging_tensor(grp, (M, N), BF)
                be.gemm(a, b, layout, out=staged)
                return be.reduce_scatter_first_dim(staged, grp) if op == "gemm_reduce_scatter" else be.all_reduce(staged, grp)
            unfused_ms = timed(unfused)

            def nccl():
                f = torch.matmul(a, b.t() if layout == "tn" else b)
                if op == "gemm_reduce_scatter":
                    dist.reduce_scatter_tensor(ref, f)
                else:
                    dist.all_reduce(f)
            nccl_ms = timed(nccl)
            gemm_ms = timed(lambda: be.gemm(a, b, layout))
            ok = err < 2e-2 and same
            ok_all &= ok
            nv = M * N * 2 * (p - 1) / p * (2 if op == "gemm_all_reduce" else 1)
            lb = bound_ms(2.0 * M * N * K, nv)
            emit({"op": op, "layout": layout, "M": M, "N": N, "K": K, "p": p, "fused_ms": round(fused_ms, 4),
                  "ours_gemm_then_collective_ms": round(unfused_ms, 4), "cublas_then_nccl_ms": round(nccl_ms, 4), "gemm_only_ms": round(gemm_ms, 4),
                  "roofline_ms": round(lb, 4), "frac_of_roofline": round(lb / fused_ms, 3), "max_rel_err_vs_nccl": round(err, 5),
                  "deterministic_and_replicated": same, "ok": ok})
    # ---- all-gather + GEMM: column-parallel forward under SP (QKV N = 6144/p, gate/up N = 28672/p) and row-parallel dgrad --------
    for layout, K, N in (("tn", 4096, 6144 // p), ("tn", 4096, 28672 // p), ("nn", 4096, 14336 // p)):
        torch.manual_seed(11 + rank)
        a_loc = (torch.randn(M // p, K, device="cuda") * 0.5).to(BF)
        b = (torch.randn((N, K) if layout == "tn" else (K, N), device="cuda") * 0.5).to(BF)
        out, gathered = be.all_gather_gemm(a_loc, b, layout, grp)
        torch.cuda.synchronize()
        a_full = torch.empty(M, K, device="cuda", dtype=BF)
        dist.all_gather_into_tensor(a_full, a_loc)
        want = be.gemm(a_full, b, layout)
        torch.cuda.synchronize()
        exact = bool(torch.equal(out.view(torch.int16), want.view(torch.int16))) and bool(torch.equal(gathered.view(torch.int16), a_full.view(torch.int16)))
        for _ in range(3):
            out2, _ = be.all_gather_gemm(a_loc, b, layout, grp)
        torch.cuda.synchronize()
        exact = exact and bool(torch.equal(out2.view(torch.int16), want.view(torch.int16)))
        fused_ms = timed(lambda: be.all_gather_gemm(a_loc, b, layout, grp))

        def unfused():
            total = be.all_gather_into_staging(a_loc, grp)
            return be.gemm(total, b, layout)
        unfused_ms = timed(unfused)

        def nccl():
            dist.all_gather_into_tensor(a_full, a_loc)
            return torch.matmul(a_full, b.t() if layout == "tn" else b)
        nccl_ms = timed(nccl)
        gemm_ms = timed(lambda: be.gemm(a_full, b, layout))
        ok_all &= exact
        lb = bound_ms(2.0 * M * N * K, M * K * 2 * (p - 1) / p)
        emit({"op": "all_gather_gemm", "layout": layout, "M": M, "N": N, "K": K, "p": p, "fused_ms": round(fused_ms, 4),
              "ours_gather_then_gemm_ms": round(unfused_ms, 4), "nccl_then_cublas_ms": round(nccl_ms, 4), "gemm_only_ms": round(gemm_ms, 4),
              "roofline_ms": round(lb, 4), "frac_of_roofline": round(lb / fused_ms, 3), "bit_exact_vs_plain_gemm": exact, "ok": exact})
    assert be.comm.error_flag() == 0
    dist.barrier()
    if rank == 0:
        print("FUSED_OK" if ok_all else "FUSED_FAIL", flush=True)
    reset_backend()
    dist.destroy_process_group()
    sys.exit(0 if ok_all else 1)


if __name__ == "__main__":
    try:
        main()
    except Exception:
        try:
            sys.stderr.write("rank %s: device error info %s\n" % (os.environ.get("RANK", "0"), get_backend().comm.error_info()))
        except Exception:
            pass
        raise

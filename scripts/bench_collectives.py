"""Real multi-GPU micro-benchmark + parity check of the peer-memory collectives against NCCL (torchrun, one process per GPU).

    torchrun --nproc-per-node N --master-addr 127.0.0.1 scripts/bench_collectives.py [--max-mb 1024] [--sizes-mb 1,64,1024]

For each message size and collective: the slim peer-to-peer kernel, the same kernel on the multicast path (NVLS: multimem.st /
multimem.ld_reduce, when the fabric supports it) and the torch.distributed (NCCL) sequence the reference issues at the same call
site -- all CUDA-event timed (median launch, max over ranks), bus bandwidth by the nccl-tests convention (AG/RS/A2A (p-1)/p*N,
AR 2(p-1)/p*N) against 450 GB/s nominal (H100 NVLink 4, per direction), and a result comparison (bit-exact for data movement,
bf16 tolerance for reductions).  JSON lines on rank 0; COLLECTIVES_OK / COLLECTIVES_FAIL last."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hetu_galvatron_b200 import _bg as bg  # noqa: E402
from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup  # noqa: E402

BF = torch.bfloat16


def timed(fn, iters=20, warm=5):
    """Per-launch CUDA events (the kernels wait for their peers, so a launch's span includes rank skew): report the
    MEDIAN launch, max over ranks.  A back-to-back loop time is dominated by host launch skew for sub-ms messages."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
    evs = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        evs.append((e0, e1))
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) for a, b in evs)
    t = torch.tensor([ts[len(ts) // 2]], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-mb", type=int, default=1024)
    ap.add_argument("--sizes-mb", default="")
    ap.add_argument("--ctas", type=int, default=0)
    opts = ap.parse_args()
    if os.environ.get("BENCH_QUICK") and not opts.sizes_mb:
        opts.max_mb, opts.sizes_mb = 64, "1,16,64"
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    max_bytes = opts.max_mb << 20
    bg.set_tunable("timeout_ms", 30000)
    bg.set_tunable("nvls_min_ranks", 2)         # measure the multicast paths at every group size
    nvls = os.environ.get("HGB_NVLS", "1") == "1"
    try:
        comm = bg.BgComm(rank, world, local, 3 * max_bytes + (64 << 20), vmm=nvls)
        nvls = nvls and comm.arena_mode()[1]
    except bg.BgError:
        comm, nvls = bg.BgComm(rank, world, local, 3 * max_bytes + (64 << 20)), False
    comm.connect_vmm() if comm.vmm else comm.connect_ipc()
    if opts.ctas:
        bg.set_tunable("comm_ctas", opts.ctas)
    grp = CommGroup(list(range(world)))
    full = comm.sym_alloc(grp, max_bytes)      # unsharded buffer (AG dst / RS src / AR src / A2A src)
    comm.exchange()
    regions = comm.setup_nvls() if nvls else {}
    nvls = bool(regions)
    p = world
    ok_all = True

    def emit(rec):
        if rank == 0:
            print(json.dumps(rec), flush=True)

    emit({"arena": "vmm" if comm.vmm else "cudaMalloc+ipc", "nvls_regions": {"-".join(map(str, k)): v for k, v in regions.items()},
          "comm_ctas": bg.get_tunable("comm_ctas"), "p": p})

    def both(fn):
        """(p2p ms, nvls ms or None): the same call with the multicast paths switched off / on"""
        bg.set_tunable("nvls_gather", 0); bg.set_tunable("nvls_reduce", 0); bg.set_tunable("nvls_min_bytes", 1 << 60)
        a = timed(fn)
        b = None
        if nvls:
            bg.set_tunable("nvls_gather", 1); bg.set_tunable("nvls_reduce", 1); bg.set_tunable("nvls_min_bytes", 1 << 20)
            b = timed(fn)
        return a, b

    if opts.sizes_mb:
        sizes = [int(x) << 20 for x in opts.sizes_mb.split(",")]
    else:
        sizes = [1 << 20]
        while sizes[-1] * 4 <= max_bytes:
            sizes.append(sizes[-1] * 4)
        if sizes[-1] != max_bytes:
            sizes.append(max_bytes)
    torch.manual_seed(1234 + rank)
    gb = lambda nbytes, factor, ms: None if ms is None else round(nbytes * factor / ms / 1e6, 1)  # noqa: E731
    for nbytes in sizes:
        n = nbytes // 2                     # bf16 elements of the full buffer
        shard = n // p
        # ---- all-gather (+cast): fp32 shard -> bf16 full ------------------------------------------------------
        master = torch.randn(shard, device="cuda")
        p2p_ms, nvls_ms = both(lambda: comm.all_gather_cast(grp, master, full, shard_elems=shard, lane=0))
        got = full.view(BF, n).clone()
        ref = torch.empty(n, device="cuda", dtype=BF)
        nccl_ms = timed(lambda: dist.all_gather_into_tensor(ref, master.to(BF)))
        ok = bool(torch.equal(got.view(torch.int16), ref.view(torch.int16)))
        ok_all &= ok
        f = (p - 1) / p
        emit({"op": "all_gather_cast", "bytes": nbytes, "p": p, "p2p_ms": round(p2p_ms, 4), "p2p_busGBps": gb(nbytes, f, p2p_ms),
              "nvls_ms": nvls_ms and round(nvls_ms, 4), "nvls_busGBps": gb(nbytes, f, nvls_ms),
              "nccl_ms(cast+ag)": round(nccl_ms, 4), "nccl_busGBps": gb(nbytes, f, nccl_ms), "bit_exact_vs_nccl": ok})
        # ---- reduce-scatter (+scale, cast, accumulate): bf16 full -> fp32 shard ---------------------------------
        grad = torch.randn(n, device="cuda").to(BF)
        full.view(BF, n).copy_(grad)
        acc = torch.zeros(shard, device="cuda")
        torch.cuda.synchronize(); dist.barrier()
        rs = lambda: comm.reduce_scatter_acc(grp, full, BF, acc, shard_elems=shard, prescale=0.5, postscale=1.0 / p * 2, accumulate=False, lane=1)  # noqa: E731
        p2p_ms, nvls_ms = both(rs)
        ref_sh = torch.empty(shard, device="cuda", dtype=BF)

        def nccl_rs():
            g = grad / 2
            dist.reduce_scatter_tensor(ref_sh, g)
            return ref_sh.float() * (2.0 / p)
        nccl_ms = timed(nccl_rs)
        want = nccl_rs()
        errs = {}
        for name, flag in (("p2p", 0), ("nvls", 1)):
            if flag and not nvls:
                continue
            bg.set_tunable("nvls_reduce", flag); bg.set_tunable("nvls_min_bytes", (1 << 20) if flag else (1 << 60))
            rs(); torch.cuda.synchronize()
            errs[name] = round(float((acc - want).abs().max() / (want.abs().max() + 1e-6)), 5)
        ok = all(e < 2e-2 for e in errs.values())
        ok_all &= ok
        emit({"op": "reduce_scatter_acc", "bytes": nbytes, "p": p, "p2p_ms": round(p2p_ms, 4), "p2p_busGBps": gb(nbytes, f, p2p_ms),
              "nvls_ms": nvls_ms and round(nvls_ms, 4), "nvls_busGBps": gb(nbytes, f, nvls_ms),
              "nccl_ms(div+rs+cast)": round(nccl_ms, 4), "nccl_busGBps": gb(nbytes, f, nccl_ms), "max_rel_err_vs_nccl": errs, "ok": ok})
        # ---- all-reduce ------------------------------------------------------------------------------------------
        dst = torch.empty(n, device="cuda", dtype=BF)

        def ours_ar():
            full.view(BF, n).copy_(grad)
            comm.all_reduce(grp, full, dst, elems=n, lane=2)
        torch.cuda.synchronize(); dist.barrier()
        p2p_ms, nvls_ms = both(ours_ar)
        copy_ms = timed(lambda: full.view(BF, n).copy_(grad))
        ref_ar = grad.clone()
        nccl_ms = timed(lambda: dist.all_reduce(ref_ar.copy_(grad))) - timed(lambda: ref_ar.copy_(grad))
        ref_ar.copy_(grad); dist.all_reduce(ref_ar)
        ours_ar(); torch.cuda.synchronize()
        err = float((dst.float() - ref_ar.float()).abs().max() / (ref_ar.float().abs().max() + 1e-6))
        ok = err < 2e-2
        ok_all &= ok
        fa = 2 * (p - 1) / p
        emit({"op": "all_reduce", "bytes": nbytes, "p": p, "p2p_ms": round(p2p_ms - copy_ms, 4), "p2p_busGBps": gb(nbytes, fa, p2p_ms - copy_ms),
              "nvls_ms": nvls_ms and round(nvls_ms - copy_ms, 4), "nvls_busGBps": None if nvls_ms is None else gb(nbytes, fa, nvls_ms - copy_ms),
              "nccl_ms": round(nccl_ms, 4), "nccl_busGBps": gb(nbytes, fa, nccl_ms), "max_rel_err_vs_nccl": round(err, 5), "ok": ok})
        # ---- Ulysses all-to-all with fused transpose: [b, s/p, heads, d] -> [b, s, heads/p, d] ----------------------
        d, heads = 128, 32
        if heads % p == 0:
            b = 1
            s_loc = n // (heads * d * b)
            if s_loc >= 1:
                x = torch.randn(b, s_loc, heads, d, device="cuda").to(BF)
                full.view(BF, x.numel()).copy_(x.flatten())
                hp = heads // p
                y = torch.empty(b, s_loc * p, hp, d, device="cuda", dtype=BF)
                desc = [dict(src=full, dst=y, batch=b, rows=s_loc, row_elems=hp * d, src_bs=s_loc * heads * d, src_rs=heads * d, src_me_off=hp * d,
                             dst_bs=s_loc * p * hp * d, dst_rs=hp * d, dst_peer_off=s_loc * hp * d)]
                torch.cuda.synchronize(); dist.barrier()
                ours_ms = timed(lambda: comm.all_to_all_rows(grp, desc, BF, lane=3))

                def nccl_a2a():   # transformer.py:1928-1987: permute copy, all_to_all_single, permute copy
                    t = x.reshape(b, s_loc, p, hp, d).permute(2, 0, 1, 3, 4).contiguous()
                    o_ = torch.empty_like(t)
                    dist.all_to_all_single(o_, t)
                    return o_.permute(1, 0, 2, 3, 4).contiguous().reshape(b, p * s_loc, hp, d)
                nccl_ms = timed(nccl_a2a)
                ok = bool(torch.equal(y.view(torch.int16), nccl_a2a().view(torch.int16)))
                ok_all &= ok
                nb = x.numel() * 2
                emit({"op": "ulysses_all_to_all", "bytes": nb, "p": p, "p2p_ms": round(ours_ms, 4), "p2p_busGBps": gb(nb, f, ours_ms),
                      "nccl_ms(permute+a2a+permute)": round(nccl_ms, 4), "nccl_busGBps": gb(nb, f, nccl_ms), "bit_exact_vs_nccl": ok})
    assert comm.error_flag() == 0
    dist.barrier()
    emit({"verdict": "COLLECTIVES_OK" if ok_all else "COLLECTIVES_FAIL"})
    comm.close()
    dist.destroy_process_group()
    sys.exit(0 if ok_all else 1)


if __name__ == "__main__":
    main()

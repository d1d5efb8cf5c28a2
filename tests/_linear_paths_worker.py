"""Worker for tests/test_gpu_linear_paths.py: ``LinearWithGradAccumulationAndAsyncCommunication`` forward and backward over a tensor-
parallel group of 2 virtual ranks (``BgComm.local_world``) on one device, in each of its communicating modes, with the fused GEMM +
collective kernels forced on (HGB_FUSE_*=force) and switched off (=0).  Every output and gradient is compared with fp32 torch on the
same bf16 operands; ``n_fused`` tells which path ran.  Prints one ``LINEAR_CASE`` JSON line per case.

  rs_out     row-parallel under Megatron-SP: GEMM + reduce-scatter forward, all-gather + dgrad GEMM backward
  sp_gather  column-parallel under Megatron-SP: all-gather + GEMM forward, dgrad GEMM + reduce-scatter backward (the wgrad
             re-gather overlaps it when fused)
  ar_out     row-parallel: GEMM + all-reduce forward
  ar_dgrad   column-parallel: dgrad GEMM + all-reduce backward

Each rank has its own backend, staging and stream, and its whole forward (then backward) is issued before the next rank's, so a
collective of rank 0 waits on the device for work the host issues later.  As in tests/_usp_gpu_worker.py nothing the host does in
between may wait for the device: CUDA modules load eagerly and the caching allocator is grown before the ranks run."""
import os

if __name__ == "__main__":          # before CUDA starts (the test imports this module only for its case list)
    os.environ["CUDA_MODULE_LOADING"] = "EAGER"
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import json  # noqa: E402
import sys  # noqa: E402
import traceback  # noqa: E402

import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

P, S, B, K, N = 2, 512, 2, 512, 512          # 2 ranks; [S, B] tokens (M = 1024); GEMM [M, K] x [K, N]
M = S * B
MODES = ("rs_out", "sp_gather", "ar_out", "ar_dgrad")
EXPECT_FUSED = {"rs_out": {"gemm_rs": 1, "ag_gemm": 1}, "sp_gather": {"ag_gemm": 1, "gemm_rs": 1}, "ar_out": {"gemm_ar": 1},
                "ar_dgrad": {"gemm_ar": 1}}
FUSE_ENV = ("HGB_FUSE_GEMM_RS", "HGB_FUSE_GEMM_AR", "HGB_FUSE_AG_GEMM")


def _excess(got, parts):
    """test_gpu_fused.py's bound: bf16 partials (half an ulp each) summed in fp32 and rounded once more -- |got - exact| <=
    (sum |part| + |exact|) * 2^-8 (+ accumulation-order noise).  -> the largest amount by which the error exceeds it (<= 0: within)"""
    want = sum(parts)
    tol = (sum(p.abs() for p in parts) + want.abs()) * 2 ** -8 * 1.01 + 1e-2
    return float(((got.float() - want).abs() - tol).max())


def _case(bg, mode, fused):
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend, set_backend
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    from hetu_galvatron_b200.core.runtime.tensor_parallel.layers import linear_with_grad_accumulation_and_async_allreduce as linear
    g = torch.Generator(device="cpu").manual_seed(7 + MODES.index(mode))
    X, W, dY = [(torch.randn(*shape, generator=g) * 0.5).to(torch.bfloat16).cuda() for shape in ((M, K), (N, K), (M, N))]
    Xf, Wf, dYf = X.float(), W.float(), dY.float()
    rows = [slice(r * M // P, (r + 1) * M // P) for r in range(P)]
    ks = [slice(r * K // P, (r + 1) * K // P) for r in range(P)]
    ns = [slice(r * N // P, (r + 1) * N // P) for r in range(P)]
    # per rank: (input, weight, dy, layer arguments) and the exact output / input-grad / weight-grad as lists of fp32 partials
    if mode in ("rs_out", "ar_out"):
        ins = [(X[:, ks[r]].reshape(S, B, K // P), W[:, ks[r]]) for r in range(P)]
        parts = [Xf[:, ks[q]] @ Wf[:, ks[q]].t() for q in range(P)]
        if mode == "rs_out":
            dys = [dY[rows[r]].reshape(S // P, B, N) for r in range(P)]
            want_out = [[t[rows[r]] for t in parts] for r in range(P)]
            args = dict(reduce_scatter_out=True)
        else:
            dys = [dY.reshape(S, B, N) for r in range(P)]
            want_out = [parts for r in range(P)]
            args = dict(allreduce_out=True)
        want_dx = [[dYf @ Wf[:, ks[r]]] for r in range(P)]
        want_dw = [[dYf.t() @ Xf[:, ks[r]]] for r in range(P)]
    else:
        parts = [dYf[:, ns[q]] @ Wf[ns[q]] for q in range(P)]
        dys = [dY[:, ns[r]].reshape(S, B, N // P) for r in range(P)]
        want_out = [[Xf @ Wf[ns[r]].t()] for r in range(P)]
        want_dw = [[dYf[:, ns[r]].t() @ Xf] for r in range(P)]
        if mode == "sp_gather":
            ins = [(X[rows[r]].reshape(S // P, B, K), W[ns[r]]) for r in range(P)]
            want_dx = [[t[rows[r]] for t in parts] for r in range(P)]
            args = dict(sequence_parallel=True)
        else:
            ins = [(X.reshape(S, B, K), W[ns[r]]) for r in range(P)]
            want_dx = [parts for r in range(P)]
            args = dict(async_grad_allreduce=True)
    ins = [tuple(t.contiguous().clone().requires_grad_(True) for t in pair) for pair in ins]
    dys = [d.contiguous() for d in dys]

    for env in FUSE_ENV:
        os.environ[env] = "force" if fused else "0"
    comms = bg.BgComm.local_world(P, device=0, arena_bytes=64 << 20)
    group = CommGroup(list(range(P)))
    bes = [CudaBackend(comm=cm) for cm in comms]
    for be in bes:
        be.reserve_staging(group, 2 * M * max(K, N))
    for cm in comms:
        cm.exchange()
    streams = [torch.cuda.Stream() for _ in range(P)]
    # grow the caching allocator before the ranks run: one large segment and a stock of small-pool ones
    big, small = torch.empty(1 << 30, dtype=torch.uint8, device="cuda"), [torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
                                                                          for _ in range(64)]
    del big, small
    torch.cuda.synchronize()

    def run(fn):
        out = []
        for r in range(P):
            set_backend(bes[r])
            with torch.cuda.stream(streams[r]):
                out.append(fn(r))
        torch.cuda.synchronize()
        for cm in comms:
            assert cm.error_flag() == 0, cm.error_info()
        return out

    try:
        outs = run(lambda r: linear(ins[r][0], ins[r][1], None, tp_group=group, **args))
        run(lambda r: outs[r].backward(dys[r]))
        rec = {"mode": mode, "fused": fused, "n_fused": [{k: v for k, v in be.n_fused.items() if v} for be in bes],
               "out_excess": max(_excess(outs[r].detach().reshape(-1, outs[r].shape[-1]), want_out[r]) for r in range(P)),
               "dx_excess": max(_excess(ins[r][0].grad.reshape(-1, ins[r][0].shape[-1]), want_dx[r]) for r in range(P)),
               "dw_excess": max(_excess(ins[r][1].grad, want_dw[r]) for r in range(P))}
    except Exception:
        print("LINEAR_ERROR_INFO " + json.dumps([cm.error_info() for cm in comms]), flush=True)
        raise
    finally:
        torch.cuda.synchronize()
        set_backend(None)
        for cm in comms:
            cm.close()
    return rec


def main():
    import hetu_galvatron_b200._bg as bg
    assert torch.cuda.is_available(), "needs a GPU"
    bg.lib()
    bg.set_tunable("timeout_ms", 20000)
    bg.set_tunable("comm_ctas", 16)
    for mode in MODES:
        for fused in (True, False):
            print("LINEAR_CASE " + json.dumps(_case(bg, mode, fused)), flush=True)
    print("LINEAR_DONE", flush=True)


if __name__ == "__main__":
    try:
        main()
    except Exception:
        traceback.print_exc()
        sys.exit(1)

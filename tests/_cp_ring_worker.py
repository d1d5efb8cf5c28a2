"""Worker for tests/test_cp_ring.py and tests/test_gpu_cp_ring.py: one rank of a context-parallel job with ``cp_comm="ring"``.

Mode "parity" (default) runs tests/_host_worker.py unchanged (the product against the single-process oracle on the global batch:
loss 5e-3, gradients 3e-2 rel-L2) -- on the CPU with the gloo backend extended by the ring's methods (tests/_cp_ring_ref.py) -- and
adds the number of ring pushes to the report (``ring_pushes``).
Mode "saved" (``_mode: "saved"``) runs ONE context-parallel attention forward of each path under saved_tensors_hooks and reports
the largest dimension of any tensor autograd keeps for backward, with the local and the whole sequence length."""
import json
import os
import sys
import traceback

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _saved(over):
    import _cp_ring_ref as cref
    from hetu_galvatron_b200.core.runtime.backend import set_backend
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    from hetu_galvatron_b200.core.runtime.tensor_parallel import transformer as tr
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo", rank=rank, world_size=world)
    set_backend(cref.CpRingOracleBackend())
    group = CommGroup(list(range(world)))
    b, s_full, n, ng, d = 1, over["seq"], 4, 2, 16
    s_loc = s_full // world
    g = torch.Generator().manual_seed(5 + rank)
    q, k, v = [torch.randn(b, s_loc, h, d, generator=g).bfloat16().requires_grad_(True) for h in (n, ng, ng)]
    report = {"s_loc": s_loc, "s_full": s_full}
    for name, fn in (("ring", lambda: tr._CpRingAttnFn.apply(q, k, v, group, d ** -0.5)),
                     ("allgather", lambda: tr._cp_attention(q, k, v, group, d ** -0.5))):
        shapes = []

        def pack(t):
            shapes.append(list(t.shape))
            return t
        with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
            out = fn()
        out.float().sum().backward()           # (the saved tensors are usable)
        report[name] = {"max_dim": max(max(sh) for sh in shapes if sh), "n_saved": len(shapes)}
    if rank == 0:
        print("HOST_TEST_REPORT " + json.dumps(report), flush=True)
    dist.barrier()
    dist.destroy_process_group()


def main():
    over = json.loads(os.environ["HOST_TEST_CONFIG"])
    if over.pop("_mode", "parity") == "saved":
        return _saved(over)
    use_cuda = os.environ.get("HOST_TEST_BACKEND", "oracle") == "cuda"
    if not use_cuda:
        import _cp_ring_ref as cref
        import oracle.gloo_backend
        oracle.gloo_backend.OracleBackend = cref.CpRingOracleBackend
    over["cp_comm"] = "ring"
    os.environ["HOST_TEST_CONFIG"] = json.dumps(over)
    import _host_worker
    report = _host_worker.main()
    if use_cuda:
        report["ring_pushes"] = report.get("fused_calls", {}).get("cp_ring", 0)
    else:
        from hetu_galvatron_b200.core.runtime.backend import get_backend
        report["ring_pushes"] = get_backend().n_fused.get("cp_ring", 0)
    if int(os.environ["RANK"]) == 0:
        print("HOST_TEST_REPORT " + json.dumps(report), flush=True)


if __name__ == "__main__":
    try:
        main()
    except Exception:
        traceback.print_exc()
        sys.exit(1)

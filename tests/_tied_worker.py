"""Worker for tests/test_tied_embeddings.py and tests/test_gpu_tied.py: one rank of tests/_family_worker.py's run (the GPT family
against the HF-pinned oracle), with two additions.
  * On the CPU the gloo oracle backend carries the deferred-clipping methods of tests/_clip_worker.py's ``ClipOracleBackend``, so the
    fused optimizer with ``clip_grad`` > 0 runs there too.
  * On GPUs rank 0's report also lists the tied gradient ranges the backend registered ([rank list, bytes]) and the largest staging
    buffer it reserved per rank list: the in-place exchange of the tied gradients must not need a staging buffer the matrix's size."""
import json
import os
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import _clip_worker
    import _family_worker
    import oracle.gloo_backend as gloo
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend
    gloo.OracleBackend = _clip_worker.ClipOracleBackend      # (this rank process only)
    registered, staging = [], {}
    register, reserve = CudaBackend.register_tied_grad, CudaBackend.reserve_staging

    def register_tied_grad(self, unit, param, group):
        buf = register(self, unit, param, group)
        registered.append([list(group.ranks), buf.nbytes])
        return buf

    def reserve_staging(self, group, nbytes):
        if group is not None and group.size > 1:
            key = ",".join(str(r) for r in group.ranks)
            staging[key] = max(staging.get(key, 0), int(nbytes))
        return reserve(self, group, nbytes)

    CudaBackend.register_tied_grad, CudaBackend.reserve_staging = register_tied_grad, reserve_staging
    rank = int(os.environ["RANK"])
    report = _family_worker.main()                           # (destroys the process group when it is done)
    if os.environ.get("HOST_TEST_BACKEND", "oracle") == "cuda":
        report = dict(report, tied_registered=registered, staging=staging)
    if rank == 0:
        print("HOST_TEST_REPORT " + json.dumps(report), flush=True)
    return report


if __name__ == "__main__":
    try:
        main()
    except Exception:
        traceback.print_exc()
        sys.exit(1)

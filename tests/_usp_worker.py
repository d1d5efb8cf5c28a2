"""Worker for tests/test_usp.py: tests/_host_worker.py with the token layout replaced by a wrong one (HGB_TEST_USP_LAYOUT=sp_first:
each sp rank's share is cut from the whole sequence first and zigzagged inside it).  Tokens, labels and RoPE rows all move to the
wrong layout together, so only the attention can tell.

The host worker's own parity assertions (loss against the oracle, then gradients) carry its report; this worker catches exactly
those and reports their numbers (``parity_failed``), so the test can tell a failed parity check from any other error, which still
fails the rank."""
import json
import os
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _parity_report(err):
    """the report dict a parity assertion of tests/_host_worker.py carries, or None for any other assertion"""
    arg = err.args[0] if err.args else None
    if isinstance(arg, tuple) and arg and isinstance(arg[0], dict):
        arg = arg[0]
    if isinstance(arg, dict) and {"loss", "ref_loss", "max_grad_err"} <= set(arg):
        return arg
    return None


def main():
    from hetu_galvatron_b200.llama_hf import LlamaModel_sequential, LlamaModel_tensor_parallel
    from hetu_galvatron_b200.core.runtime.redistribute import local_positions

    def sp_first(seq, cp=1, cp_rank=0, sp=1, sp_rank=0):
        n = seq // sp
        return local_positions(n, cp, cp_rank) + sp_rank * n

    assert os.environ.get("HGB_TEST_USP_LAYOUT") == "sp_first"
    LlamaModel_sequential.local_positions = sp_first
    LlamaModel_tensor_parallel.local_positions = sp_first
    import _host_worker
    try:
        report = dict(_host_worker.main(), parity_failed=False)
    except AssertionError as err:
        report = _parity_report(err)
        if report is None:
            raise
        report = {"parity_failed": True, "loss": report["loss"], "ref_loss": report["ref_loss"],
                  "max_grad_err": report["max_grad_err"]}
    if int(os.environ["RANK"]) == 0:
        print("HOST_TEST_REPORT " + json.dumps(report), flush=True)
    return report


if __name__ == "__main__":
    try:
        main()
    except Exception:
        traceback.print_exc()
        sys.exit(1)

"""Worker for tests/test_gpt_cp.py and tests/test_gpu_gpt_cp.py: one rank of a GPT job with context parallelism.

It runs tests/_family_worker.py unchanged (the product against the single-process oracle on the global batch: loss 5e-3, gradients
3e-2 rel-L2, the loss after one AdamW step) -- through tests/_dropout_worker.py's oracle patch when the spec has dropout, and on the CPU
with the gloo backend extended by the ring's methods (tests/_cp_ring_ref.py) when ``cp_comm`` is "ring" -- and checks on EVERY rank:
  * the split is real: each GPT layer's input has s / (cp x Ulysses x Megatron-SP degree) rows, the degrees of its row of the strategy;
  * the context-parallel attention keeps nothing for backward with a dimension beyond s/c under the ring (reported, with the largest
    such dimension, for both exchanges).
Config keys of this worker: ``_strategy_json`` (a strategy dict, as tests/_host_worker.py takes it)."""
import json
import os
import sys
import traceback

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _backend_class(ring, dropout):
    import _cp_ring_ref as cref
    import _dropout_ref as dref
    from oracle.gloo_backend import OracleBackend
    bases = tuple(b for b, on in ((cref.CpRingOracleBackend, ring), (dref.DropoutOracleBackend, dropout)) if on) or (OracleBackend,)
    return type("GptCpOracleBackend", bases, {})


def _instrument(seen):
    """record the rows of every GPT layer's input and the largest dimension autograd keeps inside the cp attention"""
    from hetu_galvatron_b200 import gpt_hf
    from hetu_galvatron_b200.gpt_hf.GPTModel_tensor_parallel import GPTLayer_tp
    from hetu_galvatron_b200.core.runtime.tensor_parallel import transformer as tr
    build = gpt_hf.gpt_model_hp

    def hooked(*a, **k):
        model = build(*a, **k)
        seen["hp"] = model.hp_configs_whole
        for m in model.modules():
            if isinstance(m, GPTLayer_tp):
                m.register_forward_pre_hook(lambda mod, inp: seen["rows"].setdefault(mod.idx, set()).add(int(inp[0].shape[0])))
        return model
    gpt_hf.gpt_model_hp = hooked
    inner = tr.cp_attention

    def cp_attention(q, k, v, group, scale, comm):
        def pack(t):
            if t.dim() > 0:
                seen["saved_max_dim"] = max(seen["saved_max_dim"], max(t.shape))
            return t
        seen["cp_calls"] += 1
        with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
            return inner(q, k, v, group, scale, comm)
    tr.cp_attention = cp_attention


def main():
    over = json.loads(os.environ["HOST_TEST_CONFIG"])
    use_cuda = os.environ.get("HOST_TEST_BACKEND", "oracle") == "cuda"
    spec = over.get("_spec", {})
    dropout = any(spec.get(k, 0.0) > 0.0 for k in ("resid_pdrop", "embd_pdrop", "attn_pdrop"))
    ring = over.get("cp_comm", "allgather") == "ring"
    strategy = over.pop("_strategy_json", None)
    if strategy is not None:
        over["galvatron_config_path"] = strategy
    if dropout:
        import _dropout_worker
        _dropout_worker._patch(over)
    if not use_cuda:
        import oracle.gloo_backend
        oracle.gloo_backend.OracleBackend = _backend_class(ring, dropout)
    seen = {"rows": {}, "saved_max_dim": 0, "cp_calls": 0}
    _instrument(seen)
    os.environ["HOST_TEST_CONFIG"] = json.dumps(over)
    import _family_worker
    report = _family_worker.main()
    hp, seq = seen["hp"], int(over.get("seq_length", 0)) or _family_worker.TINY["gpt"]["n_positions"]
    seq = int(spec.get("n_positions", seq))
    want = {}
    for i, rows in seen["rows"].items():
        row = i + 1             # whole-model rows: [embed, layer_0 .., norm, cls]
        tp, cp, sp = hp["tp_sizes_whole"][row], hp["cp_sizes_whole"][row], hp["sp_sizes_whole"][row]
        split = cp * (sp if sp > 1 else (tp if over.get("sequence_parallel") else 1))
        want[i] = seq // split
        assert rows == {want[i]}, "layer %d sees %s rows, want s / %d = %d" % (i, sorted(rows), split, want[i])
    cps = {hp["cp_sizes_whole"][i + 1] for i in seen["rows"]}
    report.update(layer_rows={str(i): sorted(r) for i, r in seen["rows"].items()}, seq=seq, layer_cp=sorted(cps),
                  saved_max_dim=seen["saved_max_dim"], cp_calls=seen["cp_calls"])
    if ring and max(cps) > 1:
        bound = seq // max(cps)
        assert seen["saved_max_dim"] <= bound, "the ring kept a tensor with a dimension of %d > s/c = %d" % (seen["saved_max_dim"], bound)
    if use_cuda:
        report["ring_pushes"] = report.get("fused_calls", {}).get("cp_ring", 0)
    else:
        from hetu_galvatron_b200.core.runtime.backend import get_backend
        report["ring_pushes"] = getattr(get_backend(), "n_fused", {}).get("cp_ring", 0)
    if int(os.environ["RANK"]) == 0:
        print("HOST_TEST_REPORT " + json.dumps(report), flush=True)
    return report


if __name__ == "__main__":
    try:
        main()
    except Exception:
        traceback.print_exc()
        sys.exit(1)

"""Worker for tests/test_dropout.py and tests/test_gpu_dropout.py: one rank of a GPT / BERT job with dropout on.

Mode "parity" runs tests/_family_worker.py unchanged (the product against the single-process oracle on the global batch: loss 5e-3,
gradients 3e-2 rel-L2, the loss after one AdamW step) with the dropout probabilities in the model spec, the CPU backend extended by
the dropout methods (tests/_dropout_ref.py) and the oracle replaced by its dropout restatement, drawing the same masks: iteration 0
for the step's forward, 1 for the forward after the optimizer step.  Config keys of this worker:
  _oracle_sample_shift / _oracle_position_shift  deliberately wrong oracle coordinates (the check must then fail)
  _check_replicas                                assert every layer's output is bit-identical on all ranks of the job
Mode "loss" (``_mode: "loss"``) runs one training step and reports its loss only (attention-probability dropout, whose masks are
torch's and have no oracle counterpart)."""
import json
import os
import sys
import traceback

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _patch(over):
    import _dropout_ref as dref
    import oracle.gloo_backend
    from oracle import gpt_bert_ref
    oracle.gloo_backend.OracleBackend = dref.DropoutOracleBackend
    family, spec = over["_family"], dict(over.get("_spec", {}))
    if family == "gpt":
        hidden, attention = spec.get("resid_pdrop", 0.0), spec.get("attn_pdrop", 0.0)
    else:
        hidden, attention = spec.get("hidden_dropout_prob", 0.0), spec.get("attention_probs_dropout_prob", 0.0)
    seed = over.get("seed", 1234)
    sample_shift, position_shift = over.pop("_oracle_sample_shift", 0), over.pop("_oracle_position_shift", 0)
    calls = [0]

    def drop():
        d = dref.Drop(hidden, attention, seed, iteration=calls[0], sample_base=sample_shift, position_shift=position_shift)
        calls[0] += 1
        return d

    gpt_bert_ref.gpt_forward_loss = lambda w, tokens, labels, cfg, dtype=torch.bfloat16: dref.gpt_forward_loss(w, tokens, labels, cfg,
                                                                                                              drop(), dtype)
    gpt_bert_ref.bert_forward_loss = (lambda w, tokens, labels, cfg, dtype=torch.bfloat16, attention_mask=None, token_type_ids=None:
                                      dref.bert_forward_loss(w, tokens, labels, cfg, drop(), dtype, attention_mask, token_type_ids))
    if over.pop("_check_replicas", False):
        _check_replicas(family)


def _check_replicas(family):
    """Every transformer layer's output of the first forward, compared bit for bit across all ranks (at the oracle's first call,
    while the process group is up)."""
    import _dropout_ref  # noqa: F401
    from oracle import gpt_bert_ref
    from hetu_galvatron_b200 import bert_hf, gpt_hf
    mod = gpt_hf if family == "gpt" else bert_hf
    layer_cls = gpt_hf.GPTModel_tensor_parallel.GPTLayer_tp if family == "gpt" else bert_hf.BertModel_tensor_parallel.BertLayer_tp
    name = "gpt_model_hp" if family == "gpt" else "bert_model_hp"
    build, outs = getattr(mod, name), {}

    def hooked(*a, **k):
        model = build(*a, **k)
        def keep(name):
            def hook(module, inputs, out):       # (returns None: the output itself is left alone)
                outs.setdefault(name, out.detach().float().cpu().clone())
            return hook
        for n, m in model.named_modules():
            if isinstance(m, layer_cls):
                m.register_forward_hook(keep(n))
        return model
    setattr(mod, name, hooked)
    fn_name = "%s_forward_loss" % family
    inner = getattr(gpt_bert_ref, fn_name)

    def compare(*a, **k):
        if outs:
            allo = [None] * dist.get_world_size()
            dist.all_gather_object(allo, outs)
            for n, t in outs.items():
                for other in allo:
                    assert torch.equal(other[n], t), "layer %s differs between replicas" % n
            print("REPLICAS_BIT_IDENTICAL %d layers" % len(outs), flush=True)
            outs.clear()
        return inner(*a, **k)
    setattr(gpt_bert_ref, fn_name, compare)


def _loss_only(over):
    """One forward_backward of the family with the given args; rank 0 prints the mean loss."""
    import smoke_model as sm
    from hetu_galvatron_b200.core.runtime.backend import get_backend, reset_backend, set_backend
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    use_cuda = os.environ.get("HOST_TEST_BACKEND", "oracle") == "cuda"
    family = over.pop("_family")
    spec = dict({"gpt": dict(n_layer=2, n_embd=128, n_head=4, vocab_size=512, n_positions=64),
                 "bert": dict(hidden_size=128, num_hidden_layers=2, num_attention_heads=4, vocab_size=512, max_position_embeddings=64,
                              layer_norm_eps=1e-5)}[family], **over.pop("_spec", {}))
    over.pop("_mode")
    if use_cuda:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", torch.cuda.current_device()))
        os.environ.setdefault("HGB_ARENA_BYTES", str(256 << 20))
        dev = get_backend().device
    else:
        import _dropout_ref as dref
        dist.init_process_group("gloo", rank=rank, world_size=world)
        set_backend(dref.DropoutOracleBackend())
        dev = torch.device("cpu")
    torch.manual_seed(0)
    args = sm.tiny_args(**over)
    if family == "gpt":
        from hetu_galvatron_b200.gpt_hf import config_from_meta, gpt_model_hp as build, set_model_config
    else:
        from hetu_galvatron_b200.bert_hf import bert_model_hp as build, config_from_meta, set_model_config
    config = set_model_config(config_from_meta(spec), args)
    model = build(config, args)
    gbs, seq = args.global_train_batch_size, config.max_position_embeddings
    dp_idx, dp = model.vtp_data_group.rank_in_group(rank), model.vtp_data_group.size
    x = torch.randint(0, config.vocab_size, (gbs, seq + 1), generator=torch.Generator().manual_seed(11))
    lo, hi = dp_idx * gbs // dp, (dp_idx + 1) * gbs // dp
    loss = model.forward_backward([x[lo:hi, :-1].contiguous().to(dev)], 0, None, loss_func=None, labels=x[lo:hi, 1:].contiguous().to(dev),
                                  attention_mask=None)
    lt = torch.tensor([loss if loss is not None else 0.0, 1.0 if loss is not None else 0.0], dtype=torch.float64, device=dev)
    dist.all_reduce(lt)
    if rank == 0:
        print("HOST_TEST_REPORT " + json.dumps(dict(loss=float(lt[0] / lt[1]))), flush=True)
    dist.barrier()
    if use_cuda:
        reset_backend()
    dist.destroy_process_group()


def main():
    over = json.loads(os.environ["HOST_TEST_CONFIG"])
    if over.get("_mode") == "loss":
        return _loss_only(over)
    _patch(over)
    os.environ["HOST_TEST_CONFIG"] = json.dumps(over)
    import _family_worker
    return _family_worker.main()


if __name__ == "__main__":
    try:
        main()
    except Exception:
        traceback.print_exc()
        sys.exit(1)

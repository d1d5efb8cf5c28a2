"""Worker for tests/test_dropout_relocation.py: one rank of a GPT / BERT / ViT job whose layers hold other samples than the vocabulary
rows (a relocation split or gathered the batch), with hidden dropout on.

``RelocationOracleBackend`` / ``RelocationViTOracleBackend``: the gloo backends of tests/_dropout_ref.py and tests/_vit_backend.py plus
``dropout_add_fwd_ids`` / ``dropout_bwd_ids`` of ``CudaBackend`` restated on the CPU (``keep_mask`` at the listed samples).

Modes (config key ``_mode``):
  "parity" (default)  tests/_dropout_worker.py's parity run (GPT / BERT) or tests/_vit_worker.py's (ViT) on these backends: the product
                      against the single-process oracle on the global batch, which draws every mask at the true global sample.
                      ``_old_numbering``: every row draws at the embedding's numbering, sample_base + local index, as if no
                      relocation had moved the batch (the parity check must then fail).
                      ``_no_padding_mask``: BERT without its key-padding mask, in the product and in the oracle (a per-microbatch
                      keyword argument that, as in the reference, relocations do not move: a layer holding a re-split batch
                      cannot take it).
  "ids"               every sample of the global batch carries its own index as its value (the tokens, then every row's output), so
                      the activation entering each row after the real relocation / pipeline path says which samples the row holds;
                      compared, at every row and microbatch (and at the recompute of checkpointed rows), with the sample ids the
                      dropout context derived for that row.
"""
import json
import os
import sys
import traceback

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _dropout_ref as dref  # noqa: E402


class _IdsMixin:
    """The sample-map dropout pair, restated: row r of x [s, b, h] is sample sample_ids[r % b]."""

    def dropout_add_fwd_ids(self, x, bias, residual, p, seed, iteration, site, seq_base, sample_ids):
        s, b, h = x.shape
        assert sample_ids.dtype == torch.int32 and sample_ids.shape == (b,)
        keep = dref.keep_mask(seed, iteration, site, seq_base + np.arange(s), sample_ids.numpy().astype(np.uint32), h, p)
        return dref.dropout_add_ref(x, bias, residual, keep, p, dtype=x.dtype)

    def dropout_bwd_ids(self, dy, p, seed, iteration, site, seq_base, sample_ids, with_bias):
        s, b, h = dy.shape
        assert sample_ids.dtype == torch.int32 and sample_ids.shape == (b,)
        keep = dref.keep_mask(seed, iteration, site, seq_base + np.arange(s), sample_ids.numpy().astype(np.uint32), h, p)
        dx, db = dref.dropout_bwd_ref(dy, keep, p)
        return dx, (db if with_bias else None)


class RelocationOracleBackend(_IdsMixin, dref.DropoutOracleBackend):
    pass


def _vit_backend_class():
    from _vit_backend import ViTOracleBackend

    class RelocationViTOracleBackend(_IdsMixin, ViTOracleBackend):
        pass
    return RelocationViTOracleBackend


def _strategy(over):
    """``_strategy``: a strategy JSON in the reference's format (a file under tests/golden, or inline), ``_strategy_over`` overriding
    some of its keys."""
    strategy = over.pop("_strategy", None)
    if strategy is not None:
        if isinstance(strategy, str):
            with open(os.path.join(ROOT, strategy)) as f:
                strategy = json.load(f)
        over["galvatron_config_path"] = dict(strategy, **over.pop("_strategy_over", {}))


def _old_numbering():
    from hetu_galvatron_b200.core.runtime.tensor_parallel import random as drandom
    drandom._row_sample = lambda ctx, row, x: ctx.sample_base


def _drop_padding_mask():
    from oracle import gpt_bert_ref
    from hetu_galvatron_b200 import bert_hf
    build, oracle_loss = bert_hf.bert_model_hp, gpt_bert_ref.bert_forward_loss

    def build_without_mask(*a, **k):
        model = build(*a, **k)
        fb = model.forward_backward
        model.forward_backward = lambda *fa, **fk: fb(*fa, **dict(fk, attention_mask=None))
        return model
    bert_hf.bert_model_hp = build_without_mask
    gpt_bert_ref.bert_forward_loss = lambda *a, **k: oracle_loss(*a, **dict(k, attention_mask=None))


def _parity(over):
    if over.pop("_old_numbering", False):
        _old_numbering()
    if over["_family"] == "vit":
        over.pop("_family")
        import _vit_backend
        _vit_backend.ViTOracleBackend = _vit_backend_class()
        os.environ["HOST_TEST_CONFIG"] = json.dumps(over)
        import _vit_worker
        return _vit_worker.main()
    import _dropout_worker
    import oracle.gloo_backend
    no_mask = over.pop("_no_padding_mask", False)
    _dropout_worker._patch(over)
    oracle.gloo_backend.OracleBackend = RelocationOracleBackend
    if no_mask:
        _drop_padding_mask()
    os.environ["HOST_TEST_CONFIG"] = json.dumps(over)
    import _family_worker
    return _family_worker.main()


def _ids(over):
    import smoke_model as sm
    from hetu_galvatron_b200.core.runtime.backend import set_backend
    from hetu_galvatron_b200.core.runtime.parallel import DataParallelModule, Module_with_relocation
    from hetu_galvatron_b200.core.runtime.tensor_parallel import random as drandom
    from _family_worker import TINY
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    family = over.pop("_family")
    spec = dict(TINY[family], **over.pop("_spec", {}))
    over.pop("_no_padding_mask", None)             # (this mode runs without a padding mask)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    set_backend(RelocationOracleBackend())
    args = sm.tiny_args(**over)
    if family == "gpt":
        from hetu_galvatron_b200.gpt_hf import config_from_meta, gpt_model_hp as build, set_model_config
    else:
        from hetu_galvatron_b200.bert_hf import bert_model_hp as build, config_from_meta, set_model_config
    config = set_model_config(config_from_meta(spec), args)
    model = build(config, args)
    gbs, seq = args.global_train_batch_size, config.max_position_embeddings
    assert gbs <= 256 and gbs < config.vocab_size          # every sample index is a token and a bf16 integer
    stats = dict(checks=0, rows=set(), mapped=0, bad=[])

    def check(row, held):
        want = drandom.row_samples(row)
        stats["checks"] += 1
        stats["rows"].add(row)
        if want is None or held != want:
            stats["bad"].append((rank, row, held, want))
        elif want != list(range(want[0], want[0] + len(want))):
            stats["mapped"] += 1

    def pre_hook(row):
        def hook(module, inputs):
            x = inputs[0]
            held = x[:, 0] if not x.is_floating_point() else x[0, :, 0]     # tokens [b, s]; activations [s, b, h]
            check(row, [int(v) for v in held.float().round().tolist()])
        return hook

    def carry(row):
        def hook(module, inputs, out):                   # the row's output carries the sample indices on
            x = inputs[0]
            ids = x[:, 0].to(out.dtype)[None, :, None] if not x.is_floating_point() else x
            return out * 0 + ids
        return hook

    last = len(model.hp_configs_whole["tp_sizes_whole"]) - 1       # the head: its loss is left as it is
    for m in model.model.model_cur_stage:
        assert isinstance(m, DataParallelModule)
        row = int(m.unit.name.rsplit("_", 1)[1])
        inner = m.module.module if isinstance(m.module, Module_with_relocation) else m.module
        inner.register_forward_pre_hook(pre_hook(row))
        if row != last:
            inner.register_forward_hook(carry(row))
    sample = torch.arange(gbs)[:, None].expand(gbs, seq).contiguous()
    dp_group = model.vtp_data_group
    dp_idx, dp = dp_group.rank_in_group(rank), dp_group.size
    lo, hi = dp_idx * gbs // dp, (dp_idx + 1) * gbs // dp
    model.forward_backward([sample[lo:hi]], 0, None, loss_func=None, labels=sample[lo:hi].clone(), attention_mask=None)
    allst = [None] * world
    dist.all_gather_object(allst, dict(stats, rows=sorted(stats["rows"])))
    report = dict(checks=sum(s["checks"] for s in allst), mapped=sum(s["mapped"] for s in allst),
                  rows=len(set(r for s in allst for r in s["rows"])), bad=[b for s in allst for b in s["bad"]][:4])
    assert not report["bad"], report
    if rank == 0:
        print("HOST_TEST_REPORT " + json.dumps(report), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    return report


def main():
    over = json.loads(os.environ["HOST_TEST_CONFIG"])
    if over.pop("_mode", "parity") == "ids":
        _strategy(over)
        return _ids(over)
    _strategy(over)
    return _parity(over)


if __name__ == "__main__":
    try:
        main()
    except Exception:
        traceback.print_exc()
        sys.exit(1)

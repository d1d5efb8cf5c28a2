"""Hidden dropout under per-layer strategies whose relocations re-split the batch (CPU, gloo).

When a layer's tensor-parallel degree differs from its predecessor's, the relocation gathers or splits the batch between ranks, so
the layer holds other samples than the vocabulary rows (sample_layout.py).  Checked here:
  * the derived sample layouts against closed-form expectations, and a strided-TP grouping change (same degree, other ranks),
    which the strategy checks refuse, so no layer can hold the same number of samples as the vocabulary rows but other ones;
  * N ranks on the gloo backend against the single-process oracle, which draws every mask at the true global sample (hidden dropout
    0.1: loss 5e-3 rel, every gradient 3e-2 rel-L2, the loss after one AdamW step), for gathers, splits, mixed per-layer degrees,
    Megatron-SP, Ulysses, a pipeline boundary with checkpointing, and the reference's BERT-base and GPT-2.7B strategy JSONs;
  * that the check has teeth: drawing every row at the embedding's numbering fails it;
  * that the derived ids are what the real relocation / pipeline path delivers: a batch whose values are the sample indices, moved
    through the model, matches the derived ids at every row and microbatch.
"""
import json
import os
import sys
from fractions import Fraction

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

BERT_BASE_JSON = "tests/golden/bert_base_tp2_vtp1_8gpus.json"
GPT_2_7B_JSON = "tests/golden/gpt_2.7b_pp2_8gpus.json"
_PORT = [30300]

GPT_DROP = dict(resid_pdrop=0.1, embd_pdrop=0.1, attn_pdrop=0.0)
BERT_DROP = dict(hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.0)


def row_strategy(tps, pp_division, chunks, gbs, checkpoint=None, vtp=1, consec=None):
    j = lambda v: ",".join(str(x) for x in v)  # noqa: E731
    n = len(tps)
    return {"pp_deg": len(pp_division), "tp_sizes_enc": j(tps), "tp_consecutive_flags": j(consec or [1] * n),
            "dp_types_enc": j([0] * n), "use_sp": j([0] * n), "checkpoint": j(checkpoint or [0] * n), "global_bsz": gbs,
            "chunks": chunks, "pp_division": j(pp_division), "pipeline_type": "pipedream_flush", "default_dp_type": "zero2",
            "vtp": vtp, "vsp": 0}


CASES = {
    # vocabulary rows at tp 1, layers at tp 2: each layer gathers the two data-parallel ranks' microbatches
    "gpt_gather_chunks1": (2, dict(_family="gpt", _spec=GPT_DROP, global_tp_deg=2, vocab_tp=1, global_train_batch_size=4)),
    "gpt_gather_chunks2": (2, dict(_family="gpt", _spec=GPT_DROP, global_tp_deg=2, vocab_tp=1, chunks=2, global_train_batch_size=8)),
    # vocabulary rows at tp 2, layers at tp 1: each layer keeps half of the shared microbatch
    "gpt_split": (2, dict(_family="gpt", _spec=GPT_DROP, global_tp_deg=1, vocab_tp=2, global_train_batch_size=4)),
    "gpt_layers_tp1212_chunks2": (2, dict(_family="gpt", _spec=dict(GPT_DROP, n_layer=4), chunks=2, global_train_batch_size=8,
                                          _strategy=row_strategy([1, 2, 1, 2], [4], 2, 8))),
    "gpt_gather_megatron_sp": (2, dict(_family="gpt", _spec=GPT_DROP, global_tp_deg=2, vocab_tp=1, sequence_parallel=True, chunks=2,
                                       global_train_batch_size=8)),
    "gpt_gather_ulysses": (2, dict(_family="gpt", _spec=GPT_DROP, global_tp_deg=2, use_ulysses=True, vocab_tp=1, sequence_parallel=True,
                                   chunks=2, global_train_batch_size=8)),
    # PP2 1F1B: stage 0 at tp 1 (with the vocabulary rows), stage 1 at tp 2, relocated layers checkpointed
    "gpt_pp2_tp_changes_at_boundary_ckpt": (4, dict(_family="gpt", _spec=dict(GPT_DROP, n_layer=4), chunks=4, global_train_batch_size=16,
                                                    _strategy=row_strategy([1, 1, 2, 2], [2, 2], 4, 16, checkpoint=[0, 0, 1, 1]))),
    # (unpadded: the key-padding mask is a per-microbatch keyword argument that relocations do not move, as in the reference)
    "bert_reference_base_json": (8, dict(_family="bert", _spec=dict(BERT_DROP, num_hidden_layers=12), _strategy=BERT_BASE_JSON,
                                         _strategy_over=dict(global_bsz=16), _no_padding_mask=True)),
    "gpt_reference_2.7b_json": (8, dict(_family="gpt", _spec=dict(GPT_DROP, n_layer=32), _strategy=GPT_2_7B_JSON,
                                        _strategy_over=dict(global_bsz=32))),
}
VIT_CASE = (2, dict(_family="vit", _spec=dict(hidden_dropout_prob=0.1), global_tp_deg=2, vocab_tp=1, global_train_batch_size=4))


def launch(world, config, backend="oracle", timeout=1500):
    from _launch import launch_ranks
    _PORT[0] += 1
    return launch_ranks("_dropout_relocation_worker", world, config, _PORT[0] + os.getpid() % 500, timeout=timeout, backend=backend)


# ---- the derived layouts -------------------------------------------------------------------------------------------------------
def _layouts(tps, world, pp_division=None, vtp=1, consec=None, sp=None):
    from hetu_galvatron_b200.core.runtime.sample_layout import derive_sample_layouts
    n = len(tps) + 3        # embedding, layers, norm, head (the GPT rows)
    pp_division = pp_division or [len(tps)]
    stages = [0]
    for s, k in enumerate(pp_division):
        stages += [s] * k
    stages += [len(pp_division) - 1] * 2
    whole = dict(tp_sizes_whole=[vtp] + list(tps) + [vtp, vtp], sp_sizes_whole=[1] * n if sp is None else sp,
                 cp_sizes_whole=[1] * n, tp_consec_whole=[1] + list(consec or [1] * len(tps)) + [1, 1], pp_deg=len(pp_division),
                 pp_ranks_whole=stages)
    return [derive_sample_layouts(whole, r, world) for r in range(world)]


F0, F1, FH = Fraction(0), Fraction(1), Fraction(1, 2)


def test_layouts_gather_and_split():
    lay = _layouts([2, 2], 2)
    assert [l[0] for l in lay] == [((0, F0, F1),), ((1, F0, F1),)]          # the embedding: the data-parallel split
    assert lay[0][1] == lay[1][1] == lay[0][2] == ((0, F0, F1), (1, F0, F1))  # tp 2: both microbatches, rank order
    assert [l[3] for l in lay] == [((0, F0, F1),), ((1, F0, F1),)]          # back at tp 1: split again
    lay = _layouts([1], 2, vtp=2)
    assert [l[1] for l in lay] == [((0, F0, FH),), ((0, FH, F1),)]          # vocabulary rows at tp 2: one shared microbatch, halved


def test_layouts_cross_pipeline_stages():
    lay = _layouts([1, 1, 2, 2], 4, pp_division=[2, 2])
    # stage 1 = ranks 2, 3: at tp 2 they gather what ranks 0 and 1 (data-parallel indices 0 and 1) sent them
    assert lay[2][3] == lay[3][3] == ((0, F0, F1), (1, F0, F1))
    assert 3 not in lay[0] and 0 not in lay[2]


def test_layouts_instantiate_runs():
    from hetu_galvatron_b200.core.runtime.sample_layout import instantiate
    gathered = ((0, F0, F1), (1, F0, F1))
    assert instantiate(gathered, 8, 0, 8) == list(range(16))                             # one microbatch: contiguous
    assert instantiate(gathered, 8, 4, 4) == [4, 5, 6, 7, 12, 13, 14, 15]                # microbatch 1 of 2: two runs
    assert instantiate(((0, FH, F1),), 4, 0, 4) == [2, 3]
    with pytest.raises(ValueError, match="unequal"):
        instantiate(((0, FH, F1),), 4, 0, 3)


def test_grouping_only_change_is_refused():
    """Same tensor-parallel degree, other ranks (tp_consecutive_flags 0 against the vocabulary rows' 1): the layer would hold as many
    samples as the vocabulary rows but other ones.  Strided TP has no runtime path, so the strategy is refused before any layer
    exists, and with consecutive groups a layer of unchanged degree keeps its predecessor's samples."""
    with pytest.raises(ValueError, match="strided TP"):
        _layouts([2, 2], 4, consec=[0, 0])
    lay = _layouts([2, 2], 4, vtp=2)
    assert all(l[1] == l[0] and l[2] == l[0] for l in lay)


def test_golden_strategies_are_the_reference_search_engine_output():
    with open(os.path.join(ROOT, BERT_BASE_JSON)) as f:
        b = json.load(f)
    assert (b["tp_sizes_enc"], b["vtp"], b["global_bsz"], b["pp_deg"]) == (",".join(["2"] * 12), 1, 128, 1)
    with open(os.path.join(ROOT, GPT_2_7B_JSON)) as f:
        g = json.load(f)
    assert "vtp" not in g and (g["pp_deg"], g["chunks"], g["global_bsz"], g["pp_division"]) == (2, 4, 64, "16,16")
    assert g["tp_sizes_enc"] == "2,2,2,2,2,2,2,2,2,1,1,1,1,1,1,1,2,2,2,2,2,2,2,2,2,2,1,1,1,1,1,1"


# ---- N ranks against the oracle ------------------------------------------------------------------------------------------------
def _check(rep):
    assert rep["max_grad_err"] < 3e-2
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_relocated_dropout_matches_the_oracle(name):
    world, cfg = CASES[name]
    _check(launch(world, dict(cfg)))


def test_vit_relocated_dropout_matches_the_oracle():
    world, cfg = VIT_CASE
    _check(launch(world, dict(cfg)))


def test_old_numbering_fails_the_parity_check():
    """The check has teeth: a relocated layer that draws at the embedding's numbering (sample_base + local index) misses it."""
    world, cfg = CASES["gpt_gather_chunks2"]
    with pytest.raises(AssertionError, match="max_grad_err|loss"):
        launch(world, dict(cfg, _old_numbering=True))


@pytest.mark.parametrize("name", sorted(CASES))
def test_relocation_delivers_the_derived_sample_ids(name):
    world, cfg = CASES[name]
    cfg = dict(cfg, _mode="ids", _spec={k: v for k, v in cfg["_spec"].items() if "drop" not in k})
    rep = launch(world, cfg)
    assert rep["checks"] > 0 and not rep["bad"]
    if name not in ("gpt_gather_chunks1", "gpt_split", "bert_reference_base_json"):
        assert rep["mapped"] > 0                    # some row held samples that are not one run of consecutive indices

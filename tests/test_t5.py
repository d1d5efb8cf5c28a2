"""The T5 family (galvatron/models/T5) on the product's core: N ranks over gloo run the family's layers / schedules on the CPU
restatement of its kernels and must reproduce the single-process oracle (oracle/t5_ref.py, pinned to HF T5 here) on the global
batch -- loss 5e-3 rel, per-parameter gradients 3e-2 rel-L2, and the loss after one AdamW step.  Tiny model: d_model 64, inner
width 4 x 32 = 128, ffn 128, vocabulary 256, encoder 32 tokens, decoder 16, 2 + 2 layers unless stated."""
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
_PORT = [30350]

T5_3B_JSON = "tests/golden/t5_3b_dp8_8gpus.json"


def launch(world, config, timeout=1800, backend="oracle"):
    from _launch import launch_ranks
    _PORT[0] += 1
    return launch_ranks("_t5_worker", world, config, _PORT[0] + os.getpid() % 500, timeout=timeout, backend=backend)


def row_strategy(tps, pp_division, chunks, gbs, pipeline_type="pipedream_flush", vtp=1, checkpoint=0):
    """A strategy in the reference Search Engine's format with one tp degree per t5_enc / t5_dec layer."""
    n = len(tps)
    j = lambda v: ",".join(str(x) for x in v)  # noqa: E731
    return {"pp_deg": len(pp_division), "tp_sizes_enc": j(tps), "tp_consecutive_flags": j([1] * n), "dp_types_enc": j([0] * n),
            "use_sp": j([0] * n), "checkpoint": j([checkpoint] * n), "global_bsz": gbs, "chunks": chunks, "pp_division": j(pp_division),
            "pipeline_type": pipeline_type, "default_dp_type": "zero2", "vtp": vtp, "vsp": 0}


# name -> (world, worker config)
CASES = {
    "world1": (1, dict(global_train_batch_size=4)),
    "world1_ckpt": (1, dict(global_train_batch_size=4, global_checkpoint=1)),
    "dp2_zero2": (2, dict(global_train_batch_size=8)),
    "dp2_zero3_ckpt": (2, dict(global_train_batch_size=8, sdp=1, global_checkpoint=1)),
    "tp2": (2, dict(global_tp_deg=2, vocab_tp=2, global_train_batch_size=4)),
    "tp2_megatron_sp": (2, dict(global_tp_deg=2, vocab_tp=2, global_train_batch_size=4, sequence_parallel=True)),
    # decoder row 0 at tp 1 (dp 2), decoder row 1 at tp 2: both boundary tensors are relocated between two decoder rows
    "tp_changes_between_decoder_rows": (2, dict(_strategy=row_strategy([1, 1, 1, 2], [4], 1, 8))),
    # layers at tp 1 (dp 2), the vocabulary rows at tp 2: relocations at embed_1 -> enc 0, enc 1 -> pre_norm_1 and embed_2 -> dec 0
    "vocab_tp_differs_from_layer_tp": (2, dict(_strategy=row_strategy([1, 1, 1, 1], [4], 1, 8, vtp=2))),
    # 7 samples in 3 micro-batches (3, 3, 1)
    "pp2_1f1b_split_at_encoder_decoder_boundary": (2, dict(_strategy=row_strategy([1] * 4, [2, 2], 3, 7))),
    "pp2_gpipe_split_inside_decoder": (2, dict(_strategy=row_strategy([1] * 4, [3, 1], 3, 7, pipeline_type="gpipe"))),
    "pp4_splits_in_both_halves": (4, dict(_strategy=row_strategy([1] * 4, [1, 1, 1, 1], 3, 7))),
    # checkpoint recompute of decoder rows at a two-tensor boundary (their cross K / V recomputed from the saved encoder input)
    "pp2_1f1b_split_inside_decoder_ckpt": (2, dict(_strategy=row_strategy([1] * 4, [3, 1], 3, 7, checkpoint=1))),
    # labels -1 on the padding of every decoder sequence, the reference's masked-mean loss, 2 micro-batches
    "masked_padding_labels": (1, dict(global_train_batch_size=4, chunks=2, _masked=True)),
    "masked_padding_labels_tp2": (2, dict(global_tp_deg=2, vocab_tp=2, global_train_batch_size=4, _masked=True)),
    # the reference's t5-3B strategy (dp 8, zero3 / zero2 mix, checkpointing) on 24 + 24 tiny layers, global batch 1024 -> 16
    "reference_t5_3b_json": (8, dict(_strategy=T5_3B_JSON, _strategy_over=dict(global_bsz=16),
                                     _spec=dict(num_layers=24, num_decoder_layers=24))),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_t5_family(name):
    world, cfg = CASES[name]
    rep = launch(world, dict(cfg))
    assert rep["max_grad_err"] < 3e-2
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])


def test_golden_strategy_is_the_reference_search_engine_output():
    with open(os.path.join(ROOT, T5_3B_JSON)) as f:
        s = json.load(f)
    assert s["tp_sizes_enc"] == ",".join(["1"] * 48) and s["pp_division"] == "48" and s["pp_deg"] == 1
    assert s["dp_types_enc"].split(",").count("0") == 7 and s["checkpoint"] == ",".join(["1"] * 48)
    assert (s["global_bsz"], s["chunks"], s["default_dp_type"], s["pipeline_type"], s["vtp"]) == (1024, 1, "zero2", "pipedream_flush", 1)


def test_meta_configs_match_the_reference_specs():
    from hetu_galvatron_b200.t5 import config_from_meta
    want = {"t5-small": (512, 64, 2048, 8, 6), "t5-base": (768, 64, 3072, 12, 12), "t5-large": (1024, 64, 4096, 16, 24),
            "t5-3B": (1024, 128, 16384, 32, 24)}
    for name, (h, dkv, ff, heads, layers) in want.items():
        c = config_from_meta(name)
        assert (c.hidden_size, c.d_kv, c.ffn_hidden_size, c.num_attention_heads, c.num_layers, c.num_decoder_layers) == (h, dkv, ff, heads,
                                                                                                                        layers, layers)
        assert (c.vocab_size, c.n_positions, c.n_decoder_positions, c.layer_norm_epsilon, c.dropout_rate) == (32128, 512, 512, 1e-6, 0.0)


def test_model_info_rows_of_t5_3b():
    """48 layer rows in 53 (embed_1, 24 t5_enc, pre_norm_1, embed_2, 24 t5_dec, pre_norm_2, cls); the encoder rows carry one boundary
    tensor, the decoder rows two, and the rows after the last layer none."""
    from hetu_galvatron_b200.core.runtime.hybrid_parallel_config import layer_shapes_dtypes_whole_model
    from hetu_galvatron_b200.t5 import T5ModelInfo, config_from_meta, row_index
    import smoke_model as sm
    config = config_from_meta("t5-3B")
    info = T5ModelInfo(config, sm.tiny_args())
    types_ = info.module_types()
    rows = row_index(config)
    assert len(types_) == 53 and types_.count("t5_enc") == 24 and types_.count("t5_dec") == 24
    assert [types_[rows[k]] for k in ("embed_1", "enc", "pre_norm_1", "embed_2", "dec", "pre_norm_2", "cls")] == \
        ["embed_1", "t5_enc", "pre_norm_1", "embed_2", "t5_dec", "pre_norm_2", "cls"]
    shapes, dtypes = layer_shapes_dtypes_whole_model(types_, info.layernums(), info.shapes(), info.dtypes())
    assert shapes[0] is None and shapes[1] == [[512, -1, 1024]] and shapes[24] == [[512, -1, 1024]]
    assert shapes[rows["dec"]] == [[512, -1, 1024], [512, -1, 1024]] and shapes[-1] is None and shapes[-2] is None
    assert dtypes[rows["dec"]] == [torch.bfloat16, torch.bfloat16]


@pytest.mark.parametrize("option", ["use_ulysses", "global_cp_deg", "load", "save", "tied_embeddings", "dropout", "json_use_sp",
                                    "json_vsp"])
def test_refused_options_raise(option):
    from hetu_galvatron_b200.core.runtime import world as _world
    from hetu_galvatron_b200.t5 import config_from_meta, set_model_config, t5_model_hp
    import smoke_model as sm
    from _t5_worker import TINY
    over = {"use_ulysses": dict(use_ulysses=True), "global_cp_deg": dict(global_cp_deg=2), "load": dict(load="/nonexistent"),
            "save": dict(save="/nonexistent"), "tied_embeddings": dict(untie_embeddings_and_output_weights=False),
            "json_use_sp": dict(galvatron_config_path=dict(row_strategy([1] * 4, [4], 1, 4), use_sp="1,1,1,1")),
            "json_vsp": dict(galvatron_config_path=dict(row_strategy([1] * 4, [4], 1, 4), vsp=1))}.get(option, {})
    spec = dict(TINY, dropout_rate=0.1) if option == "dropout" else dict(TINY)
    args = sm.tiny_args(**over)
    config = set_model_config(config_from_meta(spec), args)
    with _world.simulated(0, 1):
        with pytest.raises(NotImplementedError, match="T5 family does not support"):
            t5_model_hp(config, args)


def test_cross_attention_refusals():
    """cross-attention refuses Ulysses, context parallelism and GQA"""
    import types
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    from hetu_galvatron_b200.core.runtime.tensor_parallel import AttnType, ParallelAttention
    conf = types.SimpleNamespace(hidden_size=64, num_attention_heads=4, num_query_groups=4, kv_channels=32, add_bias_linear=True)
    two = CommGroup([0, 1])
    with pytest.raises(NotImplementedError, match="Ulysses"):
        ParallelAttention(conf, 1, attention_type=AttnType.cross_attn, sp_group=two, use_ulysses=True, device="meta")
    with pytest.raises(NotImplementedError, match="context parallelism"):
        ParallelAttention(conf, 1, attention_type=AttnType.cross_attn, use_zigzag_cp=True, device="meta")
    with pytest.raises(NotImplementedError, match="grouped-query"):
        ParallelAttention(types.SimpleNamespace(**dict(vars(conf), num_query_groups=2)), 1, attention_type=AttnType.cross_attn,
                          device="meta")


def test_oracle_matches_hf_t5():
    """oracle/t5_ref.py in fp64 against HF T5ForConditionalGeneration: gelu_new, untied embeddings, relative-attention tables and all
    biases zero, q pre-scaled by 1 / sqrt(d_kv), shared = dec_shared.  HF's T5 takes the norm's variance and the attention softmax in
    fp32 even in an fp64 model, which bounds the agreement at ~1e-7; everything else is fp64."""
    transformers = pytest.importorskip("transformers")
    from oracle import t5_ref
    h, n, hn, f, V = 32, 4, 16, 48, 64
    w = t5_ref.init_weights(h, n * hn, f, V, 2, 2, seed=3, std=0.2, dtype=torch.float64)
    for p in w["enc"] + w["dec"]:
        for k in p:
            if k.endswith("_b"):
                p[k].zero_()
    w["dec_shared"] = w["shared"]
    g = torch.Generator().manual_seed(5)
    enc, dec = torch.randint(0, V, (2, 12), generator=g), torch.randint(0, V, (2, 8), generator=g)
    labels = torch.randint(0, V, (2, 8), generator=g)
    loss, _ = t5_ref.forward_loss(w, enc, dec, labels, dict(heads=n, eps=1e-6), dtype=torch.float64)
    cfg = transformers.T5Config(vocab_size=V, d_model=h, d_kv=hn, d_ff=f, num_layers=2, num_decoder_layers=2, num_heads=n,
                                dropout_rate=0.0, layer_norm_epsilon=1e-6, feed_forward_proj="gelu_new", tie_word_embeddings=False)
    cfg.tie_word_embeddings = False             # (transformers 5 drops the keyword for T5)
    model = transformers.T5ForConditionalGeneration(cfg).double().eval()
    assert model.lm_head.weight is not model.shared.weight
    missing, unexpected = model.load_state_dict(t5_ref.to_hf_state_dict(w, n), strict=False)
    assert not unexpected and all("relative_attention_bias" in k for k in missing)

    with torch.no_grad():
        for name, p in model.named_parameters():
            if "relative_attention_bias" in name:
                p.zero_()
        logits = model(input_ids=enc, decoder_input_ids=dec).logits
    want = torch.nn.functional.cross_entropy(logits.reshape(-1, V), labels.reshape(-1), reduction="none").view(2, 8)
    torch.testing.assert_close(loss, want, rtol=1e-6, atol=1e-6)


def test_label_minus_one_is_scored_as_megatron_does():
    """a -1 label scores logsumexp - max (Megatron's target logit 0 after the row maximum is taken off), not 0"""
    from oracle import t5_ref
    logits = torch.tensor([[[1.0, 3.0, 2.0]]], dtype=torch.float64)
    got = t5_ref.token_loss(logits, torch.tensor([[-1]]))
    assert torch.allclose(got, torch.logsumexp(logits, -1) - 3.0)

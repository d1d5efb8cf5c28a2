"""The ViT family (galvatron/models/vit_hf) on the product's core: N ranks over gloo run the family's layers / schedules on the oracle
backend and must reproduce the single-process oracle (oracle/vit_ref.py, pinned to HF ViT here) on the global batch -- loss 5e-3 rel,
per-parameter gradients 3e-2 rel-L2, and the loss after one AdamW step.  Tiny model: image 32, patch 8 (17 tokens), 20 classes."""
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
_PORT = [29700]

HUGE_JSON = "tests/golden/vit_huge_tp2_4gpus.json"


def launch(world, config, timeout=900, backend="oracle"):
    from _launch import launch_ranks
    _PORT[0] += 1
    return launch_ranks("_vit_worker", world, config, _PORT[0] + os.getpid() % 500, timeout=timeout, backend=backend)


def reference_format_strategy(layers, pp, tp, chunks, gbs, pipeline_type="pipedream_flush", checkpoint=0, vtp=None):
    """A strategy in the format the reference's Search Engine writes (its configs/galvatron_config_*.json)."""
    row = lambda v: ",".join([str(v)] * layers)  # noqa: E731
    return {"pp_deg": pp, "tp_sizes_enc": row(tp), "tp_consecutive_flags": row(1), "dp_types_enc": row(0), "use_sp": row(0),
            "checkpoint": row(checkpoint), "global_bsz": gbs, "chunks": chunks,
            "pp_division": ",".join([str(layers // pp)] * pp), "pipeline_type": pipeline_type, "default_dp_type": "zero2",
            "vtp": tp if vtp is None else vtp, "vsp": 0}


# name -> (world, worker config, the token count the layers must run)
CASES = {
    # 17 tokens x micro-batch 8 = 136 rows: no padding
    "world1": (1, dict(global_train_batch_size=8), 17),
    "world1_ckpt_chunks2": (1, dict(global_checkpoint=1, chunks=2, global_train_batch_size=8), 24),
    "tp2_vtp2": (2, dict(global_tp_deg=2, vocab_tp=2), 24),
    "dp2_zero3_embed_sdp": (2, dict(sdp=1, embed_sdp=1, global_train_batch_size=16), 17),
    "pp2_1f1b": (2, dict(pp_deg=2, chunks=2, pipeline_type="pipedream_flush", global_train_batch_size=16), 17),
    "pp2_tp2_gpipe": (4, dict(pp_deg=2, global_tp_deg=2, vocab_tp=2, chunks=2, pipeline_type="gpipe"), 24),
    # the embedding row at vtp 1 (data-parallel over both ranks), the layers TP2: the activations are relocated between them
    "relocation_embed_vtp1_layers_tp2": (2, dict(global_tp_deg=2, vocab_tp=1), 24),
    # micro-batch 1: 17 tokens -> 24 (7 padding tokens masked out as keys)
    "padded_tokens_microbatch1": (1, dict(chunks=2, global_train_batch_size=2, _check_padded_token_grad=True), 24),
    "hidden_dropout": (2, dict(global_tp_deg=2, vocab_tp=2, _spec=dict(hidden_dropout_prob=0.1)), 24),
    # the reference's ViT-huge strategy (TP2 on all 32 layers, vtp 2, ZeRO-2, 1F1B) on a 32-layer tiny model, global batch 160 -> 16
    "reference_vit_huge_tp2_4gpus_json": (4, dict(_strategy=HUGE_JSON, _strategy_over=dict(global_bsz=16),
                                                  _spec=dict(num_hidden_layers=32)), 17),
    # a Search Engine JSON whose micro-batch is 1 (as the reference's ViT-xhuge one: PP2 x TP2, chunks = global batch)
    "reference_format_json_pp2_tp2_microbatch1": (4, dict(_strategy=reference_format_strategy(2, 2, 2, 4, 4, checkpoint=1)), 24),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_vit_family(name):
    world, cfg, s_run = CASES[name]
    rep = launch(world, dict(cfg))
    assert rep["s_run"] == s_run and rep["seq"] == 17
    assert rep["max_grad_err"] < 3e-2
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])
    assert rep["classifier_pad_rows_max"] == 0.0
    if cfg.get("_check_padded_token_grad"):
        assert rep["pad_token_grad_max"] == 0.0 and rep["real_token_grad_max"] > 0.0


def test_golden_strategy_is_the_reference_search_engine_output():
    with open(os.path.join(ROOT, HUGE_JSON)) as f:
        s = json.load(f)
    assert s["tp_sizes_enc"] == ",".join(["2"] * 32) and s["vtp"] == 2 and s["vsp"] == 0 and s["pp_deg"] == 1
    assert (s["global_bsz"], s["chunks"], s["default_dp_type"], s["pipeline_type"]) == (160, 1, "zero2", "pipedream_flush")


def test_token_rows_rule():
    """seq_run = S unless some row's micro-batch makes S x m a multiple of 8 fail; then S rounded up to 8 (197 -> 200)."""
    from hetu_galvatron_b200.core.runtime import world as _world
    from hetu_galvatron_b200.vit_hf import config_from_meta, token_rows
    import smoke_model as sm
    config = config_from_meta("vit-huge-patch16-224")
    assert config.seq_length == 197
    hp = lambda tp, pp=1, vtp=1: {"pp_deg": pp, "tp_sizes_enc": [tp] * 32, "vocab_tp": vtp}  # noqa: E731
    assert _world.get_world_size() == 1
    assert token_rows(config, sm.tiny_args(global_train_batch_size=8, chunks=1), hp(1)) == 197
    assert token_rows(config, sm.tiny_args(global_train_batch_size=16, chunks=2), hp(1)) == 197
    assert token_rows(config, sm.tiny_args(global_train_batch_size=64, chunks=64), hp(1)) == 200     # the xhuge JSON: micro-batch 1
    assert token_rows(config, sm.tiny_args(global_train_batch_size=12, chunks=1), hp(1)) == 200
    assert token_rows(config, sm.tiny_args(global_train_batch_size=20, chunks=2), hp(1)) == 200     # 10 per micro-batch


def test_meta_configs_match_the_reference_specs():
    from hetu_galvatron_b200.vit_hf import config_from_meta
    for name, (h, layers, heads, ffn) in {"vit-base-patch16-224": (768, 12, 12, 3072), "vit-large-patch16-224": (1024, 24, 16, 4096),
                                          "vit-huge-patch16-224": (1280, 32, 16, 5120),
                                          "vit-xhuge-patch16-224": (2560, 128, 32, 10240)}.items():
        c = config_from_meta(name)
        assert (c.hidden_size, c.num_hidden_layers, c.num_attention_heads, c.intermediate_size) == (h, layers, heads, ffn)
        assert (c.image_size, c.patch_size, c.num_channels, c.num_labels, c.layer_norm_eps) == (224, 16, 3, 1000, 1e-12)
        assert (c.hidden_dropout_prob, c.attention_probs_dropout_prob, c.seq_length) == (0.0, 0.0, 197)


@pytest.mark.parametrize("option", ["sequence_parallel", "use_ulysses", "global_cp_deg", "load", "save", "json_use_sp"])
def test_refused_options_raise(option):
    from hetu_galvatron_b200.vit_hf import config_from_meta, set_model_config, vit_model_hp
    import smoke_model as sm
    over = {"sequence_parallel": dict(sequence_parallel=True), "use_ulysses": dict(use_ulysses=True), "global_cp_deg": dict(global_cp_deg=2),
            "load": dict(load="/nonexistent"), "save": dict(save="/nonexistent"),
            "json_use_sp": dict(galvatron_config_path=dict(reference_format_strategy(2, 1, 1, 1, 8), use_sp="1,1"))}[option]
    args = sm.tiny_args(**over)
    from _vit_worker import TINY
    config = set_model_config(config_from_meta(TINY), args)
    with pytest.raises(NotImplementedError, match="ViT family does not support"):
        vit_model_hp(config, args)


def test_model_info_goes_through_gen_comm_groups():
    """The ViT rows (embed, vit_enc x L, prenorm, cls) through the whole-model strategy and the group builder, as the other families."""
    from hetu_galvatron_b200.core.runtime.hybrid_parallel_config import hp_config_whole_model
    from hetu_galvatron_b200.core.runtime import world as _world
    from hetu_galvatron_b200.core.runtime.comm_groups import gen_comm_groups
    from hetu_galvatron_b200.vit_hf import ViTModelInfo, config_from_meta
    import smoke_model as sm
    args = sm.tiny_args()
    config = config_from_meta("vit-huge-patch16-224")
    info = ViTModelInfo(config, args)
    types_ = info.module_types()
    assert types_[0] == "embed" and types_[-2:] == ["prenorm", "cls"] and types_[1:-2] == ["vit_enc"] * 32
    assert info.shapes() == [[[197, -1, 1280]]]
    hp = {"pp_deg": 2, "tp_sizes_enc": [2] * 32, "tp_consecutive_flags": [1] * 32, "cp_sizes_enc": [1] * 32, "dp_types_enc": [0] * 32,
          "checkpoint_flags_enc": [0] * 32, "pp_ranks_enc": [0] * 16 + [1] * 16, "use_sp": [0] * 32}
    with _world.simulated(0, 4):
        whole = hp_config_whole_model(types_, hp, vocab_tp=2)
        groups = gen_comm_groups(whole["tp_sizes_whole"], whole["sp_sizes_whole"], whole["cp_sizes_whole"], whole["pp_deg"],
                                 whole["tp_consec_whole"])
    assert len(whole["tp_sizes_whole"]) == 35 and whole["pp_ranks_whole"][:2] == [0, 0] and whole["pp_ranks_whole"][-1] == 1
    assert whole["dp_sizes_whole"] == [1] * 35
    pp_group, tp_groups = groups[0], groups[1]
    assert list(pp_group.ranks) == [0, 2] and all(g is None or list(g.ranks) == [0, 1] for g in tp_groups)
    assert any(g is not None for g in tp_groups)


def test_oracle_matches_hf_vit():
    """oracle/vit_ref.py in fp64 against HF ViTModel(add_pooling_layer=True, gelu_pytorch_tanh) + a bias-free linear."""
    transformers = pytest.importorskip("transformers")
    from oracle import vit_ref
    cfg = dict(hidden=64, ffn=128, n_heads=4, head_dim=16, n_layers=2, patch=8, channels=3, seq=17, num_labels=20, eps=1e-12,
               gelu_tanh=True)
    w = vit_ref.init_weights(cfg, seed=3, std=0.2, dtype=torch.float64)
    g = torch.Generator().manual_seed(5)
    for lw in w["layers"]:                       # non-trivial norms and biases
        for k in ("ln1", "ln2"):
            lw[k] = 1 + 0.1 * torch.randn(64, generator=g, dtype=torch.float64)
        for k in ("ln1_b", "ln2_b", "qkv_b", "dense_b", "h_to_4h_b", "4h_to_h_b"):
            lw[k] = 0.1 * torch.randn(lw[k].shape, generator=g, dtype=torch.float64)
    pixels = torch.randn(3, 3, 32, 32, generator=g, dtype=torch.float64)
    labels = torch.randint(0, 20, (3,), generator=g)
    loss, _ = vit_ref.forward_loss(w, pixels, labels, cfg, dtype=torch.float64)
    hf_cfg = transformers.ViTConfig(hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128, image_size=32,
                                    patch_size=8, num_channels=3, hidden_act="gelu_pytorch_tanh", layer_norm_eps=1e-12,
                                    hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    model = transformers.ViTModel(hf_cfg, add_pooling_layer=True).double().eval()
    sd, classifier = vit_ref.to_hf_state_dict(w, cfg)
    model.load_state_dict(sd, strict=True)
    with torch.no_grad():
        pooled = model(pixel_values=pixels).pooler_output
    logits = pooled @ classifier.t()
    want = torch.nn.functional.cross_entropy(logits, labels, reduction="none")
    torch.testing.assert_close(loss, want, rtol=1e-10, atol=1e-10)

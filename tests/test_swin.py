"""The Swin family (galvatron/models/swin) on the product's core: N ranks over gloo run the family's layers / schedules on the CPU
restatement of its kernels and must reproduce the single-process oracle (oracle/swin_ref.py, pinned to HF Swin here) on the global
batch -- loss 5e-3 rel, per-parameter gradients 3e-2 rel-L2, and the loss after one AdamW step.  Tiny model: 224 px, patch 4,
window 7 (stages of 3136, 784, 196 and 49 tokens), embed 16, heads 1 / 2 / 4 / 8, 20 classes."""
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
_PORT = [29950]

HUGE_JSON = "tests/golden/swin_huge_pp8_8gpus.json"
UNPADDED, PADDED = [3136, 784, 196, 49], [3136, 784, 200, 56]
# tensor-parallel cases: heads 2 / 4 / 8 / 16 (head dim 8), so that stage 0 splits over two ranks
TP_HEADS = dict(num_heads=[2, 4, 8, 16])


def launch(world, config, timeout=1800, backend="oracle"):
    from _launch import launch_ranks
    _PORT[0] += 1
    return launch_ranks("_swin_worker", world, config, _PORT[0] + os.getpid() % 500, timeout=timeout, backend=backend)


def row_strategy(tps, pp_division, chunks, gbs, pipeline_type="pipedream_flush", vtp=1, checkpoint=0):
    """A strategy in the reference Search Engine's format with one tp degree per swin_enc layer."""
    n = len(tps)
    j = lambda v: ",".join(str(x) for x in v)  # noqa: E731
    return {"pp_deg": len(pp_division), "tp_sizes_enc": j(tps), "tp_consecutive_flags": j([1] * n), "dp_types_enc": j([0] * n),
            "use_sp": j([0] * n), "checkpoint": j([checkpoint] * n), "global_bsz": gbs, "chunks": chunks, "pp_division": j(pp_division),
            "pipeline_type": pipeline_type, "default_dp_type": "zero2", "vtp": vtp, "vsp": 0}


# name -> (world, worker config, the tokens each stage must run)
CASES = {
    "world1": (1, dict(global_train_batch_size=8, _check_padded_token_grad=True), UNPADDED),
    "world1_ckpt": (1, dict(global_train_batch_size=8, global_checkpoint=1), UNPADDED),
    # micro-batches of 7: 196 x 7 and 49 x 7 are not multiples of 8, so stages 2 and 3 run 200 and 56 tokens
    "world1_padded_microbatch7": (1, dict(global_train_batch_size=7, _check_padded_token_grad=True), PADDED),
    "dp2_zero2": (2, dict(global_train_batch_size=16), UNPADDED),
    "dp2_zero3_ckpt": (2, dict(global_train_batch_size=16, sdp=1, global_checkpoint=1), UNPADDED),
    "tp2_vtp1": (2, dict(global_tp_deg=2, vocab_tp=1, global_train_batch_size=16, _spec=TP_HEADS), UNPADDED),
    "tp2_vtp2": (2, dict(global_tp_deg=2, vocab_tp=2, global_train_batch_size=8, _spec=TP_HEADS), UNPADDED),
    # tp changes at the first downsample row: stage-0 layers tp 1 (dp 2), the downsample (vtp) and stage 1 onwards tp 2
    "mixed_tp_across_width_change": (2, dict(_strategy=row_strategy([1, 1, 2, 2, 2, 2, 2, 2], [8], 1, 16, vtp=2), _spec=TP_HEADS),
                                     UNPADDED),
    # pp 2, 1F1B: stage 0 = embed + stage-0 layers, split just before the first downsample row
    "pp2_1f1b_split_before_downsample": (2, dict(_strategy=row_strategy([1] * 8, [2, 6], 2, 16)), UNPADDED),
    # pp 2, GPipe: split between the two blocks of stage 1 (inside a stage)
    "pp2_gpipe_split_inside_stage": (2, dict(_strategy=row_strategy([1] * 8, [3, 5], 2, 16, pipeline_type="gpipe")), UNPADDED),
    "drop_path_world1": (1, dict(global_train_batch_size=8, _spec=dict(drop_path_rate=0.3)), UNPADDED),
    # the checkpoint recompute draws the forward's masks (the dropout context is captured with the checkpoint)
    "drop_path_world1_ckpt": (1, dict(global_train_batch_size=8, global_checkpoint=1, _spec=dict(drop_path_rate=0.3)), UNPADDED),
    "drop_path_tp2_ckpt": (2, dict(global_tp_deg=2, vocab_tp=2, global_train_batch_size=8, global_checkpoint=1,
                                   _spec=dict(TP_HEADS, drop_path_rate=0.3)), UNPADDED),
    "drop_path_dp2": (2, dict(global_train_batch_size=16, _spec=dict(drop_path_rate=0.3)), UNPADDED),
    "drop_path_tp2": (2, dict(global_tp_deg=2, vocab_tp=2, global_train_batch_size=8, _spec=dict(TP_HEADS, drop_path_rate=0.3)),
                      UNPADDED),
    "drop_path_pp2": (2, dict(_strategy=row_strategy([1] * 8, [3, 5], 2, 16), _spec=dict(drop_path_rate=0.3)), UNPADDED),
    # the reference's swin-huge strategy (pp 8, 41 chunks) on depths [2, 2, 42, 2] at tiny widths, global batch 1024 -> 16 (16 chunks)
    "reference_swin_huge_pp8_json": (8, dict(_strategy=HUGE_JSON, _strategy_over=dict(global_bsz=16, chunks=16),
                                             _spec=dict(depths=[2, 2, 42, 2])), PADDED),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_swin_family(name):
    world, cfg, tokens_run = CASES[name]
    rep = launch(world, dict(cfg))
    assert rep["tokens_run"] == tokens_run and rep["tokens"] == UNPADDED
    assert rep["max_grad_err"] < 3e-2
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])
    assert rep["classifier_pad_rows_max"] == 0.0
    if cfg.get("_check_padded_token_grad"):
        assert rep["real_token_grad_max"] > 0.0


def test_padding_gives_the_loss_of_the_unpadded_run():
    """micro-batches of 8 (no padding) and 7 (stages 2 and 3 padded) over the same 56 samples: the same oracle loss, reproduced."""
    a = launch(1, dict(global_train_batch_size=56, chunks=7))
    b = launch(1, dict(global_train_batch_size=56, chunks=8))
    assert a["tokens_run"] == UNPADDED and b["tokens_run"] == PADDED
    assert a["ref_loss"] == b["ref_loss"]
    assert abs(a["loss"] - b["loss"]) <= 5e-3 * abs(a["ref_loss"])


def test_golden_strategy_is_the_reference_search_engine_output():
    with open(os.path.join(ROOT, HUGE_JSON)) as f:
        s = json.load(f)
    assert s["tp_sizes_enc"] == ",".join(["1"] * 48) and s["pp_division"] == "3,7,7,7,7,7,7,3" and s["pp_deg"] == 8
    assert (s["global_bsz"], s["chunks"], s["default_dp_type"], s["pipeline_type"], s["vtp"]) == (1024, 41, "zero2", "pipedream_flush", 1)


def test_token_rows_rule():
    """T_k unless some row's micro-batch m makes T_k x m a multiple of 8 fail; then ceil8(T_k): Swin-H 196 -> 200, 49 -> 56."""
    from hetu_galvatron_b200.core.runtime import world as _world
    from hetu_galvatron_b200.swin import config_from_meta, token_rows
    import smoke_model as sm
    config = config_from_meta("swin-huge-patch4-window7-224")
    hp = lambda tp=1, vtp=1: {"pp_deg": 1, "tp_sizes_enc": [tp] * 48, "vocab_tp": vtp}  # noqa: E731
    assert _world.get_world_size() == 1
    assert token_rows(config, sm.tiny_args(global_train_batch_size=64, chunks=1), hp()) == UNPADDED
    assert token_rows(config, sm.tiny_args(global_train_batch_size=63, chunks=1), hp()) == PADDED
    assert token_rows(config, sm.tiny_args(global_train_batch_size=1024, chunks=41), hp()) == PADDED      # micro-batches 25 and 24
    assert token_rows(config, sm.tiny_args(global_train_batch_size=16, chunks=2), hp()) == UNPADDED
    large = config_from_meta("swin-large-patch4-window12-384")
    assert token_rows(large, sm.tiny_args(global_train_batch_size=7, chunks=1), hp()) == [9216, 2304, 576, 144]


def test_meta_configs_match_the_reference_specs():
    from hetu_galvatron_b200.swin import config_from_meta
    h = config_from_meta("swin-huge-patch4-window7-224")
    assert (h.embed_dim, h.depths, h.num_heads, h.window_size, h.image_size) == (320, [2, 2, 42, 2], [8, 16, 32, 64], 7, 224)
    assert [s["tokens"] for s in h.stages] == UNPADDED and [s["width"] for s in h.stages] == [320, 640, 1280, 2560]
    assert [(s["window"], s["shift"]) for s in h.stages] == [(7, 3), (7, 3), (7, 3), (7, 0)]
    large = config_from_meta("swin-large-patch4-window12-384")
    assert (large.embed_dim, large.depths, large.num_heads, large.window_size, large.image_size) == (192, [2, 2, 18, 2], [6, 12, 24, 48],
                                                                                                     12, 384)
    assert [(s["window"], s["shift"]) for s in large.stages] == [(12, 6), (12, 6), (12, 6), (12, 0)]
    for c in (h, large):
        assert (c.patch_size, c.num_channels, c.num_labels, c.layer_norm_eps, c.mlp_ratio, c.drop_path_rate) == (4, 3, 1000, 1e-5, 4, 0.1)
    # about 1.0 B parameters in Swin-H: 12 C^2 per block, 8 C^2 per merge (biases and norms aside)
    n = sum(12 * s["width"] ** 2 * s["depth"] for s in h.stages) + sum(8 * s["width"] ** 2 for s in h.stages[:-1])
    assert 0.95e9 < n < 1.05e9


@pytest.mark.parametrize("res,window,shift", [(56, 7, 3), (28, 7, 3), (14, 7, 3), (7, 7, 0), (16, 4, 2), (24, 12, 6)])
def test_token_map_is_hf_roll_and_window_partition(res, window, shift):
    """The token map equals HF's roll(-s, -s) + window_partition as an index permutation, exactly; the mask is HF's."""
    from oracle import swin_ref
    from hetu_galvatron_b200.swin import shift_mask, token_map
    grid = torch.arange(res * res, dtype=torch.float64).view(1, res, res, 1)
    rolled = torch.roll(grid, shifts=(-shift, -shift), dims=(1, 2)) if shift else grid
    want = swin_ref.window_partition(rolled, window).reshape(-1).long()
    assert torch.equal(token_map(res, window, shift), want)
    assert sorted(want.tolist()) == list(range(res * res))
    if shift:
        assert torch.equal(shift_mask(res, window, shift), swin_ref.hf_shift_mask(res, window, shift))
    else:
        assert shift_mask(res, window, shift) is None


def test_shift_mask_matches_hf_get_attn_mask():
    transformers = pytest.importorskip("transformers")
    from transformers.models.swin.modeling_swin import SwinLayer
    from hetu_galvatron_b200.swin import shift_mask
    cfg = transformers.SwinConfig(embed_dim=16, window_size=7)
    layer = SwinLayer(cfg, dim=16, input_resolution=(28, 28), num_heads=1, shift_size=3)
    hf = layer.get_attn_mask(28, 28, dtype=torch.float32, device=torch.device("cpu"))
    assert torch.equal(shift_mask(28, 7, 3), hf != 0)


@pytest.mark.parametrize("option", ["sequence_parallel", "use_ulysses", "global_cp_deg", "load", "save", "hidden_dropout",
                                    "attention_dropout", "absolute_embeddings", "window_not_dividing", "json_use_sp",
                                    "drop_path_layers_tp2_vocab_tp1", "drop_path_layers_tp1_vocab_tp2",
                                    "drop_path_layers_tp2_not_consecutive"])
def test_refused_options_raise(option):
    from hetu_galvatron_b200.swin import config_from_meta, set_model_config, swin_model_hp
    import smoke_model as sm
    from _swin_worker import TINY
    spec = dict(TINY)
    over = {"sequence_parallel": dict(sequence_parallel=True), "use_ulysses": dict(use_ulysses=True), "global_cp_deg": dict(global_cp_deg=2),
            "load": dict(load="/nonexistent"), "save": dict(save="/nonexistent"),
            "json_use_sp": dict(galvatron_config_path=dict(row_strategy([1] * 8, [8], 1, 8), use_sp="1,1,1,1,1,1,1,1")),
            # drop path with blocks that hold another slice of the batch than the embedding / head rows (relocation)
            "drop_path_layers_tp2_vocab_tp1": dict(galvatron_config_path=row_strategy([2] * 8, [8], 1, 8, vtp=1)),
            "drop_path_layers_tp1_vocab_tp2": dict(galvatron_config_path=row_strategy([1, 1, 2, 2, 2, 2, 2, 2], [8], 1, 8, vtp=2)),
            "drop_path_layers_tp2_not_consecutive": dict(galvatron_config_path=dict(row_strategy([2] * 8, [8], 1, 8, vtp=2),
                                                                                    tp_consecutive_flags="0,0,0,0,0,0,0,0"))}.get(option, {})
    spec.update({"hidden_dropout": dict(hidden_dropout_prob=0.1), "attention_dropout": dict(attention_probs_dropout_prob=0.1),
                 "absolute_embeddings": dict(use_absolute_embeddings=True),
                 "window_not_dividing": dict(window_size=6)}.get(option, {}))
    if option.startswith("drop_path"):
        spec.update(num_heads=[2, 4, 8, 16], drop_path_rate=0.1)
    args = sm.tiny_args(**over)
    config = set_model_config(config_from_meta(spec), args)
    from hetu_galvatron_b200.core.runtime import world as _world
    with _world.simulated(0, 4 if option.startswith("drop_path") else 1):     # (the refusal comes before any group exists)
        with pytest.raises(NotImplementedError, match="Swin family does not support.*%s" % ("drop path" if option.startswith("drop_path")
                                                                                            else "")):
            swin_model_hp(config, args)


def test_model_info_rows_of_swin_huge():
    """54 rows for swin-huge (embed, 48 blocks, 3 downsample rows, pooler, cls); the downsample rows take the vocabulary degree and
    the next stage's boundary shape, and the reference's 48-entry JSON fills the 48 swin_enc rows."""
    from hetu_galvatron_b200.core.runtime.hybrid_parallel_config import layer_shapes_dtypes_whole_model
    from hetu_galvatron_b200.swin import SwinModelInfo, config_from_meta
    import smoke_model as sm
    info = SwinModelInfo(config_from_meta("swin-huge-patch4-window7-224"), sm.tiny_args())
    types_ = info.module_types()
    assert len(types_) == 54 and types_.count("swin_enc") == 48 and types_.count("swin_downsample") == 3
    assert types_[0] == "embed" and types_[-2:] == ["pooler", "cls"] and types_[3] == "swin_downsample"
    shapes, _ = layer_shapes_dtypes_whole_model(types_, info.layernums(), info.shapes(), info.dtypes())
    assert shapes[0] is None and shapes[1] == [[3136, -1, 320]] and shapes[3] == [[784, -1, 640]] and shapes[-1] is None


def test_oracle_matches_hf_swin():
    """oracle/swin_ref.py in fp64 against HF SwinForImageClassification with zeroed relative-position tables and classifier bias."""
    transformers = pytest.importorskip("transformers")
    from oracle import swin_ref
    cfg = dict(embed_dim=16, depths=[2, 2, 2, 2], heads=[1, 2, 4, 8], window=2, patch=4, image=64, eps=1e-5)
    w = swin_ref.init_weights(cfg, 10, seed=3, std=0.2, dtype=torch.float64)
    g = torch.Generator().manual_seed(5)
    for st in w["stages"]:
        for bw in st["blocks"]:
            for k in ("ln1", "ln2"):
                bw[k] = 1 + 0.1 * torch.randn(bw[k].shape, generator=g, dtype=torch.float64)
            for k in ("ln1_b", "ln2_b"):
                bw[k] = 0.1 * torch.randn(bw[k].shape, generator=g, dtype=torch.float64)
    pixels = torch.randn(2, 3, 64, 64, generator=g, dtype=torch.float64)
    labels = torch.randint(0, 10, (2,), generator=g)
    loss, _ = swin_ref.forward_loss(w, pixels, labels, cfg, dtype=torch.float64)
    hc = transformers.SwinConfig(image_size=64, patch_size=4, num_channels=3, embed_dim=16, depths=[2, 2, 2, 2], num_heads=[1, 2, 4, 8],
                                 window_size=2, mlp_ratio=4.0, qkv_bias=True, hidden_act="gelu_pytorch_tanh", drop_path_rate=0.0,
                                 hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-5,
                                 use_absolute_embeddings=False, num_labels=10)
    model = transformers.SwinForImageClassification(hc).double().eval()
    missing, unexpected = model.load_state_dict(swin_ref.to_hf_state_dict(w, cfg), strict=False)
    assert not unexpected and all("relative_position" in k for k in missing)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "relative_position_bias_table" in n:
                p.zero_()
        logits = model(pixel_values=pixels).logits
    want = torch.nn.functional.cross_entropy(logits, labels, reduction="none")
    torch.testing.assert_close(loss, want, rtol=1e-10, atol=1e-10)

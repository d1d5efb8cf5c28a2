"""The Swin family with HF's learned relative-position bias (spec key ``relative_position_bias``) on the product's core: N ranks over
gloo run it on the CPU restatement of its kernels (tests/_swin_rpb.py) and must reproduce the oracle with per-block tables on the
global batch -- loss 5e-3 rel, every gradient (the tables included) 3e-2 rel-L2, and the loss after one AdamW step -- as
tests/test_swin.py checks the plain model.  The oracle itself is pinned in fp64 to HF ``SwinForImageClassification`` with non-zero
tables."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_swin import HUGE_JSON, PADDED, TP_HEADS, UNPADDED, row_strategy  # noqa: E402

_PORT = [30450]


def launch(world, config, timeout=1800):
    from _launch import launch_ranks
    _PORT[0] += 1
    return launch_ranks("_swin_rpb_worker", world, config, _PORT[0] + os.getpid() % 500, timeout=timeout)


# name -> (world, worker config, the tokens each stage must run)
CASES = {
    "world1": (1, dict(global_train_batch_size=8), UNPADDED),
    "world1_ckpt": (1, dict(global_train_batch_size=8, global_checkpoint=1), UNPADDED),
    "world1_padded_microbatch7": (1, dict(global_train_batch_size=7), PADDED),
    "dp2_zero3": (2, dict(global_train_batch_size=16, sdp=1), UNPADDED),
    "tp2_vtp2": (2, dict(global_tp_deg=2, vocab_tp=2, global_train_batch_size=8, _spec=TP_HEADS), UNPADDED),
    # stage-0 layers tp 1 (dp 2), the downsample (vtp) and stage 1 onwards tp 2
    "mixed_tp_across_width_change": (2, dict(_strategy=row_strategy([1, 1, 2, 2, 2, 2, 2, 2], [8], 1, 16, vtp=2), _spec=TP_HEADS),
                                     UNPADDED),
    "pp2_1f1b_split_before_downsample": (2, dict(_strategy=row_strategy([1] * 8, [2, 6], 2, 16)), UNPADDED),
    "reference_swin_huge_pp8_json": (8, dict(_strategy=HUGE_JSON, _strategy_over=dict(global_bsz=16, chunks=16),
                                             _spec=dict(depths=[2, 2, 42, 2])), PADDED),
}
_REPORTS = {}


@pytest.mark.parametrize("name", sorted(CASES))
def test_swin_rel_bias_family(name):
    world, cfg, tokens_run = CASES[name]
    rep = launch(world, dict(cfg))
    _REPORTS[name] = rep
    assert rep["tokens_run"] == tokens_run
    assert rep["max_grad_err"] < 3e-2 and rep["table_grad_err"] < 3e-2 and rep["table_grad_max"] > 0.0
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])


def test_tables_are_one_draw_under_every_tensor_parallel_layout():
    """the same spec at tp 2 everywhere and at tp 1 in stage 0 / tp 2 after: every block starts from the same whole table"""
    a = _REPORTS.get("tp2_vtp2") or launch(*CASES["tp2_vtp2"][:2])
    b = _REPORTS.get("mixed_tp_across_width_change") or launch(*CASES["mixed_tp_across_width_change"][:2])
    assert a["table_sums"] == b["table_sums"] and len(set(a["table_sums"])) == len(a["table_sums"])


def test_shipped_specs_have_no_table():
    from hetu_galvatron_b200.swin import config_from_meta
    from _swin_worker import TINY
    assert not config_from_meta("swin-huge").relative_position_bias and not config_from_meta("swin-large").relative_position_bias
    assert not config_from_meta(dict(TINY)).relative_position_bias
    assert config_from_meta(dict(TINY, relative_position_bias=True)).relative_position_bias


@pytest.mark.parametrize("window", [1, 2, 7, 12])
def test_index_maps_are_hf_relative_position_index(window):
    """WindowLayout's index is HF's relative_position_index; cells / offsets list every cell of each entry once, ascending"""
    from _swin_rpb import relative_position_index
    from hetu_galvatron_b200.swin.SwinModel_tensor_parallel import WindowLayout
    index, mask, cells, offsets = WindowLayout(2 * window, window, window // 2).rel_maps("cpu")
    assert torch.equal(index.long(), relative_position_index(window).reshape(-1))
    assert offsets[0] == 0 and offsets[-1] == window ** 4 and offsets.numel() == (2 * window - 1) ** 2 + 1
    for t in range(offsets.numel() - 1):
        cs = cells[offsets[t]:offsets[t + 1]].long()
        assert torch.equal(cs, torch.nonzero(index == t).reshape(-1))
    if window // 2:
        from hetu_galvatron_b200.swin import shift_mask
        assert torch.equal(mask.bool(), shift_mask(2 * window, window, window // 2))
    transformers = pytest.importorskip("transformers")
    from transformers.models.swin.modeling_swin import SwinSelfAttention
    hf = SwinSelfAttention(transformers.SwinConfig(), dim=8, num_heads=1, window_size=window)
    assert torch.equal(index.long(), hf.create_relative_position_index().reshape(-1))


def test_restated_kernels_are_the_oracle_bias_and_its_gradient():
    """the CPU restatement of bg_swin_rel_bias_fwd / _bwd against autograd through table[index] + the shift mask"""
    from _swin_rpb import SwinRelBiasOracleBackend
    from hetu_galvatron_b200.swin.SwinModel_tensor_parallel import WindowLayout
    be = SwinRelBiasOracleBackend.__new__(SwinRelBiasOracleBackend)
    lay = WindowLayout(14, 7, 3)
    index, mask, cells, offsets = lay.rel_maps("cpu")
    g = torch.Generator().manual_seed(3)
    table = (torch.randn(169, 4, generator=g) * 0.1).to(torch.bfloat16).double().requires_grad_(True)
    mb = 3
    bias = be.swin_rel_bias_fwd(table.detach().float(), index, mask, mb, lay.n_windows, 7)
    want = table[index.long()].t().reshape(1, 4, 49, 49).repeat(lay.n_windows, 1, 1, 1)
    want = want.masked_fill(mask.bool()[:, None], float("-inf")).repeat(mb, 1, 1, 1)
    assert torch.equal(bias.double(), want.detach())
    dbias = torch.randn(bias.shape, generator=g).to(torch.bfloat16).masked_fill(torch.isinf(bias), 0)
    want.backward(dbias.double())
    got = be.swin_rel_bias_bwd(dbias, cells, offsets, lay.n_windows, 7)
    torch.testing.assert_close(got.double(), table.grad, rtol=1e-5, atol=1e-5)


def test_oracle_with_tables_matches_hf_swin():
    """tests/_swin_rpb.py in fp64 against HF SwinForImageClassification with the same non-zero tables, window 4 on a 128 px image
    (grids 32 / 16 / 8 / 4, every one at least the window; stages 0-2 shifted)"""
    transformers = pytest.importorskip("transformers")
    import _swin_rpb as rpb
    from oracle import swin_ref
    cfg = dict(embed_dim=16, depths=[2, 2, 2, 2], heads=[1, 2, 4, 8], window=4, patch=4, image=128, eps=1e-5)
    w = rpb.add_tables(swin_ref.init_weights(cfg, 10, seed=3, std=0.2, dtype=torch.float64), cfg, seed=4, std=1.0)
    pixels = torch.randn(2, 3, 128, 128, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    labels = torch.tensor([3, 7])
    loss, _ = rpb.forward_loss(w, pixels, labels, cfg, dtype=torch.float64)
    hc = transformers.SwinConfig(image_size=128, patch_size=4, num_channels=3, embed_dim=16, depths=[2, 2, 2, 2], num_heads=[1, 2, 4, 8],
                                 window_size=4, mlp_ratio=4.0, qkv_bias=True, hidden_act="gelu_pytorch_tanh", drop_path_rate=0.0,
                                 hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, layer_norm_eps=1e-5,
                                 use_absolute_embeddings=False, num_labels=10)
    model = transformers.SwinForImageClassification(hc).double().eval()
    missing, unexpected = model.load_state_dict(rpb.to_hf_state_dict(w, cfg), strict=False)
    assert not unexpected and all("relative_position_index" in k for k in missing)
    with torch.no_grad():
        logits = model(pixel_values=pixels).logits
    want = torch.nn.functional.cross_entropy(logits, labels, reduction="none")
    torch.testing.assert_close(loss, want, rtol=1e-10, atol=1e-10)
    # without the tables the oracle is swin_ref's model, bit for bit
    for st in w["stages"]:
        for bw in st["blocks"]:
            del bw["rpb"]
    assert torch.equal(rpb.forward_loss(w, pixels, labels, cfg, dtype=torch.float64)[0],
                       swin_ref.forward_loss(w, pixels, labels, cfg, dtype=torch.float64)[0])

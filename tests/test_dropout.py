"""Dropout of the GPT / BERT families on the CPU: the Philox definition (numpy restatement and the library's host entry), the mask's
statistics, argument checks, and N ranks on the gloo backend reproducing the single-process oracle with the same masks
(hidden_dropout 0.1: loss 5e-3, gradients 3e-2 rel-L2, the loss after one AdamW step)."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _dropout_ref as dref  # noqa: E402

KAT = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
       ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
       ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
_PORT = [29700]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_restatement_known_answers(ctr, key, want):
    assert tuple(int(w) for w in dref.philox4x32_10(ctr, key)) == want


@pytest.fixture(scope="module")
def bg():
    import __graft_entry__ as ge
    from hetu_galvatron_b200 import _bg
    if not os.path.exists(_bg.LIB_PATH):
        ge.build()
    return _bg


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_library_philox_known_answers(bg, ctr, key, want):
    u = ctypes.c_uint32
    out = (u * 4)()
    bg.lib().bg_philox4x32_10((u * 4)(*ctr), (u * 2)(*key), out)
    assert tuple(out) == want


def test_library_philox_matches_restatement_on_random_blocks(bg):
    rng = np.random.default_rng(0)
    u = ctypes.c_uint32
    for _ in range(64):
        ctr, key = rng.integers(0, 2 ** 32, 4, dtype=np.uint64), rng.integers(0, 2 ** 32, 2, dtype=np.uint64)
        out = (u * 4)()
        bg.lib().bg_philox4x32_10((u * 4)(*map(int, ctr)), (u * 2)(*map(int, key)), out)
        assert tuple(out) == tuple(int(w) for w in dref.philox4x32_10(ctr, key))


def test_mask_matches_per_element_loop():
    seed, it, site, p = 77, 5, 7, 0.3
    tokens, samples, h = [3, 4, 5], [10, 11], 12
    keep = dref.keep_mask(seed, it, site, tokens, samples, h, p)
    thr = dref.threshold(p)
    for a, t in enumerate(tokens):
        for b, s in enumerate(samples):
            for j in range(h):
                u = int(dref.philox4x32_10((j // 4, t, s, it), (seed, site))[j % 4])
                assert bool(keep[a, b, j]) == (u >= thr)


def test_keep_fraction_has_no_bias():
    """2^24 elements at p = 0.1: the keep fraction within 5 sigma of 0.9, and no bias per j % 4 lane or per row."""
    p, h = 0.1, 1024
    keep = dref.keep_mask(1234, 3, 4, np.arange(2048), np.arange(8), h, p).numpy()       # 2048 * 8 * 1024 = 2^24
    n = keep.size
    sigma = np.sqrt(p * (1 - p) / n)
    assert abs(keep.mean() - (1 - p)) < 5 * sigma
    lanes = keep.reshape(-1, 4).mean(0)
    assert np.all(np.abs(lanes - (1 - p)) < 5 * np.sqrt(p * (1 - p) / (n / 4))), lanes
    rows = keep.reshape(-1, h).mean(1)                      # per (token, sample) row: binomial(h, 0.9) / h
    z = (rows - (1 - p)) / np.sqrt(p * (1 - p) / h)
    assert abs(z.mean()) < 5 / np.sqrt(len(rows)) and 0.8 < z.std() < 1.2
    assert dref.keep_mask(1234, 4, 4, np.arange(4), np.arange(2), h, p).numpy().tolist() != keep[:4, :2].tolist()


def test_restated_dropout_add_and_backward():
    g = torch.Generator().manual_seed(0)
    x, r = torch.randn(6, 2, 16, generator=g).bfloat16(), torch.randn(6, 2, 16, generator=g).bfloat16()
    b = torch.randn(16, generator=g)
    keep = dref.keep_mask(1, 2, 3, np.arange(6), np.arange(2), 16, 0.25)
    y = dref.dropout_add_ref(x, b, r, keep, 0.25)
    want = torch.where(keep, (x.float() + b) * (1 / 0.75), torch.zeros(())) + r.float()
    assert (y.float() - want).abs().max() <= 2e-2 * want.abs().max()
    assert torch.equal(dref.dropout_add_ref(x, b, r, torch.ones_like(keep), 0.0), (x.float() + b + r.float()).bfloat16())
    dy = torch.randn(6, 2, 16, generator=g).bfloat16()
    dx, db = dref.dropout_bwd_ref(dy, keep, 0.25)
    assert torch.equal(dx, torch.where(keep, dy.float() * np.float32(1 / 0.75), torch.zeros(())).bfloat16())
    assert torch.allclose(db, (dy.float() * keep / 0.75).reshape(-1, 16).sum(0), rtol=1e-5, atol=1e-5)   # unrounded fp32 sums


@pytest.mark.parametrize("p", [1.0, 1.5, -0.1, float("nan")])
def test_probability_out_of_range_raises(p):
    from hetu_galvatron_b200.core.runtime.tensor_parallel.random import check_probability
    with pytest.raises(ValueError):
        check_probability(p)


def test_out_of_range_dropout_raises_at_construction():
    import smoke_model as sm
    from hetu_galvatron_b200.gpt_hf import config_from_meta, set_model_config
    from hetu_galvatron_b200.gpt_hf.GPTModel_tensor_parallel import core_transformer_config_from_args
    args = sm.tiny_args()
    set_model_config(config_from_meta(dict(n_layer=1, n_embd=64, n_head=2, vocab_size=128, n_positions=16, resid_pdrop=1.0,
                                           embd_pdrop=1.0)), args)
    with pytest.raises(ValueError):
        core_transformer_config_from_args(args)
    with pytest.raises(AssertionError):      # the reference's GPT rule: one hidden dropout for the embedding and the residuals
        set_model_config(config_from_meta(dict(n_layer=1, n_embd=64, n_head=2, vocab_size=128, n_positions=16, resid_pdrop=0.1,
                                               embd_pdrop=0.2)), args)


def test_family_configs_map_hf_dropouts():
    import smoke_model as sm
    from hetu_galvatron_b200 import bert_hf, gpt_hf
    args = sm.tiny_args()
    gpt_hf.set_model_config(gpt_hf.config_from_meta("gpt-0.3b"), args)
    assert (args.hidden_dropout, args.attention_dropout) == (0.0, 0.0)          # the shipped specs keep 0
    gpt_hf.set_model_config(gpt_hf.config_from_meta(dict(n_layer=1, n_embd=64, n_head=2, vocab_size=128, n_positions=16, resid_pdrop=0.1,
                                                         attn_pdrop=0.2)), args)
    assert (args.hidden_dropout, args.attention_dropout) == (0.1, 0.2)
    bert_hf.set_model_config(bert_hf.config_from_meta(dict(hidden_size=64, num_hidden_layers=1, num_attention_heads=2, vocab_size=128,
                                                           max_position_embeddings=16, hidden_dropout_prob=0.1,
                                                           attention_probs_dropout_prob=0.05)), args)
    assert (args.hidden_dropout, args.attention_dropout) == (0.1, 0.05)
    from hetu_galvatron_b200.core.runtime.arguments import DEFAULTS
    assert DEFAULTS["hidden_dropout"] == 0.0 and DEFAULTS["attention_dropout"] == 0.0


def launch(world, config, backend="oracle", timeout=900):
    from _launch import launch_ranks
    _PORT[0] += 1
    return launch_ranks("_dropout_worker", world, config, _PORT[0] + os.getpid() % 500, timeout=timeout, backend=backend)


GPT_DROP = dict(resid_pdrop=0.1, embd_pdrop=0.1)
BERT_DROP = dict(hidden_dropout_prob=0.1)
CASES = {
    "gpt_world1": (1, dict(_family="gpt", _spec=GPT_DROP)),
    "gpt_world1_ckpt_chunks2": (1, dict(_family="gpt", _spec=GPT_DROP, global_checkpoint=1, chunks=2)),
    "gpt_tp2": (2, dict(_family="gpt", _spec=GPT_DROP, global_tp_deg=2, vocab_tp=2)),
    "gpt_tp2_megatron_sp": (2, dict(_family="gpt", _spec=GPT_DROP, global_tp_deg=2, vocab_tp=2, sequence_parallel=True)),
    "gpt_dp2_zero3": (2, dict(_family="gpt", _spec=GPT_DROP, sdp=1, embed_sdp=1)),
    "gpt_pp2_1f1b": (2, dict(_family="gpt", _spec=GPT_DROP, pp_deg=2, chunks=2, pipeline_type="pipedream_flush")),
    "gpt_baseline3_pp2_tp2_sp_zero2": (4, dict(_family="gpt", _spec=GPT_DROP, pp_deg=2, global_tp_deg=2, vocab_tp=2, sequence_parallel=True,
                                               default_dp_type="zero2", chunks=4, pipeline_type="pipedream_flush", global_train_batch_size=8)),
    "bert_tp2_megatron_sp": (2, dict(_family="bert", _spec=BERT_DROP, global_tp_deg=2, vocab_tp=2, sequence_parallel=True)),
    "bert_ulysses2": (2, dict(_family="bert", _spec=BERT_DROP, global_tp_deg=2, use_ulysses=True, sequence_parallel=True, vocab_tp=2)),
    "bert_baseline4_ulysses2_dp2": (4, dict(_family="bert", _spec=BERT_DROP, global_tp_deg=2, use_ulysses=True, sequence_parallel=True,
                                            vocab_tp=2, default_dp_type="zero2", chunks=2, global_train_batch_size=8)),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_family_parity_with_hidden_dropout(name):
    world, cfg = CASES[name]
    rep = launch(world, dict(cfg))
    assert rep["max_grad_err"] < 3e-2
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])


@pytest.mark.parametrize("shift", ["_oracle_sample_shift", "_oracle_position_shift"])
def test_wrong_coordinates_fail_the_parity_check(shift):
    """The check has teeth: an oracle that draws its masks one sample (or one position) off misses the tolerance."""
    cfg = dict(CASES["gpt_tp2_megatron_sp"][1], **{shift: 1})
    with pytest.raises(AssertionError, match="max_grad_err|loss"):
        launch(2, cfg)


def test_tensor_parallel_replicas_stay_bit_identical():
    """TP2 without SP: both ranks hold the whole hidden state and draw the same masks, so every layer's output is bit-identical."""
    rep = launch(2, dict(CASES["gpt_tp2"][1], _check_replicas=True))
    assert rep["max_grad_err"] < 3e-2


def _attn_loss(seed=1234, **over):
    return launch(1, dict(_mode="loss", _family="gpt", _spec=dict(attn_pdrop=0.1), seed=seed, chunks=2, **over))["loss"]


def test_attention_dropout_is_reproducible_and_replayed_on_recompute():
    base = _attn_loss()
    assert _attn_loss() == base                                           # fixed seed: bit-identical
    assert abs(_attn_loss(global_checkpoint=1) - base) <= 1e-6 * abs(base)  # recompute replays the tracker's and the default stream
    other = _attn_loss(seed=99)
    assert abs(other - base) > 1e-4 * abs(base)                           # a different seed: 100x the recompute tolerance or more
    no_drop = launch(1, dict(_mode="loss", _family="gpt", seed=1234, chunks=2))["loss"]
    assert abs(no_drop - base) > 1e-4 * abs(base)


def test_attention_dropout_streams_differ_between_tensor_parallel_ranks():
    from hetu_galvatron_b200.core.runtime.tensor_parallel.random import RngTracker, model_parallel_seed
    seeds = {model_parallel_seed(1234, layer, tp, sp) for layer in range(4) for tp in range(8) for sp in range(8)}
    assert len(seeds) == 4 * 8 * 8
    t = RngTracker()
    draws = []
    for tp in range(2):
        with t.fork(("attention", 0, tp, 0), model_parallel_seed(1234, 0, tp, 0), torch.device("cpu")):
            draws.append(torch.rand(8))
    assert not torch.equal(draws[0], draws[1])
    before = torch.get_rng_state()
    states = t.get_states()
    with t.fork(("attention", 0, 0, 0), 0, torch.device("cpu")):
        a = torch.rand(4)
    t.set_states(states)
    with t.fork(("attention", 0, 0, 0), 0, torch.device("cpu")):
        assert torch.equal(torch.rand(4), a)                              # replay after restoring the tracker state
    assert torch.equal(torch.get_rng_state(), before)                     # the default stream is untouched

"""Context parallelism in the GPT family on the CPU: zigzag tokens, learned positions at their global token positions, zigzag labels
and dropout masks drawn per run of consecutive tokens.  N ranks over gloo (tests/_gpt_cp_worker.py) reproduce the single-process
oracle (loss 5e-3, every gradient 3e-2 rel-L2, the loss after one AdamW step) under both K/V exchanges, and every rank's GPT layers
see only their share of the sequence (the ring keeps nothing wider than s/c for backward); the per-run dropout layout reassembles the
single-process mask bit for bit for every (cp, Ulysses, Megatron-SP) layout up to 16 ranks; the HF-layered checkpoint loads at cp 2;
attention dropout and bad sequence lengths are refused when the model is built."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

_PORT = [32300]
CP_COMM = ("allgather", "ring")
_CP2 = dict(_family="gpt", global_cp_deg=2, vocab_cp=2)
_DROP = dict(resid_pdrop=0.1, embd_pdrop=0.1)
CASES = {
    "cp2": (2, dict(_CP2)),
    "cp2_tp2_megatron_sp": (4, dict(_CP2, global_tp_deg=2, vocab_tp=2, sequence_parallel=True)),
    "cp2_dp2_zero3_ckpt": (4, dict(_CP2, sdp=1, embed_sdp=1, global_checkpoint=1, chunks=2, global_train_batch_size=8)),
    "cp2_pp2_1f1b": (4, dict(_CP2, pp_deg=2, chunks=2, pipeline_type="pipedream_flush")),
    # embedding / layer 0 / head tensor-parallel 2 with Megatron-SP, layer 1 cp 2: relocated into the zigzag layout and back
    "cp_mixed_tp2_to_cp2": (2, dict(_family="gpt", sequence_parallel=True, _strategy_json={
        "pp_deg": 1, "tp_sizes_enc": "2,1", "tp_consecutive_flags": "1,1", "dp_types_enc": "0,0", "use_sp": "0,0", "cp_sizes_enc": "1,2",
        "checkpoint": "0,0", "global_bsz": 4, "chunks": 1, "default_dp_type": "zero2", "vtp": 2, "vsp": 0, "vcp": 1})),
    "usp_sp2_cp2": (4, dict(_CP2, global_tp_deg=2, vocab_tp=2, use_ulysses=True, sequence_parallel=True)),
    "cp2_tied": (2, dict(_CP2, untie_embeddings_and_output_weights=False)),
    "cp2_hidden_dropout": (2, dict(_CP2, _spec=_DROP)),
    "cp2_tp2_megatron_sp_hidden_dropout": (4, dict(_CP2, _spec=_DROP, global_tp_deg=2, vocab_tp=2, sequence_parallel=True)),
    "usp_sp2_cp2_hidden_dropout": (4, dict(_CP2, _spec=_DROP, global_tp_deg=2, vocab_tp=2, use_ulysses=True, sequence_parallel=True)),
}
PARAMS = [(name, comm) for name in sorted(CASES) for comm in CP_COMM]


def launch(world, config, backend="oracle", timeout=900):
    from _launch import launch_ranks
    _PORT[0] += 1
    return launch_ranks("_gpt_cp_worker", world, config, _PORT[0] + os.getpid() % 500, timeout=timeout, backend=backend)


def _check(rep, world, cfg, comm):
    assert rep["max_grad_err"] < 3e-2
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])
    assert max(rep["layer_cp"]) == 2 and rep["cp_calls"] > 0
    # every rank asserted its own layer rows; here: some layer runs on s/(2 x ...) rows, never the whole sequence
    assert all(max(rows) < rep["seq"] for rows in rep["layer_rows"].values()), rep["layer_rows"]
    if comm == "ring":
        assert rep["ring_pushes"] > 0 and rep["saved_max_dim"] <= rep["seq"] // 2, rep
    else:
        assert rep["ring_pushes"] == 0 and rep["saved_max_dim"] >= rep["seq"], rep      # the gathered K/V spans the sequence


@pytest.mark.parametrize("name,comm", PARAMS, ids=["%s-%s" % p for p in PARAMS])
def test_gpt_cp_matches_oracle(name, comm):
    world, cfg = CASES[name]
    rep = launch(world, dict(cfg, cp_comm=comm))
    _check(rep, world, cfg, comm)


def test_gpt_cp_loads_hf_layered_checkpoint():
    import json
    golden = os.path.join(ROOT, "tests", "golden", "ckpt_gpt_tiny")
    expected = json.load(open(os.path.join(golden, "expected.json")))
    rep = launch(2, dict(_CP2, load=golden, _golden_ckpt=golden))
    assert rep["ckpt_tensors_bit_exact"] == 3 + 2 * 12 + 2
    assert rep["max_grad_err"] < 3e-2
    assert abs(rep["loss"] - expected["hf_loss_fp32"]) <= 5e-3 * expected["hf_loss_fp32"], (rep["loss"], expected["hf_loss_fp32"])
    assert rep["layer_rows"] and all(rows == [rep["seq"] // 2] for rows in rep["layer_rows"].values())


# ---- the layout of the dropout runs -------------------------------------------------------------------------------------------
class _G:
    def __init__(self, size, rank):
        self.size, self.rank = size, rank

    def rank_in_group(self):
        return self.rank


_LAYOUTS = [(c, p, t) for c in (1, 2, 4, 8) for p in (1, 2, 4) for t in (1, 2, 4) if c * p * t <= 16 and not (p > 1 and t > 1)]


@pytest.mark.parametrize("c,p,t", _LAYOUTS, ids=["cp%d_sp%d_tp%d" % x for x in _LAYOUTS])
def test_dropout_runs_reassemble_the_whole_mask(c, p, t):
    """For every rank of a (cp, Ulysses | Megatron-SP) layout, the rows of the per-run masks are the single-process mask's rows at that
    rank's tokens (redistribute.local_positions), at most two runs; together the ranks cover every token once."""
    import _dropout_ref as dref
    from hetu_galvatron_b200.core.runtime.redistribute import local_positions
    from hetu_galvatron_b200.gpt_hf.GPTModel_tensor_parallel import row_runs
    seq, b, h, prob = 16 * c * p * t, 2, 8, 0.3
    rows = seq // (c * p * t)
    whole = dref.keep_mask(7, 3, 5, np.arange(seq), np.arange(b), h, prob)
    covered = []
    for r in range(c):
        for j in range(p):
            for k in range(t):
                runs = row_runs(rows, _G(c, r) if c > 1 else None, _G(p, j) if p > 1 else None, _G(t, k) if t > 1 else None)
                assert len(runs) <= 2 and runs[0][0] == 0 and sum(n for _, n, _ in runs) == rows
                mask = torch.cat([dref.keep_mask(7, 3, 5, t0 + np.arange(n), np.arange(b), h, prob) for _, n, t0 in runs])
                pos = local_positions(seq, c, r, p, j)[k * rows:(k + 1) * rows]
                assert torch.equal(mask, whole[pos]), (r, j, k, runs)
                covered.append(pos)
    assert torch.equal(torch.sort(torch.cat(covered)).values, torch.arange(seq))


def test_dropout_run_one_chunk_off_differs():
    """a rank whose second run is placed one chunk off draws different masks: the parity check would see it"""
    import _dropout_ref as dref
    from hetu_galvatron_b200.gpt_hf.GPTModel_tensor_parallel import row_runs
    runs = row_runs(16, _G(2, 0))
    assert runs == ((0, 8, 0), (8, 8, 24))
    good = torch.cat([dref.keep_mask(1, 0, 4, t0 + np.arange(n), np.arange(2), 16, 0.5) for _, n, t0 in runs])
    bad = torch.cat([dref.keep_mask(1, 0, 4, t0 + np.arange(n), np.arange(2), 16, 0.5) for _, n, t0 in ((0, 8, 0), (8, 8, 16))])
    assert not torch.equal(good, bad)


def test_bias_dropout_add_runs_match_one_call(monkeypatch):
    """bias_dropout_add over token runs (one backend call per run, dbias partials summed) equals per-run calls of the backend; one
    run covering the rows is today's single call"""
    import _dropout_ref as dref
    from hetu_galvatron_b200.core.runtime.tensor_parallel import random as rnd
    be = dref.DropoutOracleBackend.__new__(dref.DropoutOracleBackend)       # (its dropout methods keep no state)
    monkeypatch.setattr(rnd, "get_backend", lambda: be)
    g = torch.Generator().manual_seed(1)
    x, res = [torch.randn(12, 2, 16, generator=g).bfloat16().requires_grad_(True) for _ in range(2)]
    bias = torch.randn(16, generator=g).requires_grad_(True)
    rnd.begin_iteration(9, 4, 6)
    runs = ((0, 5, 3), (5, 7, 40))
    y = rnd.bias_dropout_add(x, bias, res, 0.25, 7, runs)
    dy = torch.randn(12, 2, 16, generator=g).bfloat16()
    y.backward(dy)
    want = torch.cat([be.dropout_add_fwd(x[a:a + n].detach(), bias.detach(), res[a:a + n].detach(), 0.25, 9, 4, 7, t0, 6)
                      for a, n, t0 in runs])
    assert torch.equal(y, want)
    parts = [be.dropout_bwd(dy[a:a + n], 0.25, 9, 4, 7, t0, 6, True) for a, n, t0 in runs]
    assert torch.equal(x.grad, torch.cat([d for d, _ in parts])) and torch.equal(res.grad, dy)
    assert torch.allclose(bias.grad, parts[0][1] + parts[1][1])
    one = rnd.bias_dropout_add(x.detach(), bias.detach(), res.detach(), 0.25, 7, 3)
    assert torch.equal(one, be.dropout_add_fwd(x.detach(), bias.detach(), res.detach(), 0.25, 9, 4, 7, 3, 6))
    with pytest.raises(ValueError, match="runs"):
        rnd.bias_dropout_add(x.detach(), None, None, 0.25, 7, ((0, 5, 3), (6, 6, 40)))


# ---- refusals ---------------------------------------------------------------------------------------------------------------
def _build_world1(monkeypatch, spec, **over):
    """build a GPT model with a cp-2 strategy on one process: construction-time checks run before any communication"""
    import smoke_model as sm
    from hetu_galvatron_b200 import gpt_hf
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    from hetu_galvatron_b200.gpt_hf import GPTModel_tensor_parallel as tp
    args = sm.tiny_args(**over)
    config = gpt_hf.set_model_config(gpt_hf.config_from_meta(dict(dict(n_layer=1, n_embd=64, n_head=2, vocab_size=128, n_positions=16),
                                                                  **spec)), args)
    return args, config, tp.GPTAttention_tp(config, 0, tp_group=None, sp_group=None, cp_group=CommGroup([0, 1]))


def test_attention_dropout_with_cp_is_refused(monkeypatch):
    with pytest.raises(NotImplementedError, match="attn_pdrop"):
        _build_world1(monkeypatch, dict(attn_pdrop=0.1))


def test_bad_sequence_length_with_cp_is_refused(monkeypatch):
    with pytest.raises(ValueError, match="multiple of 2 x cp"):
        _build_world1(monkeypatch, dict(n_positions=18))


def test_hidden_dropout_with_cp_is_allowed(monkeypatch):
    _, _, layer = _build_world1(monkeypatch, dict(resid_pdrop=0.1, embd_pdrop=0.1))
    assert layer.use_zigzag_cp and layer.attention.use_cp

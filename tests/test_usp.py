"""Ulysses and zigzag context parallelism on the same layer (the reference's two-dimensional sequence parallelism) on the CPU.

* Strategies with ``use_sp=1`` and cp > 1 on one row run the product's layer and schedule code over gloo on the oracle backend and
  reproduce the single-process oracle under the criteria of tests/test_host_runtime.py (loss 5e-3 rel, every parameter's gradient
  3e-2 rel-L2, then one AdamW step), with each cp exchange: ``cp_comm="allgather"`` and ``"ring"`` (tests/_cp_ring_ref.py's transport).
* The token layout: ``redistribute.local_positions`` against a restatement of the reference's
  ``get_pos_emb_on_this_cp_sp_rank_galvatron``; the RoPE rows and the token ids a Llama rank holds are those positions; a layout
  that slices the sp share before the zigzag fails the parity test.
* The communication groups of such strategies are held bit-exact by tests/test_comm_groups.py (the golden file has them).
* Construction limits: a composed layer no longer raises; attention dropout with CP still does; a sequence length that is not a
  multiple of 2 x cp x sp is refused."""
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

_PORT = [31400]

_USP = dict(use_ulysses=True, sequence_parallel=True, global_cp_deg=2, vocab_cp=2)
CASES = {
    # --use-ulysses sp2 x cp2: every row (vocabulary rows too) is sp 2 x cp 2
    "usp_sp2_cp2": (4, dict(_USP, global_tp_deg=2, vocab_tp=2)),
    "usp_sp2_cp2_dp2_zero3_ckpt": (8, dict(_USP, global_tp_deg=2, vocab_tp=2, sdp=1, global_checkpoint=1, chunks=2,
                                           global_train_batch_size=8)),
    # 2 KV heads over sp 4: K/V are replicated to the query heads before the exchange
    "usp_sp4_cp2_kv_replicated": (8, dict(_USP, global_tp_deg=4, vocab_tp=4)),
    "usp_sp2_cp2_pp2_1f1b": (8, dict(_USP, global_tp_deg=2, vocab_tp=2, pp_deg=2, chunks=2, pipeline_type="pipedream_flush")),
    # relocation: Megatron-SP tp2 rows -> a use_sp=1, cp=2 layer -> back
    "usp_mixed_tp2_to_sp2cp2": (4, dict(sequence_parallel=True, _strategy_json={
        "pp_deg": 1, "tp_sizes_enc": "2,2", "tp_consecutive_flags": "1,1", "dp_types_enc": "0,0", "use_sp": "0,1", "cp_sizes_enc": "1,2",
        "checkpoint": "0,0", "global_bsz": 4, "chunks": 1, "default_dp_type": "zero2", "vtp": 2, "vsp": 0, "vcp": 1})),
}
PARAMS = [(name, comm) for name in CASES for comm in ("allgather", "ring")]


def launch(world, config, comm, timeout=900, backend="oracle", worker=None):
    from _launch import launch_ranks
    _PORT[0] += 1
    extra_env = config.pop("_env", {})
    if worker is None:
        worker = "_cp_ring_worker" if comm == "ring" else "_host_worker"
    return launch_ranks(worker, world, config, _PORT[0] + os.getpid() % 500, timeout=timeout, backend=backend, extra_env=extra_env)


@pytest.mark.parametrize("name,comm", PARAMS, ids=["%s-%s" % p for p in PARAMS])
def test_usp_strategy_matches_oracle(name, comm):
    world, cfg = CASES[name]
    rep = launch(world, dict(cfg), comm)
    assert rep["max_grad_err"] < 3e-2
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert len(rep["losses"]) == 2          # the second loss follows one AdamW step on the re-gathered parameters
    if comm == "ring":
        assert rep["ring_pushes"] > 0


# ---- layout ---------------------------------------------------------------------------------------------------------------------
def reference_positions(seq, cp, cp_rank, sp, sp_rank):
    """Restatement of get_pos_emb_on_this_cp_sp_rank_galvatron (galvatron/site_package/megatron/core/models/common/embeddings/
    rotary_pos_embedding.py:33-56) on a [seq] table of positions: view as 2cp chunks, index_select chunks (r, 2cp-1-r), then keep the
    sp rank's contiguous slice.  (The function itself moves its index to CUDA.)"""
    pos_emb = torch.arange(seq)
    if cp == 1:
        return pos_emb
    cp_idx = torch.tensor([cp_rank, 2 * cp - cp_rank - 1])
    pos_emb = pos_emb.view(2 * cp, -1).index_select(0, cp_idx).view(-1)
    if sp > 1:
        n = pos_emb.shape[0] // sp
        pos_emb = pos_emb[sp_rank * n:(sp_rank + 1) * n]
    return pos_emb


def sp_first_positions(seq, cp, cp_rank, sp, sp_rank):
    """the wrong composition: the sp share taken from the whole sequence first, then zigzagged inside it"""
    n = seq // sp
    inner = reference_positions(n, cp, cp_rank, 1, 0)
    return inner + sp_rank * n


_LAYOUTS = [(c, p) for c in (1, 2, 4, 8) for p in (1, 2, 3, 4, 8) if c * p <= 16 and (c, p) != (1, 1)]


@pytest.mark.parametrize("c,p", _LAYOUTS)
def test_local_positions_known_answer(c, p):
    from hetu_galvatron_b200.core.runtime.redistribute import local_positions
    seq = 2 * c * p * 5
    seen = []
    for r in range(c):
        for j in range(p):
            got = local_positions(seq, c, r, p, j)
            # (cp 1: the reference's function returns the table untouched and Ulysses alone offsets RoPE by s/p * j,
            # models/llama_hf/LlamaModel_tensor_parallel.py:65-66)
            want = reference_positions(seq, c, r, p, j) if c > 1 else torch.arange(j * seq // p, (j + 1) * seq // p)
            assert torch.equal(got, want), (c, p, r, j)
            seen.append(got)
    assert torch.equal(torch.sort(torch.cat(seen)).values, torch.arange(seq))      # every token held exactly once
    if c > 1 and p > 1:
        assert any(not torch.equal(reference_positions(seq, c, r, p, j), sp_first_positions(seq, c, r, p, j))
                   for r in range(c) for j in range(p))


def test_local_positions_refuses_bad_length():
    from hetu_galvatron_b200.core.runtime.redistribute import local_positions
    with pytest.raises(ValueError, match="2 x cp x sp"):
        local_positions(24, 2, 0, 4, 0)


@pytest.mark.parametrize("c,p", [(2, 2), (2, 4), (4, 2), (2, 3)])
def test_llama_rank_holds_reference_positions(c, p):
    """the RoPE rows and the token ids of a Llama rank (sp rank j of cp rank r) are the reference's positions"""
    import types
    from hetu_galvatron_b200.core.runtime.backend import set_backend
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    from hetu_galvatron_b200.llama_hf import LlamaModel_sequential as seqmod
    from hetu_galvatron_b200.llama_hf import LlamaModel_tensor_parallel as tpmod
    from oracle.gloo_backend import OracleBackend
    set_backend(OracleBackend())
    seq, hd = 2 * c * p * 4, 16

    class G(CommGroup):
        def __init__(self, ranks, me):
            super().__init__(ranks)
            self.me = me

        def rank_in_group(self, rank=None):
            return self.me
    tokens = torch.arange(seq)[None] * 7 + 3
    for r in range(c):
        for j in range(p):
            want = reference_positions(seq, c, r, p, j)
            cpg, spg = G(list(range(c)), r), G(list(range(p)), j)
            assert torch.equal(seqmod._zigzag_local(tokens, cpg, spg)[0], tokens[0, want])
            att = types.SimpleNamespace(cp_size=c, sp_size=p, use_ulysses=True, cp_group=cpg, sp_group=spg, head_dim=hd,
                                        rotary_base=10000.0, _rope_cache={})
            att._rope = types.MethodType(_fp32_rope, att)
            cos, sin = tpmod.LlamaAttention_tp._rope_zigzag(att, seq // (c * p), "cpu")
            full_cos, full_sin = _fp32_rope(att, seq, 0, "cpu")
            assert torch.equal(cos, full_cos[want]) and torch.equal(sin, full_sin[want])
            wrong = sp_first_positions(seq, c, r, p, j)
            if not torch.equal(want, wrong):
                assert not torch.equal(cos, full_cos[wrong])


def _fp32_rope(self, seq, offset, device):
    from hetu_galvatron_b200.core.runtime.backend import get_backend
    return get_backend().rope_tables(seq, self.head_dim, self.rotary_base, offset, torch.float32, device)


def test_sp_first_layout_fails_parity():
    """the parity test sees a wrong layout: with the sp share taken before the zigzag (tokens, labels and RoPE all moved together)
    the sp2 x cp2 run runs to the end of its first step and fails the oracle comparison itself (not some other error)"""
    world, cfg = CASES["usp_sp2_cp2"]
    rep = launch(world, dict(cfg, _env={"HGB_TEST_USP_LAYOUT": "sp_first"}), "allgather", worker="_usp_worker")
    assert rep["parity_failed"], rep
    assert abs(rep["loss"] - rep["ref_loss"]) > 5e-3 * abs(rep["ref_loss"]) or rep["max_grad_err"] >= 3e-2, rep


def test_golden_groups_hold_composed_strategies():
    """tests/test_comm_groups.py holds every golden case bit-exact; these are the ones with Ulysses and cp > 1 on one row"""
    with open(os.path.join(ROOT, "tests", "golden", "comm_groups.json")) as f:
        cases = json.load(f)["cases"]
    names = [c["name"] for c in cases if any(s > 1 and k > 1 for s, k in zip(c["hp_configs_whole"]["sp_sizes_whole"],
                                                                               c["hp_configs_whole"]["cp_sizes_whole"]))]
    assert {"uniform_w4_pp1_sp2_cp2_vtp1", "uniform_w8_pp1_sp4_cp2_vtp1", "uniform_w8_pp1_sp2_cp4_vtp1", "cp_sp_mixed"} <= set(names)


# ---- construction ---------------------------------------------------------------------------------------------------------------
def _attention(seq, sp, cp, n_heads=4, n_kv=2, attention_dropout=0.0, cp_comm="allgather"):
    import types
    import smoke_model as sm
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    from hetu_galvatron_b200.core.runtime.tensor_parallel.transformer import AttnMaskType, ParallelAttention
    sm.tiny_args(seq_length=seq, cp_comm=cp_comm)
    conf = types.SimpleNamespace(hidden_size=32 * n_heads, num_attention_heads=n_heads, num_query_groups=n_kv, kv_channels=32,
                                 init_method_std=0.02, sequence_parallel=False, attention_dropout=attention_dropout)
    return ParallelAttention(conf, 1, attn_mask_type=AttnMaskType.causal, sp_group=CommGroup(list(range(sp))),
                             cp_group=CommGroup(list(range(0, sp * cp, sp))), use_ulysses=True, use_zigzag_cp=True, device="meta")


@pytest.mark.parametrize("cp_comm", ["allgather", "ring"])
def test_composed_layer_builds(cp_comm):
    m = _attention(64, 2, 2, cp_comm=cp_comm)
    assert m.use_ulysses and m.use_cp and m.cp_comm == cp_comm
    assert m.kv_heads_attn == 1                                  # 2 KV heads over sp 2
    assert _attention(64, 4, 2).kv_heads_attn == 1              # 2 KV heads over sp 4: replicated to 4 heads, then 1 per rank
    assert _attention(96, 3, 2, n_heads=6, n_kv=6).kv_heads_attn == 2


def test_composed_layer_limits():
    with pytest.raises(ValueError, match="2 x cp x sp"):
        _attention(36, 2, 2)
    with pytest.raises(AssertionError, match="Ulysses degree"):
        _attention(64, 4, 2, n_heads=6, n_kv=6)
    with pytest.raises(NotImplementedError, match="dropout"):      # attention-probability dropout with CP stays refused
        _attention(64, 2, 2, attention_dropout=0.1)

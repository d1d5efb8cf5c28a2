"""Host-logic tests of the runtime (schedules, sharded units, TP / Megatron-SP / Ulysses layers, relocation, pipeline) on
CPU: N ranks over gloo run the product's layer/schedule code on the oracle backend and must reproduce the single-process
oracle's loss (5e-3 rel, the reference's own criterion tests/core/test_tp.py:121) and per-parameter gradients (rel-L2 < 3e-2,
bf16 rounding noise) on the global batch.  Strategy corpus follows tests/core/test_{fsdp,tp,pp,redistributed,hybrid}.py."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
_PORT = [29600]


def launch(world, config, timeout=600, backend="oracle"):
    from _launch import launch_ranks
    _PORT[0] += 1
    extra_env = config.pop("_env", {})
    return launch_ranks("_host_worker", world, config, _PORT[0] + os.getpid() % 500, timeout=timeout, backend=backend, extra_env=extra_env)


WORLD1 = {
    "plain": dict(),
    "ckpt_chunks2": dict(global_checkpoint=1, chunks=2),
    # --recompute_activations: wgrad inputs (SwiGLU / RMSNorm outputs) are redone in backward instead of saved
    "recompute_activations": dict(recompute_activations=True),
    "ddp_no_async": dict(default_dp_type="ddp", chunks=2, async_grad_reduce=False),
    "zero3": dict(sdp=1),
}

WORLD2 = {
    "dp2_zero2": dict(default_dp_type="zero2"),
    "dp2_zero3_ckpt_chunks2": dict(sdp=1, global_checkpoint=1, chunks=2),
    "dp2_ddp_chunks2": dict(default_dp_type="ddp", chunks=2),
    # --reduce_in_fp32 (fp32 unsharded gradients and reduction, arguments.py:187) and --entropy_in_fp32 (:192)
    "dp2_zero2_reduce_fp32_chunks2": dict(default_dp_type="zero2", chunks=2, reduce_in_fp32=True, entropy_in_fp32=True),
    "dp2_zero3_nopool": dict(sdp=1, embed_sdp=1, zero3_pool_slots=0),
    "dp2_zero3_pool2": dict(sdp=1, embed_sdp=1, zero3_pool_slots=2),
    "dp2_zero3_pool2_no_async_chunks2": dict(sdp=1, embed_sdp=1, zero3_pool_slots=2, chunks=2, async_grad_reduce=False),
    "dp2_zero2_no_async_chunks2": dict(default_dp_type="zero2", chunks=2, async_grad_reduce=False),
    "tp2": dict(global_tp_deg=2, vocab_tp=2),
    # context parallelism (SURVEY 8f-1): zigzag token chunks, keys/values gathered over the cp group, per-chunk causal attention
    "cp2": dict(global_cp_deg=2, vocab_cp=2),
    # the cp degree changes between rows (embedding / head cp 1, layers cp 2): relocation re-zigzags the sequence.  The
    # reference applies the wrong permutation here (SURVEY 8g, first row); this runtime reads the group slots for what they hold
    "cp_mixed_vcp1_layers_cp2": dict(sequence_parallel=True, _strategy_json={
        "pp_deg": 1, "tp_sizes_enc": "1,1", "tp_consecutive_flags": "1,1", "dp_types_enc": "0,0", "use_sp": "0,0", "cp_sizes_enc": "2,2",
        "checkpoint": "0,0", "global_bsz": 4, "chunks": 1, "default_dp_type": "zero2", "vtp": 1, "vsp": 0, "vcp": 1}),
    "tp2_megatron_sp": dict(global_tp_deg=2, vocab_tp=2, sequence_parallel=True),
    "tp2_megatron_sp_recompute_activations": dict(global_tp_deg=2, vocab_tp=2, sequence_parallel=True, recompute_activations=True),
    "dp2_zero3_ckpt_recompute_activations": dict(sdp=1, embed_sdp=1, global_checkpoint=1, zero3_pool_slots=2, recompute_activations=True),
    # shapes the fused GEMM+reduce-scatter accepts (M = 256 = p x 128): on the GPU the row-parallel forward and the
    # column-parallel dgrad run as ONE kernel pair inside the model (forced: these K are below the profitability threshold)
    "tp2_megatron_sp_fused_gemm_rs": dict(global_tp_deg=2, vocab_tp=2, sequence_parallel=True, _spec={"n_positions": 256},
                                          _env={"HGB_FUSE_GEMM_RS": "force"}),
    "ulysses2": dict(global_tp_deg=2, use_ulysses=True, sequence_parallel=True, vocab_tp=2),
    "pp2_1f1b_chunks4": dict(pp_deg=2, chunks=4, pipeline_type="pipedream_flush", global_train_batch_size=8),
    "pp2_gpipe_chunks2": dict(pp_deg=2, chunks=2, pipeline_type="gpipe"),
    "relocate_tp1_tp2": dict(_strategy_json={"pp_deg": 1, "tp_sizes_enc": "1,2", "tp_consecutive_flags": "1,1",
                                             "dp_types_enc": "0,1", "use_sp": "0,0", "checkpoint": "0,1", "global_bsz": 4,
                                             "chunks": 2, "default_dp_type": "zero2", "vtp": 2, "vsp": 0}),
}

WORLD4 = {
    "tp2_dp2_sp_zero2": dict(global_tp_deg=2, vocab_tp=2, sequence_parallel=True, default_dp_type="zero2", chunks=2),
    # tests/core/test_pp.py:126-128 (pp 4, both schedules, 8 microbatches) and test_tp.py:132-133 (tp 4: plain, Megatron-SP, Ulysses)
    "pp4_1f1b_chunks8": dict(pp_deg=4, chunks=8, pipeline_type="pipedream_flush", global_train_batch_size=8, _spec={"n_layers": 4}),
    "pp4_gpipe_chunks2": dict(pp_deg=4, chunks=2, pipeline_type="gpipe", _spec={"n_layers": 4}),
    "tp4": dict(global_tp_deg=4, vocab_tp=4, chunks=2, _spec={"n_kv_heads": 4}),
    "tp4_megatron_sp": dict(global_tp_deg=4, vocab_tp=4, sequence_parallel=True, chunks=2, _spec={"n_kv_heads": 4}),
    "tp4_ulysses": dict(global_tp_deg=4, vocab_tp=4, use_ulysses=True, sequence_parallel=True, chunks=2, _spec={"n_kv_heads": 4}),
    "pp2_tp2_1f1b": dict(pp_deg=2, global_tp_deg=2, vocab_tp=2, chunks=2, pipeline_type="pipedream_flush"),
    # BASELINE config (3) shape: PP2 x TP2 x ZeRO-2 with Megatron-SP, 1F1B-flush, 4 microbatches
    "baseline3_pp2_tp2_sp_zero2": dict(pp_deg=2, global_tp_deg=2, vocab_tp=2, sequence_parallel=True, default_dp_type="zero2",
                                       chunks=4, pipeline_type="pipedream_flush", global_train_batch_size=8),
    # BASELINE config (4) shape: Ulysses sequence parallel x data parallel (grads reduce over DP x SP)
    "baseline4_ulysses2_dp2": dict(global_tp_deg=2, use_ulysses=True, sequence_parallel=True, vocab_tp=2, default_dp_type="zero2",
                                   chunks=2, global_train_batch_size=8),
    # BASELINE config (5) shape: ZeRO-3 on every layer + activation checkpointing
    "baseline5_zero3_ckpt_dp4": dict(sdp=1, global_checkpoint=1, embed_sdp=1, chunks=1, global_train_batch_size=8),
    "cp2_dp2_zero3_ckpt": dict(global_cp_deg=2, vocab_cp=2, sdp=1, global_checkpoint=1, chunks=2, global_train_batch_size=8),
    "cp_mixed_tp2_to_cp2": dict(sequence_parallel=True, _strategy_json={
        "pp_deg": 1, "tp_sizes_enc": "2,1", "tp_consecutive_flags": "1,1", "dp_types_enc": "0,1", "use_sp": "0,0", "cp_sizes_enc": "1,2",
        "checkpoint": "0,1", "global_bsz": 4, "chunks": 2, "default_dp_type": "zero2", "vtp": 2, "vsp": 0, "vcp": 1}),
    "cp_mixed_cp4_to_tp2cp2": dict(sequence_parallel=True, _strategy_json={
        "pp_deg": 1, "tp_sizes_enc": "1,2", "tp_consecutive_flags": "1,1", "dp_types_enc": "0,0", "use_sp": "0,0", "cp_sizes_enc": "4,2",
        "checkpoint": "0,0", "global_bsz": 4, "chunks": 1, "default_dp_type": "zero2", "vtp": 1, "vsp": 0, "vcp": 2}),
    "cp2_pp2_1f1b": dict(global_cp_deg=2, vocab_cp=2, pp_deg=2, chunks=2, pipeline_type="pipedream_flush"),
    "cp2_tp2_megatron_sp": dict(global_cp_deg=2, vocab_cp=2, global_tp_deg=2, vocab_tp=2, sequence_parallel=True),
    "hybrid_mixed": dict(sequence_parallel=True, _spec={"n_kv_heads": 4},
                         _strategy_json={"pp_deg": 1, "tp_sizes_enc": "2,4", "tp_consecutive_flags": "1,1", "dp_types_enc": "1,0",
                                         "use_sp": "1,0", "checkpoint": "0,1", "global_bsz": 8, "chunks": 2,
                                         "default_dp_type": "zero2", "vtp": 2, "vsp": 0}),
}


# The reference's own 8-GPU hybrid corpus, verbatim (tests/core/test_hybrid.py:122-183): per-layer tp 1/2/4/8 with Megatron-TP
# and Ulysses layers alternating, ZeRO-2/ZeRO-3 alternating, checkpointing on the last two layers, relocation between every
# pair of layers, with and without pipeline parallelism, vocab tp 2 or Ulysses-sp 4; Megatron sequence parallelism on, as the
# reference test sets it (test_hybrid.py:45).
_HYBRID = dict(tp_consecutive_flags="1,1,1,1", use_sp="0,1,0,1", checkpoint="0,0,1,1", global_bsz=32,
               pipeline_type="pipedream_flush", default_dp_type="zero2")
# (ffn 384: a tensor-parallel degree of 8 leaves K = 48 for the row-parallel GEMM -- the wgmma kernel wants multiples of 8)
_SPEC8 = {"n_heads": 8, "n_kv_heads": 8, "n_layers": 4, "ffn_dim": 384}
def _redistributed(tp, vtp, sp):
    """tests/core/test_redistributed.py:49-69,141-146: zero2, no checkpointing, per-layer tp lists that force a relocation between
    every pair of layers and between the layers and the vocabulary rows, with and without Megatron sequence parallelism."""
    return dict(_spec=_SPEC8, sequence_parallel=sp, _strategy_json=dict(
        pp_deg=1, tp_sizes_enc=tp, tp_consecutive_flags="1,1,1,1", dp_types_enc="0,0,0,0", use_sp="0,0,0,0", checkpoint="0,0,0,0",
        global_bsz=32, chunks=2, pp_division="4", pipeline_type="pipedream_flush", default_dp_type="zero2", vtp=vtp, vsp=0))


WORLD8 = {
    "ref_redistributed_tp1248_vtp8": _redistributed("1,2,4,8", 8, False),
    "ref_redistributed_tp1248_vtp8_sp": _redistributed("1,2,4,8", 8, True),
    "ref_redistributed_tp2821_vtp4": _redistributed("2,8,2,1", 4, False),
    "ref_redistributed_tp2821_vtp4_sp": _redistributed("2,8,2,1", 4, True),
    "ref_redistributed_tp8412_vtp2": _redistributed("8,4,1,2", 2, False),
    "ref_redistributed_tp8412_vtp2_sp": _redistributed("8,4,1,2", 2, True),
    "ref_hybrid0_pp1_vtp2": dict(_spec=_SPEC8, sequence_parallel=True, _strategy_json=dict(_HYBRID, pp_deg=1, tp_sizes_enc="1,2,4,8", dp_types_enc="0,1,0,1",
                                                                  chunks=2, pp_division="4", vtp=2, vsp=0)),
    "ref_hybrid1_pp1_vsp4": dict(_spec=_SPEC8, sequence_parallel=True, _strategy_json=dict(_HYBRID, pp_deg=1, tp_sizes_enc="1,2,4,8", dp_types_enc="1,0,1,0",
                                                                  chunks=2, pp_division="4", vtp=4, vsp=1)),
    "ref_hybrid2_pp2_vtp2": dict(_spec=_SPEC8, sequence_parallel=True, _strategy_json=dict(_HYBRID, pp_deg=2, tp_sizes_enc="1,2,4,2", dp_types_enc="0,1,0,1",
                                                                  chunks=2, pp_division="3,1", vtp=2, vsp=0)),
    # TP2 x CP2 x DP2 (the SURVEY 8c known-answer mapping: tp {0,1}.. cp {0,2}.. dp {0,4}.. sdp {0,2,4,6}..), ZeRO-3 + checkpointing
    "tp2_cp2_dp2_zero3": dict(_spec=_SPEC8, sequence_parallel=True, global_tp_deg=2, vocab_tp=2, global_cp_deg=2, vocab_cp=2, sdp=1,
                              global_checkpoint=1, chunks=2, global_train_batch_size=8),
    "ref_hybrid3_pp2_vsp4": dict(_spec=_SPEC8, sequence_parallel=True, _strategy_json=dict(_HYBRID, pp_deg=2, tp_sizes_enc="1,2,4,2", dp_types_enc="1,0,1,0",
                                                                  chunks=4, pp_division="2,2", vtp=4, vsp=1)),
}


@pytest.mark.parametrize("name", sorted(WORLD1))
def test_world1(name):
    rep = launch(1, dict(WORLD1[name]))
    assert rep["max_grad_err"] < 3e-2
    if name == "recompute_activations":     # same deterministic ops, redone: identical numbers
        base = launch(1, dict(WORLD1["plain"]))
        assert rep["losses"] == base["losses"] and rep["max_grad_err"] == base["max_grad_err"]


@pytest.mark.parametrize("name", sorted(WORLD2))
def test_world2(name):
    rep = launch(2, dict(WORLD2[name]))
    assert rep["max_grad_err"] < 3e-2
    if name == "dp2_zero2":
        # one all-gather and one reduction per layer per step
        assert set(rep["n_unshard"]) <= {0, 1} and set(rep["n_reduce"]) == {1}
    if name == "dp2_zero2_no_async_chunks2":
        assert set(rep["n_reduce"]) == {2}     # --no_async_grad_reduce: every microbatch is reduced
    if name.startswith("dp2_zero3_pool2"):
        # two rotating buffers serve every layer: parameters are re-gathered for backward (FULL_SHARD), gradients share a
        # pool too, nothing stays held after the step -- and the numbers are those of the one-buffer-per-layer layout
        assert set(rep["pools"]) == {"param:0-1", "grad:0-1"} and all(v[0] == 2 and v[2] == 0 for v in rep["pools"].values())
        assert max(rep["n_unshard_2steps"]) >= 2 * 2
        base = launch(2, dict(WORLD2["dp2_zero3_nopool" if "chunks2" not in name else "dp2_zero3_nopool"], **(
            {} if "chunks2" not in name else dict(chunks=2, async_grad_reduce=False))))
        assert rep["loss"] == base["loss"] and rep["loss_step1"] == base["loss_step1"]
    if name == "dp2_zero3_nopool":
        assert rep["pools"] == {}
    if name == "tp2_megatron_sp_recompute_activations":
        base = launch(2, dict(WORLD2["tp2_megatron_sp"]))
        assert rep["losses"] == base["losses"] and rep["max_grad_err"] == base["max_grad_err"]


@pytest.mark.parametrize("name", sorted(WORLD4))
def test_world4(name):
    rep = launch(4, dict(WORLD4[name]))
    assert rep["max_grad_err"] < 3e-2


@pytest.mark.parametrize("name", sorted(WORLD8))
def test_world8(name):
    rep = launch(8, dict(WORLD8[name]), timeout=900)
    assert rep["max_grad_err"] < 3e-2

#!/usr/bin/env python
"""Run the reference's UNMODIFIED Search Engine (galvatron/core/search_engine + csrc/dp_core.cpp) on profiles measured on the
target GPU and emit Galvatron strategy JSONs for Llama-3-8B shapes (galvatron_config_llama3-8b_<N>gpus.json under --out-root).

Needs a checkout of the upstream Hetu-Galvatron sources (--reference).  Inputs:
  * computation profile  : per-layer / head forward ms per sample measured with THIS runtime on the target GPU
                           (--layer-ms/--other-ms), static mode (search_engine.py:123-131)
  * memory profile       : analytic from the model shapes in the reference's units (MB; parameter_size = fp32 MB,
                           model_states = 4 x parameter_size, cost_model.py:118), activations from the saved-tensor list
                           of our layer (DESIGN.md section 3)
  * hardware profile     : all-reduce / p2p bandwidth and sp_time tables measured with OUR collectives
                           (scripts/bench_collectives.py) -- NVSwitch makes consecutive and strided groups identical
The search DP core is compiled from <reference>/csrc/dp_core.cpp into oracle/_ref/ (never copied into the repo).
"""
import argparse
import glob
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_dp_core(ref):
    """oracle/build_ref.py owns the recipe."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("_oracle_build", os.path.join(ROOT, "oracle", "build_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    so = mod.build(ref)
    if so is None:
        raise SystemExit("the reference sources are not present: the Search Engine cannot run here")
    return os.path.dirname(so)


def llama3_8b_profiles(layer_ms, other_ms, seq, recompute_activations=False):
    h, ffn, nh, nkv, V = 4096, 14336, 32, 8, 128256
    hn = h // nh
    layer_params = (nh + 2 * nkv) * hn * h + nh * hn * h + 3 * ffn * h + 2 * h
    mb = lambda nbytes: nbytes / 2 ** 20  # noqa: E731
    # saved activations of one layer per sample (bf16): x, normed x, q/k/v, attn out, h1, normed h1, gate_up, act (+ fp32 lse / rstd)
    act_full = mb(seq * (h * 2 * 5 + (nh + 2 * nkv) * hn * 2 + 2 * ffn * 2 + ffn * 2) + seq * (nh + 2) * 4)
    if recompute_activations:   # --recompute_activations: the SwiGLU output and the two RMSNorm outputs are not kept
        act_full -= mb(seq * (ffn * 2 + 2 * h * 2))
    # tensor parallel shards everything except the two layer inputs + norm outputs (no sequence parallel): approx split
    act = {"1": act_full}
    for t in (2, 4, 8):
        replicated = mb(seq * h * 2 * 4)
        act[str(t)] = replicated + (act_full - replicated) / t
    act["checkpoint"] = mb(seq * h * 2)
    time_cfg = {"layertype_0_bsz1_seq%d" % seq: layer_ms, "layertype_other_bsz1_seq%d" % seq: other_ms}
    emb = V * h
    states = lambda n_params: mb(n_params * 16)  # noqa: E731  fp32 param + grad + 2 Adam moments
    logits_act = mb(seq * V * 2) + mb(seq * h * 2 * 3)
    mem_cfg = {
        "layertype_0": {str(seq): {"parameter_size": mb(layer_params * 4), "tp_activation_per_bsz_dict": act}},
        "other_memory_pp_off": {str(seq): {"model_states": {str(t): states(2 * emb + h) / t for t in (1, 2, 4, 8)},
                                           "activation": {str(t): logits_act / t + mb(seq * h * 2) for t in (1, 2, 4, 8)}}},
        "other_memory_pp_on_first": {str(seq): {"model_states": {str(t): states(emb) / t for t in (1, 2, 4, 8)},
                                                "activation": {str(t): mb(seq * h * 2 * 2) for t in (1, 2, 4, 8)}}},
        "other_memory_pp_on_last": {str(seq): {"model_states": {str(t): states(emb + h) / t for t in (1, 2, 4, 8)},
                                               "activation": {str(t): logits_act / t for t in (1, 2, 4, 8)}}},
    }
    return time_cfg, mem_cfg


def hardware_profiles(bus_gbs, p2p_gbs, latency_ms):
    """allreduce_size_<n>_consec_<c> in GB/s (bus bandwidth), pp_size_<n> GB/s, sp_time tables in ms: a latency + size/bandwidth
    model through the measured points (NVSwitch: identical for consecutive and strided groups)."""
    ar = {"allreduce_size_8_consec_1": bus_gbs, "allreduce_size_4_consec_1": bus_gbs, "allreduce_size_4_consec_0": bus_gbs,
          "allreduce_size_2_consec_1": bus_gbs, "allreduce_size_2_consec_0": bus_gbs}
    p2p = {"pp_size_2": p2p_gbs, "pp_size_4": p2p_gbs, "pp_size_8": p2p_gbs}
    sp = {}
    for n in (8, 4, 2):
        for mbs in (1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024):
            nbytes = mbs * 2 ** 20
            sp["allreduce_size_%d_%dMB_time" % (n, mbs)] = latency_ms + nbytes * 2 * (n - 1) / n / (bus_gbs * 1e9) * 1e3
            sp["all2all_size_%d_%dMB_time" % (n, mbs)] = latency_ms + nbytes * (n - 1) / n / (bus_gbs * 1e9) * 1e3
    return ar, p2p, {"overlap_coe": 1.05}, sp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="checkout of the upstream Hetu-Galvatron sources")
    ap.add_argument("--layer-ms", type=float, required=True, help="forward ms of one layer for one 8192-token sample (measured)")
    ap.add_argument("--other-ms", type=float, required=True, help="forward ms of embedding + lm_head + loss for one sample (measured)")
    ap.add_argument("--bus-gbs", type=float, required=True, help="collective bus GB/s (scripts/bench_collectives.py)")
    ap.add_argument("--p2p-gbs", type=float, required=True, help="peer-copy GB/s")
    ap.add_argument("--latency-ms", type=float, default=0.02)
    ap.add_argument("--memory-gb", type=int, default=64, help="memory the engine may plan with (80 GB H100 less the arena and headroom)")
    ap.add_argument("--seq", type=int, default=8192)
    ap.add_argument("--gpus", type=int, nargs="*", default=[1, 2, 4, 8])
    ap.add_argument("--hardware-dir", default=None,
                    help="measured tables from scripts/emit_hardware_profile.py (used when present; else the latency+bandwidth model)")
    ap.add_argument("--recompute-activations", action="store_true",
                    help="memory profile of the runtime's --recompute_activations mode (NOT the bench default; measure before use)")
    ap.add_argument("--out-root", required=True,
                    help="where search_profiles/ and searched/ are written (tests point this at a temp dir)")
    ap.add_argument("--debug-memory", action="store_true", help="print the engine's per-layer memory model for the dp-only strategy")
    opts = ap.parse_args()

    ref = os.path.abspath(opts.reference)
    dp_dir = build_dp_core(ref)
    sys.path[:0] = [dp_dir, os.path.join(ROOT, "oracle", "ref_shim"), ref, os.path.join(ref, "galvatron", "site_package"), ref]
    import warnings
    warnings.filterwarnings("ignore")
    from galvatron.core.search_engine.search_engine import GalvatronSearchEngine
    from tests.utils.search_args import SearchArgs

    work = os.path.join(opts.out_root, "search_profiles")
    os.makedirs(work, exist_ok=True)
    model_name = "llama3-8b_seqlen%d" % opts.seq
    time_cfg, mem_cfg = llama3_8b_profiles(opts.layer_ms, opts.other_ms, opts.seq, opts.recompute_activations)
    json.dump(time_cfg, open(os.path.join(work, "computation_profiling_bf16_%s.json" % model_name), "w"), indent=2)
    json.dump(mem_cfg, open(os.path.join(work, "memory_profiling_bf16_%s.json" % model_name), "w"), indent=2)
    results = {}
    for n in opts.gpus:
        ar, p2p, ov, sp = hardware_profiles(opts.bus_gbs, opts.p2p_gbs, opts.latency_ms)
        measured = {k: os.path.join(opts.hardware_dir, f) for k, f in (
            ("ar", "allreduce_bandwidth_1nodes_8gpus_per_node.json"), ("p2p", "p2p_bandwidth_1nodes_8gpus_per_node.json"),
            ("ov", "overlap_coefficient.json"), ("sp", "sp_time_1nodes_8gpus_per_node.json"))} if opts.hardware_dir else {}
        if measured and all(os.path.exists(f) for f in measured.values()):   # tables measured with OUR collectives
            ar.update(json.load(open(measured["ar"])))
            p2p.update(json.load(open(measured["p2p"])))
            ov = json.load(open(measured["ov"]))
            sp.update(json.load(open(measured["sp"])))
        json.dump(ar, open(os.path.join(work, "allreduce_bandwidth_1nodes_%dgpus_per_node.json" % n), "w"), indent=2)
        json.dump(p2p, open(os.path.join(work, "p2p_bandwidth_1nodes_%dgpus_per_node.json" % n), "w"), indent=2)
        json.dump(ov, open(os.path.join(work, "overlap_coefficient.json"), "w"), indent=2)
        json.dump(sp, open(os.path.join(work, "sp_time_1nodes_%dgpus_per_node.json" % n), "w"), indent=2)
        args = SearchArgs()
        args.num_nodes, args.num_gpus_per_node = 1, n
        args.memory_constraint = opts.memory_gb
        args.settle_bsz, args.settle_chunk = 8 * n, -1
        args.min_bsz = args.max_bsz = 8 * n
        args.default_dp_type, args.pipeline_type = "zero2", "pipedream_flush"
        args.mixed_precision, args.sequence_parallel, args.async_grad_reduce = "bf16", False, True
        args.max_tp_deg, args.max_pp_deg = min(8, n), min(8, n)
        args.time_profile_mode = args.memory_profile_mode = "static"
        for k in ("memory_profiling_path", "time_profiling_path", "allreduce_bandwidth_config_path", "p2p_bandwidth_config_path",
                  "overlap_coe_path", "sp_time_path"):
            setattr(args, k, work)
        out_dir = os.path.join(work, "out_%dgpus" % n)
        os.makedirs(out_dir, exist_ok=True)
        for f in glob.glob(os.path.join(out_dir, "*.json")):
            os.remove(f)
        args.output_config_path = out_dir
        args.log_dir = os.path.join(work, "logs")
        args.local_rank = 0
        args.model_size = "llama3-8b"
        # model arguments the cost models read directly (normally filled by the family's arguments.py)
        args.hidden_size, args.seq_length, args.num_hidden_layers = 4096, opts.seq, 32
        args.num_attention_heads, args.vocab_size, args.padded_vocab_size = 32, 128256, 128256
        args.ffn_hidden_size = 14336
        engine = GalvatronSearchEngine(args)
        engine.set_search_engine_info(work, [{"hidden_size": 4096, "seq_len": opts.seq, "layer_num": 32}], model_name)
        engine.initialize_search_engine()
        if opts.debug_memory:
            from galvatron.core.search_engine.cost_model import MemoryCostModel
            for strat in ([1, 1, n, {}] if n == 1 else [1, 1, n, {"fsdp": 0}], [1, 1, n, {"cpt": 1}] if n == 1 else [1, 1, n, {"fsdp": 0, "cpt": 1}]):
                m = MemoryCostModel(strat, global_batch_size=8 * n, mbsz=1, min_tp=1, max_tp=1, model_args=engine.model_args_list[0],
                                    train_args=engine.train_args_list[0], parallel_args=engine.parallel_args_list[0],
                                    profile_model_args=engine.profile_model_args_list[0]).get_memory_cost()
                print("MEMDEBUG", strat, {k: (v if not isinstance(v, dict) else v) for k, v in m.items()})
        thr = engine.parallelism_optimization()
        files = glob.glob(os.path.join(out_dir, "*.json"))
        if not files:
            print("N=%d: the search engine found no feasible strategy" % n)
            continue
        cfg = json.load(open(files[0]))
        results[n] = (thr, cfg)
        dst = os.path.join(opts.out_root, "searched", "galvatron_config_llama3-8b_%dgpus.json" % n)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        json.dump(cfg, open(dst, "w"), indent=4)
        print("N=%d predicted throughput %.4f samples/s -> %s" % (n, thr, dst))
        print("   ", {k: (v if len(str(v)) < 40 else str(v)[:37] + "...") for k, v in cfg.items()})


if __name__ == "__main__":
    main()

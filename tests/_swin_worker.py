"""Worker for tests/test_swin.py and tests/test_gpu_swin.py: one rank of a job running the Swin family on the CPU oracle backend
(gloo) or on GPUs (HOST_TEST_BACKEND=cuda), checked against the single-process oracle (oracle/swin_ref.py, pinned to HF) on the
GLOBAL batch: loss within 5e-3 rel, every parameter's gradient within 3e-2 rel-L2, and the loss after one AdamW step within 5e-3 rel.
Also reported: the tokens each stage ran, the classifier's padding rows (zero), and optionally the gradient the embedding row
receives on its padding-token rows (exactly zero)."""
import json
import os
import re
import sys
import traceback

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

# 224 px, patch 4, window 7: stages of 3136, 784, 196 and 49 tokens; widths 16 / 32 / 64 / 128, head dim 16; 20 classes
TINY = dict(embed_dim=16, depths=[2, 2, 2, 2], num_heads=[1, 2, 4, 8], window_size=7, image_size=224, patch_size=4, num_channels=3,
            num_labels=20, layer_norm_eps=1e-5, drop_path_rate=0.0)
BLOCK = {"layernorm_before.weight": ("ln1", None), "layernorm_before.bias": ("ln1_b", None),
         "attention.query_key_value.weight": ("qkv", 0), "attention.query_key_value.bias": ("qkv_b", 0),
         "attention.dense.weight": ("dense", 1), "attention.dense.bias": ("dense_b", None),
         "layernorm_after.weight": ("ln2", None), "layernorm_after.bias": ("ln2_b", None),
         "mlp.dense_h_to_4h.weight": ("h_to_4h", 0), "mlp.dense_h_to_4h.bias": ("h_to_4h_b", 0),
         "mlp.dense_4h_to_h.weight": ("4h_to_h", 1), "mlp.dense_4h_to_h.bias": ("4h_to_h_b", None)}
MERGE = {"downsample.layernorm.weight": ("norm", None), "downsample.layernorm.bias": ("norm_b", None),
         "downsample.reduction.weight": ("reduction", 0)}
OTHER = {"embeddings.weight": ("patch", 0), "embeddings.bias": ("patch_b", 0), "embeddings.norm.weight": ("emb_ln", None),
         "embeddings.norm.bias": ("emb_ln_b", None), "LayerNorm.weight": ("norm", None), "LayerNorm.bias": ("norm_b", None),
         "classifier.weight": ("classifier", 0)}


def _unit_index(name):
    return int(name.rsplit("_", 1)[1])


def assemble(model, world, rank, tensor_of, config, pad_rows):
    """every rank's per-unit named tensors -> the oracle weight dict; classifier padding rows dropped (their max |.| to pad_rows)"""
    per_unit = []
    for u in model.model.units:
        per_unit.append({"name": u.name, "tp": list(u.tp_group.ranks) if u.tp_group is not None else [rank],
                         "slices": {re.sub(r"^(module\.)*(layer\.)?", "", k): v.detach().float().cpu().clone()
                                    for k, v in u.named_slices(tensor_of(u)).items()}})
    gathered = [None] * world
    dist.all_gather_object(gathered, per_unit)
    by_name = {}
    for r, units in enumerate(gathered):
        for rec in units:
            by_name.setdefault(rec["name"], {})[r] = rec
    out, blocks, merges = {}, {}, {}
    for name, recs in by_name.items():
        first = recs[sorted(recs)[0]]
        if name.startswith("swin_enc"):
            table, target = BLOCK, blocks.setdefault(_unit_index(name), {})
        elif name.startswith("swin_downsample"):
            table, target = MERGE, merges.setdefault(_unit_index(name), {})
        else:
            table, target = OTHER, out
        for pname in first["slices"]:
            key, dim = table[pname]
            parts = [recs[r]["slices"][pname] for r in first["tp"]]
            if key == "classifier":
                n = config.num_labels // len(parts)
                pad_rows.append(max(float(p[n:].abs().max()) if p.shape[0] > n else 0.0 for p in parts))
                parts = [p[:n] for p in parts]
            target[key] = parts[0] if dim is None or len(parts) == 1 else torch.cat(parts, dim=dim)
    bl, mg = [blocks[k] for k in sorted(blocks)], [merges[k] for k in sorted(merges)]
    out["stages"], i = [], 0
    for k, d in enumerate(config.depths):
        out["stages"].append(dict(blocks=bl[i:i + d], merge=mg[k] if k < len(mg) else None))
        i += d
    return out, sorted(blocks), sorted(merges)


def leaves(w):
    yield from (t for k, t in w.items() if k != "stages")
    for st in w["stages"]:
        for b in st["blocks"]:
            yield from b.values()
        if st["merge"] is not None:
            yield from st["merge"].values()


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    over = json.loads(os.environ["HOST_TEST_CONFIG"])
    spec = dict(TINY, **over.pop("_spec", {}))
    strategy = over.pop("_strategy", None)
    if strategy is not None:
        if isinstance(strategy, str):
            with open(os.path.join(ROOT, strategy)) as f:
                strategy = json.load(f)
        over["galvatron_config_path"] = dict(strategy, **over.pop("_strategy_over", {}))
    check_pad_grad = over.pop("_check_padded_token_grad", False)
    use_cuda = os.environ.get("HOST_TEST_BACKEND", "oracle") == "cuda"
    from oracle import swin_ref as ref
    import smoke_model as sm
    from _swin_backend import DropPath
    from hetu_galvatron_b200.core.runtime.backend import get_backend, reset_backend, set_backend
    from hetu_galvatron_b200.core.runtime.utils import get_optimizer_and_param_scheduler
    if use_cuda:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", torch.cuda.current_device()))
        os.environ.setdefault("HGB_ARENA_BYTES", str(256 << 20))
        be = get_backend()
        be.bg.set_tunable("timeout_ms", 30000)
        dev = be.device
    else:
        from _swin_backend import SwinOracleBackend
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.set_num_threads(1 if world >= 4 else 2)
        be = set_backend(SwinOracleBackend())
        dev = torch.device("cpu")
    args = sm.tiny_args(**over)
    from hetu_galvatron_b200.swin import config_from_meta, set_model_config, swin_model_hp
    config = set_model_config(config_from_meta(spec), args)
    model = swin_model_hp(config, args)
    opt, _ = get_optimizer_and_param_scheduler(model, args)
    # the oracle starts from the bf16 working weights (read_full_params); round the fp32 masters to those values so that both sides
    # take the AdamW step from the same weights (otherwise the masters' sub-bf16 bits alone move the post-step loss by ~0.5 % here)
    with torch.no_grad():
        for u in model.model.units:
            u.flat_param.data.copy_(u.flat_param.data.to(torch.bfloat16).float())
    pad_rows = []
    w, block_units, merge_units = assemble(model, world, rank, lambda u: u.read_full_params(), config, pad_rows)
    cfg = dict(embed_dim=config.embed_dim, depths=config.depths, heads=config.num_heads, window=config.window_size,
               patch=config.patch_size, image=config.image_size, eps=config.layer_norm_eps)
    gbs = args.global_train_batch_size
    dp_group = model.vtp_data_group
    dp_idx, dp = dp_group.rank_in_group(rank), dp_group.size
    g = torch.Generator().manual_seed(11)
    pixels = torch.randn(gbs, config.num_channels, config.image_size, config.image_size, generator=g)
    labels = torch.randint(0, config.num_labels, (gbs,), generator=g)
    lo, hi = dp_idx * gbs // dp, (dp_idx + 1) * gbs // dp
    captured = {}
    if check_pad_grad:
        def keep_grad(g):
            captured.setdefault("dy", g.detach().float().cpu().clone())

        def on_forward(mod, inputs, out):
            if out.requires_grad:
                out.register_hook(keep_grad)
        for m in model.modules():
            if type(m).__name__ == "SwinEmbeddings_":
                m.register_forward_hook(on_forward)
    drop_calls = [0]

    def drop():
        d = DropPath(config.drop_path_rate, args.seed, iteration=drop_calls[0])
        drop_calls[0] += 1
        return d if config.drop_path_rate > 0 else None

    loss = model.forward_backward([pixels[lo:hi].to(dev)], 0, None, loss_func=None, labels=labels[lo:hi].to(dev), attention_mask=None)
    if use_cuda:
        torch.cuda.synchronize()
        assert be.comm.error_flag() == 0
    from _family_worker import gather_grads
    for t in leaves(w):
        t.requires_grad_(True)
    _, ref_loss = ref.forward_loss(w, pixels, labels, cfg, dtype=torch.bfloat16, drop=drop())
    ref_loss.backward()
    grads = gather_grads(model, world)
    got, _, _ = assemble(model, world, rank, lambda u: grads[u.name], config, pad_rows)
    rel = lambda a, b: float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))  # noqa: E731
    dp_cls = model.hp_configs_whole["dp_sizes_whole"][-1] * model.hp_configs_whole["cp_sizes_whole"][-1]
    sizes = [None] * world
    dist.all_gather_object(sizes, {u.name: u.group.size for u in model.model.units})
    scale = {k: dp_cls / v for d in sizes for k, v in d.items()}
    unit_names = sorted(scale, key=_unit_index)
    name_of = {_unit_index(n): n for n in unit_names}
    other_unit = {"patch": unit_names[0], "patch_b": unit_names[0], "emb_ln": unit_names[0], "emb_ln_b": unit_names[0],
                  "norm": unit_names[-2], "norm_b": unit_names[-2], "classifier": unit_names[-1]}
    errs, leaf_scale = {}, {}
    for key, t in got.items():
        if key != "stages":
            errs[key] = rel(t, w[key].grad * scale[other_unit[key]])
            leaf_scale[id(w[key])] = scale[other_unit[key]]
    bi = mi = 0
    for k, (gs, ws) in enumerate(zip(got["stages"], w["stages"])):
        for gb, wb in zip(gs["blocks"], ws["blocks"]):
            s = scale[name_of[block_units[bi]]]
            for key in gb:
                errs["%s.%d" % (key, bi)] = rel(gb[key], wb[key].grad * s)
                leaf_scale[id(wb[key])] = s
            bi += 1
        if gs["merge"] is not None:
            s = scale[name_of[merge_units[mi]]]
            for key in gs["merge"]:
                errs["merge_%s.%d" % (key, mi)] = rel(gs["merge"][key], ws["merge"][key].grad * s)
                leaf_scale[id(ws["merge"][key])] = s
            mi += 1
    lt = torch.tensor([loss if loss is not None else 0.0, 1.0 if loss is not None else 0.0], dtype=torch.float64, device=dev)
    dist.all_reduce(lt)
    mean_loss = float(lt[0] / lt[1])
    report = dict(loss=mean_loss, ref_loss=float(ref_loss), max_grad_err=max(errs.values()), worst=max(errs, key=errs.get),
                  tokens_run=list(config.tokens_run), tokens=[s["tokens"] for s in config.stages])
    if "dy" in captured:
        dy, t0 = captured["dy"], config.stages[0]["tokens"]
        report["pad_token_grad_max"] = float(dy[t0:].abs().max()) if dy.shape[0] > t0 else None
        report["real_token_grad_max"] = float(dy[:t0].abs().max())
    assert abs(mean_loss - float(ref_loss)) <= 5e-3 * abs(float(ref_loss)), report
    assert report["max_grad_err"] < 3e-2, (report, {k: round(v, 4) for k, v in errs.items() if v > 1e-2})
    opt.step()
    opt.zero_grad()
    loss2 = model.forward_backward([pixels[lo:hi].to(dev)], 1, None, loss_func=None, labels=labels[lo:hi].to(dev), attention_mask=None)
    lt = torch.tensor([loss2 if loss2 is not None else 0.0, 1.0 if loss2 is not None else 0.0], dtype=torch.float64, device=dev)
    dist.all_reduce(lt)
    report["loss_step1"] = float(lt[0] / lt[1])
    lv = [t for t in leaves(w) if t.grad is not None]
    with torch.no_grad():
        for t in lv:
            t.grad.mul_(leaf_scale[id(t)])
    ref_opt = torch.optim.AdamW(lv, lr=args.lr, weight_decay=args.adam_weight_decay,
                                betas=(getattr(args, "adam_beta1", 0.9), getattr(args, "adam_beta2", 0.999)), eps=getattr(args, "adam_eps", 1e-8))
    ref_opt.step()
    with torch.no_grad():
        _, ref_loss1 = ref.forward_loss(w, pixels, labels, cfg, dtype=torch.bfloat16, drop=drop())
    report["ref_loss_step1"] = float(ref_loss1)
    assemble(model, world, rank, lambda u: u.read_full_params(), config, pad_rows)
    report["classifier_pad_rows_max"] = max(pad_rows)
    assert abs(report["loss_step1"] - report["ref_loss_step1"]) <= 5e-3 * abs(report["ref_loss_step1"]), report
    assert report["classifier_pad_rows_max"] == 0.0, report
    if rank == 0:
        print("HOST_TEST_REPORT " + json.dumps(report), flush=True)
    dist.barrier()
    if use_cuda:
        reset_backend()
    dist.destroy_process_group()
    return report


if __name__ == "__main__":
    try:
        main()
    except Exception:
        traceback.print_exc()
        sys.exit(1)

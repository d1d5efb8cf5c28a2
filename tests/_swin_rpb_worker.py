"""Worker for tests/test_swin_rel_bias.py and tests/test_gpu_swin_rel_bias.py: one rank of a job running the Swin family with the
relative-position bias on the CPU restatement (gloo) or on GPUs (HOST_TEST_BACKEND=cuda), checked against the oracle of
tests/_swin_rpb.py on the GLOBAL batch as tests/_swin_worker.py checks the plain model: loss within 5e-3 rel, every parameter's
gradient (the tables included) within 3e-2 rel-L2, and the loss after one AdamW step within 5e-3 rel.  Also reported: the sum of
every block's initial table (the same under every tensor-parallel layout)."""
import json
import os
import sys
import traceback

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import _swin_worker as sw  # noqa: E402

# the block's table, split by heads (columns) over the tensor-parallel group (this process's copy of the name table)
sw.BLOCK["attention.relative_position_bias_table"] = ("rpb", 1)


def _global_loss(loss, dev):
    lt = torch.tensor([loss if loss is not None else 0.0, 1.0 if loss is not None else 0.0], dtype=torch.float64, device=dev)
    dist.all_reduce(lt)
    return float(lt[0] / lt[1])


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    over = json.loads(os.environ["HOST_TEST_CONFIG"])
    spec = dict(sw.TINY, relative_position_bias=True, **over.pop("_spec", {}))
    strategy = over.pop("_strategy", None)
    if strategy is not None:
        if isinstance(strategy, str):
            with open(os.path.join(ROOT, strategy)) as f:
                strategy = json.load(f)
        over["galvatron_config_path"] = dict(strategy, **over.pop("_strategy_over", {}))
    use_cuda = os.environ.get("HOST_TEST_BACKEND", "oracle") == "cuda"
    import _swin_rpb as rpb
    import smoke_model as sm
    from _family_worker import gather_grads
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
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.set_num_threads(1 if world >= 4 else 2)
        be = set_backend(rpb.SwinRelBiasOracleBackend())
        dev = torch.device("cpu")
    args = sm.tiny_args(**over)
    from hetu_galvatron_b200.swin import config_from_meta, set_model_config, swin_model_hp
    config = set_model_config(config_from_meta(spec), args)
    model = swin_model_hp(config, args)
    opt, _ = get_optimizer_and_param_scheduler(model, args)
    with torch.no_grad():           # both sides start from the bf16 working weights (tests/_swin_worker.py)
        for u in model.model.units:
            u.flat_param.data.copy_(u.flat_param.data.to(torch.bfloat16).float())
    pad_rows = []
    w, block_units, merge_units = sw.assemble(model, world, rank, lambda u: u.read_full_params(), config, pad_rows)
    tables = [b["rpb"] for st in w["stages"] for b in st["blocks"]]
    assert len(tables) == config.num_hidden_layers and all(float(t.abs().max()) > 0 for t in tables)
    cfg = dict(embed_dim=config.embed_dim, depths=config.depths, heads=config.num_heads, window=config.window_size,
               patch=config.patch_size, image=config.image_size, eps=config.layer_norm_eps)
    gbs = args.global_train_batch_size
    dp_group = model.vtp_data_group
    dp_idx, dp = dp_group.rank_in_group(rank), dp_group.size
    g = torch.Generator().manual_seed(11)
    pixels = torch.randn(gbs, config.num_channels, config.image_size, config.image_size, generator=g)
    labels = torch.randint(0, config.num_labels, (gbs,), generator=g)
    lo, hi = dp_idx * gbs // dp, (dp_idx + 1) * gbs // dp

    loss = model.forward_backward([pixels[lo:hi].to(dev)], 0, None, loss_func=None, labels=labels[lo:hi].to(dev), attention_mask=None)
    if use_cuda:
        torch.cuda.synchronize()
        assert be.comm.error_flag() == 0
    for t in sw.leaves(w):
        t.requires_grad_(True)
    _, ref_loss = rpb.forward_loss(w, pixels, labels, cfg, dtype=torch.bfloat16)
    ref_loss.backward()
    grads = gather_grads(model, world)
    got, _, _ = sw.assemble(model, world, rank, lambda u: grads[u.name], config, pad_rows)
    rel = lambda a, b: float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))  # noqa: E731
    dp_cls = model.hp_configs_whole["dp_sizes_whole"][-1] * model.hp_configs_whole["cp_sizes_whole"][-1]
    sizes = [None] * world
    dist.all_gather_object(sizes, {u.name: u.group.size for u in model.model.units})
    scale = {k: dp_cls / v for d in sizes for k, v in d.items()}
    unit_names = sorted(scale, key=sw._unit_index)
    name_of = {sw._unit_index(n): n for n in unit_names}
    other_unit = {"patch": unit_names[0], "patch_b": unit_names[0], "emb_ln": unit_names[0], "emb_ln_b": unit_names[0],
                  "norm": unit_names[-2], "norm_b": unit_names[-2], "classifier": unit_names[-1]}
    errs, leaf_scale = {}, {}
    for key, t in got.items():
        if key != "stages":
            errs[key] = rel(t, w[key].grad * scale[other_unit[key]])
            leaf_scale[id(w[key])] = scale[other_unit[key]]
    bi = mi = 0
    for gs, ws in zip(got["stages"], w["stages"]):
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
    mean_loss = _global_loss(loss, dev)
    report = dict(loss=mean_loss, ref_loss=float(ref_loss), max_grad_err=max(errs.values()), worst=max(errs, key=errs.get),
                  table_grad_err=max(v for k, v in errs.items() if k.startswith("rpb.")), tokens_run=list(config.tokens_run),
                  table_sums=[float(t.detach().double().sum()) for t in tables],
                  table_grad_max=min(float(b["rpb"].abs().max()) for st in got["stages"] for b in st["blocks"]))
    assert abs(mean_loss - float(ref_loss)) <= 5e-3 * abs(float(ref_loss)), report
    assert report["max_grad_err"] < 3e-2, (report, {k: round(v, 4) for k, v in errs.items() if v > 1e-2})
    opt.step()
    opt.zero_grad()
    loss2 = model.forward_backward([pixels[lo:hi].to(dev)], 1, None, loss_func=None, labels=labels[lo:hi].to(dev), attention_mask=None)
    report["loss_step1"] = _global_loss(loss2, dev)
    lv = [t for t in sw.leaves(w) if t.grad is not None]
    with torch.no_grad():
        for t in lv:
            t.grad.mul_(leaf_scale[id(t)])
    ref_opt = torch.optim.AdamW(lv, lr=args.lr, weight_decay=args.adam_weight_decay,
                                betas=(getattr(args, "adam_beta1", 0.9), getattr(args, "adam_beta2", 0.999)), eps=getattr(args, "adam_eps", 1e-8))
    ref_opt.step()
    with torch.no_grad():
        _, ref_loss1 = rpb.forward_loss(w, pixels, labels, cfg, dtype=torch.bfloat16)
    report["ref_loss_step1"] = float(ref_loss1)
    assert abs(report["loss_step1"] - report["ref_loss_step1"]) <= 5e-3 * abs(report["ref_loss_step1"]), report
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

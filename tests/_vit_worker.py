"""Worker for tests/test_vit.py and tests/test_gpu_vit.py: one rank of a job running the ViT family of the product on the CPU oracle
backend (gloo) or on GPUs (HOST_TEST_BACKEND=cuda), checked against the single-process oracle (oracle/vit_ref.py, pinned to HF) on
the GLOBAL batch: loss within 5e-3 rel, every parameter's gradient within 3e-2 rel-L2, and the loss after one AdamW step within
5e-3 rel of the oracle's after the same step.  Also checked: the classifier's padding rows (each rank's class slice padded to a
multiple of 8) stay exactly zero in weights and gradients, and the reported token count the layers ran (``s_run``)."""
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

# image 32, patch 8, 3 channels: 16 patches + CLS = 17 tokens; 20 classes = 10 per rank at vtp 2 (padded to 16)
TINY = dict(hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128, image_size=32, patch_size=8,
            num_channels=3, num_labels=20, layer_norm_eps=1e-5)
OTHER = {"embeddings.weight": ("patch", 0), "embeddings.bias": ("patch_b", 0), "embeddings.cls_token": ("cls", None),
         "embeddings.position_embeddings": ("pos", None), "LayerNorm.weight": ("norm", None), "LayerNorm.bias": ("norm_b", None),
         "pooler.weight": ("pooler", None), "pooler.bias": ("pooler_b", None), "classifier.weight": ("classifier", 0)}
UNIT_OF_KEY = {"patch": "embed", "patch_b": "embed", "cls": "embed", "pos": "embed", "norm": "prenorm", "norm_b": "prenorm",
               "pooler": "cls", "pooler_b": "cls", "classifier": "cls"}


def assemble(model, world, rank, tensor_of, num_labels, pad_rows):
    """every rank's per-unit named tensors -> the un-parallelised oracle weight dict; the classifier's padding rows are dropped and
    their largest magnitude is added to ``pad_rows``"""
    from _family_worker import LAYER
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
    out, layers = {}, {}
    for name, recs in by_name.items():
        first = recs[sorted(recs)[0]]
        table = LAYER if re.match(r"vit_enc_\d+", name) else OTHER
        target = layers.setdefault(name, {}) if table is LAYER else out
        for pname in first["slices"]:
            key, dim = table[pname]
            parts = [recs[r]["slices"][pname] for r in first["tp"]]
            if key == "classifier":
                n = num_labels // len(parts)
                pad_rows.append(max(float(p[n:].abs().max()) if p.shape[0] > n else 0.0 for p in parts))
                parts = [p[:n] for p in parts]
            target[key] = parts[0] if dim is None or len(parts) == 1 else torch.cat(parts, dim=dim)
    out["layers"] = [layers[k] for k in sorted(layers, key=lambda s: int(s.rsplit("_", 1)[1]))]
    return out


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    over = json.loads(os.environ["HOST_TEST_CONFIG"])
    spec = dict(TINY, **over.pop("_spec", {}))
    tol = over.pop("_tol", 3e-2)
    strategy = over.pop("_strategy", None)
    if strategy is not None:                   # a strategy JSON in the reference's format (a file under tests/golden, or inline)
        if isinstance(strategy, str):
            with open(os.path.join(ROOT, strategy)) as f:
                strategy = json.load(f)
        strategy = dict(strategy, **over.pop("_strategy_over", {}))
        over["galvatron_config_path"] = strategy
    check_pad_grad = over.pop("_check_padded_token_grad", False)
    use_cuda = os.environ.get("HOST_TEST_BACKEND", "oracle") == "cuda"
    hidden_p = float(spec.get("hidden_dropout_prob", 0.0))
    from oracle import vit_ref as ref
    import smoke_model as sm
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
        from _vit_backend import ViTOracleBackend
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.set_num_threads(1 if world >= 4 else 2)
        be = set_backend(ViTOracleBackend())
        dev = torch.device("cpu")
    args = sm.tiny_args(**over)
    from hetu_galvatron_b200.vit_hf import config_from_meta, set_model_config, vit_model_hp
    config = set_model_config(config_from_meta(spec), args)
    model = vit_model_hp(config, args)
    opt, _ = get_optimizer_and_param_scheduler(model, args)
    pad_rows = []
    w = assemble(model, world, rank, lambda u: u.read_full_params(), config.num_labels, pad_rows)
    cfg = dict(hidden=config.hidden_size, ffn=config.intermediate_size, n_heads=config.num_attention_heads,
               head_dim=config.hidden_size // config.num_attention_heads, eps=args.norm_epsilon, gelu_tanh=True, patch=config.patch_size)
    gbs = args.global_train_batch_size
    dp_group = model.vtp_data_group
    dp_idx, dp = dp_group.rank_in_group(rank), dp_group.size
    g = torch.Generator().manual_seed(11)
    pixels = torch.randn(gbs, config.num_channels, config.image_size, config.image_size, generator=g)
    labels = torch.randint(0, config.num_labels, (gbs,), generator=g)
    lo, hi = dp_idx * gbs // dp, (dp_idx + 1) * gbs // dp
    captured = {}
    if check_pad_grad:     # the gradient the embedding row receives, to show the padding tokens' rows are exactly zero
        emb = [m for m in model.modules() if type(m).__name__ == "ViTEmbeddings_"]
        def keep_grad(g):
            captured.setdefault("dy", g.detach().float().cpu().clone())

        def on_forward(mod, inputs, out):
            if out.requires_grad:
                out.register_hook(keep_grad)

        for m in emb:
            m.register_forward_hook(on_forward)
    drop_calls = [0]

    def drop():
        import _dropout_ref as dref
        d = dref.Drop(hidden_p, 0.0, args.seed, iteration=drop_calls[0])
        drop_calls[0] += 1
        return d if hidden_p > 0 else None

    loss = model.forward_backward([pixels[lo:hi].to(dev)], 0, None, loss_func=None, labels=labels[lo:hi].to(dev), attention_mask=None)
    if use_cuda:
        torch.cuda.synchronize()
        assert be.comm.error_flag() == 0
    from _family_worker import gather_grads, leaves_of
    for t in leaves_of(w):
        t.requires_grad_(True)
    _, ref_loss = ref.forward_loss(w, pixels, labels, cfg, dtype=torch.bfloat16, drop=drop())
    ref_loss.backward()
    grads = gather_grads(model, world)
    got = assemble(model, world, rank, lambda u: grads[u.name], config.num_labels, pad_rows)
    rel = lambda a, b: float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))  # noqa: E731
    # a unit's gradient is averaged over ITS sharded-data-parallel group (tests/_family_worker.py)
    dp_cls = model.hp_configs_whole["dp_sizes_whole"][-1] * model.hp_configs_whole["cp_sizes_whole"][-1]
    sizes = [None] * world
    dist.all_gather_object(sizes, {u.name: u.group.size for u in model.model.units})
    scale = {k: dp_cls / v for d in sizes for k, v in d.items()}
    names = [None] * world
    dist.all_gather_object(names, {re.sub(r"_\d+$", "", u.name): u.name for u in model.model.units if not u.name.startswith("vit_enc")})
    unit_of = {k: v for d in names for k, v in d.items()}
    errs = {key: rel(t, w[key].grad * scale[unit_of[UNIT_OF_KEY[key]]]) for key, t in got.items() if key != "layers"}
    layer_units = sorted([n for n in scale if re.match(r"vit_enc_\d+", n)], key=lambda s: int(s.rsplit("_", 1)[1]))
    for i, (gl, wl) in enumerate(zip(got["layers"], w["layers"])):
        for k in gl:
            errs["%s%d" % (k, i)] = rel(gl[k], wl[k].grad * scale[layer_units[i]])
    lt = torch.tensor([loss if loss is not None else 0.0, 1.0 if loss is not None else 0.0], dtype=torch.float64, device=dev)
    dist.all_reduce(lt)
    mean_loss = float(lt[0] / lt[1])
    report = dict(loss=mean_loss, ref_loss=float(ref_loss), max_grad_err=max(errs.values()), worst=max(errs, key=errs.get),
                  s_run=config.seq_run, seq=config.seq_length)
    if "dy" in captured:
        dy = captured["dy"]
        report["pad_token_grad_max"] = float(dy[config.seq_length:].abs().max()) if dy.shape[0] > config.seq_length else None
        report["real_token_grad_max"] = float(dy[:config.seq_length].abs().max())
    assert abs(mean_loss - float(ref_loss)) <= 5e-3 * abs(float(ref_loss)), report
    assert report["max_grad_err"] < tol, (report, {k: round(v, 4) for k, v in errs.items() if v > tol / 3})
    opt.step()
    opt.zero_grad()
    loss2 = model.forward_backward([pixels[lo:hi].to(dev)], 1, None, loss_func=None, labels=labels[lo:hi].to(dev), attention_mask=None)
    lt = torch.tensor([loss2 if loss2 is not None else 0.0, 1.0 if loss2 is not None else 0.0], dtype=torch.float64, device=dev)
    dist.all_reduce(lt)
    report["loss_step1"] = float(lt[0] / lt[1])
    leaf_scale = {id(t): scale[unit_of[UNIT_OF_KEY[key]]] for key, t in w.items() if key != "layers"}
    for i, wl in enumerate(w["layers"]):
        for t in wl.values():
            leaf_scale[id(t)] = scale[layer_units[i]]
    leaves = [t for t in leaves_of(w) if t.grad is not None]
    with torch.no_grad():
        for t in leaves:
            t.grad.mul_(leaf_scale[id(t)])
    ref_opt = torch.optim.AdamW(leaves, lr=args.lr, weight_decay=args.adam_weight_decay,
                                betas=(getattr(args, "adam_beta1", 0.9), getattr(args, "adam_beta2", 0.999)), eps=getattr(args, "adam_eps", 1e-8))
    ref_opt.step()
    with torch.no_grad():
        _, ref_loss1 = ref.forward_loss(w, pixels, labels, cfg, dtype=torch.bfloat16, drop=drop())
    report["ref_loss_step1"] = float(ref_loss1)
    assemble(model, world, rank, lambda u: u.read_full_params(), config.num_labels, pad_rows)       # padding rows after the step
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

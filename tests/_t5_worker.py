"""Worker for tests/test_t5.py and tests/test_gpu_t5.py: one rank of a job running the T5 family on the CPU oracle backend (gloo) or
on GPUs (HOST_TEST_BACKEND=cuda), checked against the single-process oracle (oracle/t5_ref.py, pinned to HF) on the GLOBAL batch:
loss within 5e-3 rel, every parameter's gradient within 3e-2 rel-L2, and the loss after one AdamW step within 5e-3 rel.

The product's loss is the mean over the data-parallel ranks of the mean over each rank's micro-batches (torch.chunk of its local
batch, the last one possibly smaller) of each micro-batch's loss: the token mean, or with ``_masked`` the reference's masked mean
sum(loss * mask) / sum(mask).  The oracle weighs every token of the global batch accordingly."""
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

# inner width d_kv x heads = 128 against d_model 64; encoder 32 tokens, decoder 16
TINY = dict(d_model=64, d_kv=32, d_ff=128, num_heads=4, num_layers=2, num_decoder_layers=2, vocab_size=256, n_positions=32,
            n_decoder_positions=16)
LAYER = {"attention.LayerNorm.weight": ("ln1", None), "attention.attention.query_key_value.weight": ("qkv", 0),
         "attention.attention.query_key_value.bias": ("qkv_b", 0), "attention.attention.dense.weight": ("dense", 1),
         "attention.attention.dense.bias": ("dense_b", None), "cross_attention.LayerNorm.weight": ("lnx", None),
         "cross_attention.attention.query.weight": ("q", 0), "cross_attention.attention.query.bias": ("q_b", 0),
         "cross_attention.attention.key_value.weight": ("kv", 0), "cross_attention.attention.key_value.bias": ("kv_b", 0),
         "cross_attention.attention.dense.weight": ("xdense", 1), "cross_attention.attention.dense.bias": ("xdense_b", None),
         "mlp.LayerNorm.weight": ("ln2", None), "mlp.mlp.dense_h_to_4h.weight": ("h_to_4h", 0),
         "mlp.mlp.dense_h_to_4h.bias": ("h_to_4h_b", 0), "mlp.mlp.dense_4h_to_h.weight": ("4h_to_h", 1),
         "mlp.mlp.dense_4h_to_h.bias": ("4h_to_h_b", None)}
OTHER = {"embed_1": {"embeddings.weight": ("shared", 0)}, "embed_2": {"embeddings.weight": ("dec_shared", 0)},
         "pre_norm_1": {"LayerNorm.weight": ("enc_norm", None)}, "pre_norm_2": {"LayerNorm.weight": ("dec_norm", None)},
         "cls": {"lm_head.weight": ("lm_head", 0)}}


def _kind(name):
    return name.rsplit("_", 1)[0]


def assemble(model, world, rank, tensor_of):
    """every rank's per-unit named tensors -> the oracle weight dict, and {oracle leaf path: unit name}"""
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
    out, enc, dec, owner = {}, {}, {}, {}
    for name, recs in by_name.items():
        first, kind = recs[sorted(recs)[0]], _kind(name)
        idx = int(name.rsplit("_", 1)[1])
        if kind in ("t5_enc", "t5_dec"):
            target, table = (enc if kind == "t5_enc" else dec).setdefault(idx, {}), LAYER
        else:
            target, table = out, OTHER[kind]
        for pname in first["slices"]:
            key, dim = table[pname]
            parts = [recs[r]["slices"][pname] for r in first["tp"]]
            target[key] = parts[0] if dim is None or len(parts) == 1 else torch.cat(parts, dim=dim)
            owner[(kind, idx, key)] = name
    out["enc"] = [enc[k] for k in sorted(enc)]
    out["dec"] = [dec[k] for k in sorted(dec)]
    # oracle leaf path (stack, layer, key) -> the unit that holds it
    pos = {("t5_enc", k): ("enc", i) for i, k in enumerate(sorted(enc))}
    pos.update({("t5_dec", k): ("dec", i) for i, k in enumerate(sorted(dec))})
    unit_of = {pos.get((kind, idx), ("", -1)) + (key,): name for (kind, idx, key), name in owner.items()}
    return out, unit_of


def leaves(w):
    for k, t in w.items():
        if k not in ("enc", "dec"):
            yield ("", -1, k), t
    for stack in ("enc", "dec"):
        for i, p in enumerate(w[stack]):
            for k, t in p.items():
                yield (stack, i, k), t


def token_weights(gbs, s_dec, dp, chunks, loss_mask):
    """[gbs, s_dec] weights of the product's loss: 1 / dp per rank, 1 / micro-batches per micro-batch, and the micro-batch's token
    mean (or masked mean)"""
    wts = torch.zeros(gbs, s_dec, dtype=torch.float64)
    per = gbs // dp
    for r in range(dp):
        rows = torch.arange(r * per, (r + 1) * per)
        mbs = rows.chunk(chunks)
        for mb in mbs:
            m = loss_mask[mb].double() if loss_mask is not None else torch.ones(len(mb), s_dec, dtype=torch.float64)
            wts[mb] = m / m.sum() / len(mbs) / dp
    return wts


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
    masked = over.pop("_masked", False)
    use_cuda = os.environ.get("HOST_TEST_BACKEND", "oracle") == "cuda"
    from oracle import t5_ref as ref
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
        from _t5_backend import T5OracleBackend
        dist.init_process_group("gloo", rank=rank, world_size=world)
        torch.set_num_threads(1 if world >= 4 else 2)
        be = set_backend(T5OracleBackend())
        dev = torch.device("cpu")
    args = sm.tiny_args(**over)
    from hetu_galvatron_b200.t5 import config_from_meta, set_model_config, t5_model_hp
    config = set_model_config(config_from_meta(spec), args)
    model = t5_model_hp(config, args)
    opt, _ = get_optimizer_and_param_scheduler(model, args)
    # both sides take the AdamW step from the bf16 working weights
    with torch.no_grad():
        for u in model.model.units:
            u.flat_param.data.copy_(u.flat_param.data.to(torch.bfloat16).float())
    w, unit_of = assemble(model, world, rank, lambda u: u.read_full_params())
    cfg = dict(heads=config.num_attention_heads, eps=config.layer_norm_epsilon)
    gbs, s_enc, s_dec, V = args.global_train_batch_size, config.n_positions, config.n_decoder_positions, config.vocab_size
    dp_group = model.vtp_data_group
    dp_idx, dp = dp_group.rank_in_group(rank), dp_group.size
    g = torch.Generator().manual_seed(11)
    enc = torch.randint(0, V, (gbs, s_enc), generator=g)
    dec = torch.randint(0, V, (gbs, s_dec), generator=g)
    labels = torch.randint(0, V, (gbs, s_dec), generator=g)
    loss_mask = None
    if masked:
        # padding at the end of every sample's decoder sequence: label -1, loss mask 0 (the reference's T5 batches)
        n_real = torch.randint(s_dec // 2, s_dec + 1, (gbs,), generator=g)
        loss_mask = (torch.arange(s_dec)[None, :] < n_real[:, None]).float()
        labels = labels.masked_fill(loss_mask == 0, -1)
    lo, hi = dp_idx * gbs // dp, (dp_idx + 1) * gbs // dp
    chunks = args.chunks
    loss_func = None
    if masked:
        micro = [m.to(dev) for m in loss_mask[lo:hi].chunk(chunks)]

        def loss_func(_labels, outputs):            # the reference's loss_func: masked mean of the per-token losses
            m = micro.pop(0)
            loss = (outputs[0].float().reshape(-1) * m.reshape(-1)).sum() / m.sum()
            return loss, loss.clone().detach()

    def step(it):
        if masked:
            micro[:] = [m.to(dev) for m in loss_mask[lo:hi].chunk(chunks)]
        return model.forward_backward([enc[lo:hi].to(dev)], it, None, loss_func=loss_func, dec_tokens=dec[lo:hi].to(dev),
                                      dec_labels=labels[lo:hi].to(dev))

    loss = step(0)
    if use_cuda:
        torch.cuda.synchronize()
        assert be.comm.error_flag() == 0
    from _family_worker import gather_grads
    wts = token_weights(gbs, s_dec, dp, chunks, loss_mask)
    for _, t in leaves(w):
        t.requires_grad_(True)
    tok, _ = ref.forward_loss(w, enc, dec, labels, cfg, dtype=torch.bfloat16)
    ref_loss = (tok.double() * wts).sum()
    ref_loss.backward()
    grads = gather_grads(model, world)
    got, _ = assemble(model, world, rank, lambda u: grads[u.name])
    rel = lambda a, b: float((a.float() - b.float()).norm() / (b.float().norm() + 1e-12))  # noqa: E731
    dp_cls = model.hp_configs_whole["dp_sizes_whole"][-1] * model.hp_configs_whole["cp_sizes_whole"][-1]
    sizes = [None] * world
    dist.all_gather_object(sizes, {u.name: u.group.size for u in model.model.units})
    scale = {k: dp_cls / v for d in sizes for k, v in d.items()}
    got_leaves = dict(leaves(got))
    errs, leaf_scale = {}, {}
    for path, t in leaves(w):
        stack, i, key = path
        s = scale[unit_of[path]]
        errs["%s%s.%s" % (stack, "" if i < 0 else i, key)] = rel(got_leaves[path], t.grad * s)
        leaf_scale[id(t)] = s
    lt = torch.tensor([loss if loss is not None else 0.0, 1.0 if loss is not None else 0.0], dtype=torch.float64, device=dev)
    dist.all_reduce(lt)
    mean_loss = float(lt[0] / lt[1])
    report = dict(loss=mean_loss, ref_loss=float(ref_loss), max_grad_err=max(errs.values()), worst=max(errs, key=errs.get),
                  n_leaves=len(errs))
    assert abs(mean_loss - float(ref_loss)) <= 5e-3 * abs(float(ref_loss)), report
    assert report["max_grad_err"] < 3e-2, (report, {k: round(v, 4) for k, v in errs.items() if v > 1e-2})
    opt.step()
    opt.zero_grad()
    loss2 = step(1)
    lt = torch.tensor([loss2 if loss2 is not None else 0.0, 1.0 if loss2 is not None else 0.0], dtype=torch.float64, device=dev)
    dist.all_reduce(lt)
    report["loss_step1"] = float(lt[0] / lt[1])
    lv = [t for _, t in leaves(w) if t.grad is not None]
    with torch.no_grad():
        for t in lv:
            t.grad.mul_(leaf_scale[id(t)])
    ref_opt = torch.optim.AdamW(lv, lr=args.lr, weight_decay=args.adam_weight_decay,
                                betas=(getattr(args, "adam_beta1", 0.9), getattr(args, "adam_beta2", 0.999)), eps=getattr(args, "adam_eps", 1e-8))
    ref_opt.step()
    with torch.no_grad():
        tok1, _ = ref.forward_loss(w, enc, dec, labels, cfg, dtype=torch.bfloat16)
    report["ref_loss_step1"] = float((tok1.double() * wts).sum())
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

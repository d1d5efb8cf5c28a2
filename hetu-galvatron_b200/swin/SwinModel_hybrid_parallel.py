"""Entry points of the Swin family (``galvatron/models/swin/SwinModel_hybrid_parallel.py``).

Token padding rule, decided once per stage before any layer exists: stage k's GEMMs see T_k x micro-batch rows, which must be a
multiple of 8.  With T_k real tokens (3136, 784, 196, 49 for Swin-H/224)
    tokens_run_k = T_k        when T_k x m is a multiple of 8 for every micro-batch size m any row of the strategy runs,
    tokens_run_k = ceil8(T_k) otherwise (196 -> 200, 49 -> 56).
The extra tokens are zero rows written by the embedding / patch-merge kernels at the end of each sample's token list.  No kernel
reads them as input -- the window relayout, the patch merge and the mean-pool address real tokens only, and a row-wise LayerNorm or
MLP keeps them apart from real rows -- so real rows are those of the unpadded model and the gradient reaching a padding row is
exactly zero at every row."""
import types

from ..core.runtime import world as _world
from ..core.runtime.hybrid_parallel_config import get_chunks, get_hybrid_parallel_configs_api
from ..core.runtime.hybrid_parallel_model import construct_hybrid_parallel_model_api
from ..llama_hf.LlamaModel_hybrid_parallel import estimate_arena_bytes as _estimate_arena_bytes
from ..vit_hf.ViTModel_hybrid_parallel import _microbatch_sizes
from .meta_configs import config_from_meta, set_model_config
from .SwinModel_sequential import SwinCls_, SwinDownsample_, SwinEmbeddings_, SwinModelInfo, SwinPreNorm_, construct_sequential_model
from .SwinModel_tensor_parallel import SwinBlock_tp, SwinSkeleton, ceil8, construct_tensor_parallel_model


def get_hybrid_parallel_configs(model_config, training_args):
    return get_hybrid_parallel_configs_api(model_config, training_args, SwinModelInfo)


def construct_hybrid_parallel_model(model, model_config, training_args, hybrid_parallel_configs):
    return construct_hybrid_parallel_model_api(
        model, model_config, training_args, hybrid_parallel_configs, SwinModelInfo, construct_sequential_model,
        construct_tensor_parallel_model, wrap_block_name=[SwinBlock_tp], wrap_checkpoint_block_name=[SwinBlock_tp],
        wrap_other_block_name=[SwinEmbeddings_, SwinDownsample_, SwinPreNorm_, SwinCls_], tied_wte_attr_names=None,
        layernorm_name=["layernorm", "layernorm_before", "layernorm_after", "LayerNorm", "norm"],
        all_block_name=[SwinEmbeddings_, SwinBlock_tp, SwinDownsample_, SwinPreNorm_, SwinCls_])


def get_swin_config(args, overwrite_args=True):
    return set_model_config(config_from_meta(args.model_size), args, overwrite_args)


def token_rows(config, args, hp_configs):
    """The tokens each stage's rows run (module docstring): T_k, or T_k rounded up to a multiple of 8 when some row's micro-batch
    needs it."""
    world, pp, chunks = _world.get_world_size(), hp_configs["pp_deg"], max(1, get_chunks(args))
    sizes = set()
    for degree in set(hp_configs["tp_sizes_enc"]) | {hp_configs["vocab_tp"]}:
        sizes.update(_microbatch_sizes(args.global_train_batch_size // max(1, world // pp // degree), chunks))
    return [s["tokens"] if all(s["tokens"] * m % 8 == 0 for m in sizes) else ceil8(s["tokens"]) for s in config.stages]


def _refuse(config, args, hp_configs=None):
    """What the reference forbids or has no path for, refused with an error instead of changing the caller's arguments."""
    why = []
    if args.sequence_parallel:
        why.append("Megatron sequence parallelism (sequence_parallel)")
    if args.use_ulysses:
        why.append("Ulysses sequence parallelism (use_ulysses)")
    if getattr(args, "global_cp_deg", 1) > 1 or getattr(args, "vocab_cp", 1) > 1:
        why.append("context parallelism")
    if hp_configs is not None:
        if any(c > 1 for c in hp_configs["cp_sizes_enc"]) or hp_configs.get("vocab_cp", 1) > 1:
            why.append("context parallelism")
        if any(hp_configs["use_sp"]) or hp_configs.get("vocab_sp", 0):
            why.append("Ulysses sequence parallelism (use_sp / vsp)")
    if getattr(args, "load", None) not in (None, "None") or getattr(args, "save", None) not in (None, "None"):
        why.append("checkpoint load / save (no Swin checkpoint format)")
    if config.hidden_dropout_prob > 0 or config.attention_probs_dropout_prob > 0:
        why.append("hidden / attention dropout (0 in every shipped Swin config)")
    if config.use_absolute_embeddings:
        why.append("absolute position embeddings (use_absolute_embeddings)")
    if hp_configs is not None and config.drop_path_rate > 0:
        # the drop-path masks are drawn at the global samples the embedding / head rows' data-parallel split assigns; a block whose
        # tensor-parallel degree or grouping differs from theirs holds another slice of the batch after the relocation
        vtp = hp_configs["vocab_tp"]
        if any(t != vtp or (t > 1 and c != 1) for t, c in zip(hp_configs["tp_sizes_enc"], hp_configs["tp_consecutive_flags"])):
            why.append("drop path (drop_path_rate > 0) in blocks whose tensor-parallel degree or grouping differs from the vocabulary "
                       "rows' (a relocation that re-splits the batch)")
    for k, s in enumerate(config.stages):
        if s["res"] % s["window"] or (k + 1 < len(config.stages) and s["res"] % 2):
            why.append("a %dx%d stage-%d grid that does not split into %dx%d windows and 2x2 merges" % (s["res"], s["res"], k,
                                                                                                        s["window"], s["window"]))
    if why:
        raise NotImplementedError("the Swin family does not support %s" % ", ".join(sorted(set(why))))


def estimate_arena_bytes(config, args, hp_configs):
    """The Llama estimate summed over the four stages, each with its own width, tokens and layers; the non-layer rows counted in
    rows of the stage's width (the estimate's 'vocabulary'): the patch projection + norm at stage 0, the downsample's LayerNorm(4C)
    + 4C x 2C reduction after every stage but the last, the padded classifier + final norm at the last."""
    total, n = 0, len(config.stages)
    layer_of = [k for k, s in enumerate(config.stages) for _ in range(s["depth"])]
    per_layer = ("tp_sizes_enc", "tp_consecutive_flags", "dp_types_enc", "pp_ranks_enc", "checkpoint_flags_enc", "cp_sizes_enc",
                 "use_sp")
    for k, (s, t_run) in enumerate(zip(config.stages, config.tokens_run)):
        c = s["width"]
        rows = 8 * c + 8 if k + 1 < n else 0
        if k == 0:
            rows = max(rows, config.patch_size * config.patch_size * config.num_channels + 2)
        if k == n - 1:
            rows = max(rows, args.padded_vocab_size + 2)
        hp_k = dict(hp_configs)
        for key in per_layer:
            if key in hp_configs and hp_configs[key] is not None:
                hp_k[key] = [v for v, lk in zip(hp_configs[key], layer_of) if lk == k]
        proxy_config = types.SimpleNamespace(hidden_size=c, intermediate_size=4 * c, num_attention_heads=s["heads"],
                                             num_key_value_heads=s["heads"], max_position_embeddings=t_run)
        proxy_args = types.SimpleNamespace(**dict(vars(args), padded_vocab_size=rows))
        total += _estimate_arena_bytes(proxy_config, proxy_args, hp_k)
    return total


def swin_model_hp(config, args):
    _refuse(config, args)
    hybrid_parallel_configs = get_hybrid_parallel_configs(model_config=config, training_args=args)
    _refuse(config, args, hybrid_parallel_configs)
    config.tokens_run = token_rows(config, args, hybrid_parallel_configs)
    args.seq_length = config.tokens_run[0]
    vtp = hybrid_parallel_configs["vocab_tp"]
    args.padded_vocab_size = vtp * ceil8(config.num_labels // vtp)          # classes, each rank's slice padded to a multiple of 8
    if not getattr(args, "arena_bytes", 0):
        args.arena_bytes = estimate_arena_bytes(config, args, hybrid_parallel_configs)
    return construct_hybrid_parallel_model(model=SwinSkeleton(config), model_config=config, training_args=args,
                                           hybrid_parallel_configs=hybrid_parallel_configs)

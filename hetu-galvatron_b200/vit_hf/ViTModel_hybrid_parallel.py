"""Entry points of the ViT family (``galvatron/models/vit_hf/ViTModel_hybrid_parallel.py``).

Token padding rule (decided once, here, before any layer exists): a layer's GEMMs see seq x micro-batch rows, which must be a multiple
of 8.  With the real token count S = P + 1 (197 at 224 px / patch 16) that holds only for some micro-batches, so
    seq_run = S       when S x m is a multiple of 8 for every micro-batch size m any row of the strategy runs,
    seq_run = ceil8(S) otherwise (197 -> 200).
The extra tokens are zero rows from the embedding kernel, masked out as keys in every layer; the loss reads token 0 only, so their
gradient is exactly zero and every weight gradient equals the unpadded one up to summation order."""
import types

from ..core.runtime import world as _world
from ..core.runtime.hybrid_parallel_config import get_chunks, get_hybrid_parallel_configs_api
from ..core.runtime.hybrid_parallel_model import construct_hybrid_parallel_model_api
from ..llama_hf.LlamaModel_hybrid_parallel import estimate_arena_bytes as _estimate_arena_bytes
from .meta_configs import config_from_meta, set_model_config
from .ViTModel_sequential import ViTCls_, ViTEmbeddings_, ViTModelInfo, ViTPreNorm_, construct_sequential_model
from .ViTModel_tensor_parallel import ViTLayer_tp, ViTSkeleton, ceil8, construct_tensor_parallel_model


def get_hybrid_parallel_configs(model_config, training_args):
    return get_hybrid_parallel_configs_api(model_config, training_args, ViTModelInfo)


def construct_hybrid_parallel_model(model, model_config, training_args, hybrid_parallel_configs):
    return construct_hybrid_parallel_model_api(
        model, model_config, training_args, hybrid_parallel_configs, ViTModelInfo, construct_sequential_model,
        construct_tensor_parallel_model, wrap_block_name=[ViTLayer_tp], wrap_checkpoint_block_name=[ViTLayer_tp],
        wrap_other_block_name=[ViTEmbeddings_, ViTPreNorm_, ViTCls_], tied_wte_attr_names=None, layernorm_name=["LayerNorm", "layernorm"],
        all_block_name=[ViTEmbeddings_, ViTLayer_tp, ViTPreNorm_, ViTCls_])


def get_vit_config(args, overwrite_args=True):
    return set_model_config(config_from_meta(args.model_size), args, overwrite_args)


def _microbatch_sizes(local, chunks):
    """sizes of ``Tensor.chunk(chunks)`` of ``local`` samples (the pipeline's split, pipeline/utils.py)"""
    if local <= 0:
        return []
    step = -(-local // chunks)
    return [min(step, local - i) for i in range(0, local, step)]


def token_rows(config, args, hp_configs):
    """The tokens a layer runs (module docstring): S, or S rounded up to a multiple of 8 when some row's micro-batch needs it."""
    world, pp, chunks = _world.get_world_size(), hp_configs["pp_deg"], max(1, get_chunks(args))
    seq = config.seq_length
    for degree in set(hp_configs["tp_sizes_enc"]) | {hp_configs["vocab_tp"]}:
        local = args.global_train_batch_size // max(1, world // pp // degree)
        if any(seq * m % 8 for m in _microbatch_sizes(local, chunks)):
            return ceil8(seq)
    return seq


def _refuse(args, hp_configs=None):
    """The reference forces sequence_parallel = use_ulysses = False for ViT (vit_model_hp); this runtime refuses them, and the
    options ViT has no path for, instead of changing the caller's arguments."""
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
        why.append("checkpoint load / save (no HF-layered ViT checkpoint format)")
    if why:
        raise NotImplementedError("the ViT family does not support %s" % ", ".join(sorted(set(why))))


def estimate_arena_bytes(config, args, hp_configs):
    """The Llama estimate with ViT's rows: seq_run tokens, and for the embedding / head rows the larger of the patch projection +
    CLS + position table and the padded classifier + pooler, in rows of h (the estimate's 'vocabulary')."""
    k = config.patch_size * config.patch_size * config.num_channels
    rows = max(k + config.seq_length + 2, args.padded_vocab_size + config.hidden_size + 1)
    proxy_config = types.SimpleNamespace(**dict(vars(config), max_position_embeddings=config.seq_run))
    proxy_args = types.SimpleNamespace(**dict(vars(args), padded_vocab_size=rows))
    return _estimate_arena_bytes(proxy_config, proxy_args, hp_configs)


def vit_model_hp(config, args):
    _refuse(args)
    hybrid_parallel_configs = get_hybrid_parallel_configs(model_config=config, training_args=args)
    _refuse(args, hybrid_parallel_configs)
    config.seq_run = args.seq_length = token_rows(config, args, hybrid_parallel_configs)
    vtp = hybrid_parallel_configs["vocab_tp"]
    args.padded_vocab_size = vtp * ceil8(config.num_labels // vtp)          # classes, each rank's slice padded to a multiple of 8
    if not getattr(args, "arena_bytes", 0):
        args.arena_bytes = estimate_arena_bytes(config, args, hybrid_parallel_configs)
    return construct_hybrid_parallel_model(model=ViTSkeleton(config), model_config=config, training_args=args,
                                           hybrid_parallel_configs=hybrid_parallel_configs)

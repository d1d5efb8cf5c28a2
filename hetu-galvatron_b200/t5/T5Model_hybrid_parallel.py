"""Entry points of the T5 family (``galvatron/models/T5/T5Model_hybrid_parallel.py``)."""
import types

from ..core.runtime.hybrid_parallel_config import get_hybrid_parallel_configs_api
from ..core.runtime.hybrid_parallel_model import construct_hybrid_parallel_model_api
from ..llama_hf.LlamaModel_hybrid_parallel import estimate_arena_bytes as _estimate_arena_bytes
from .meta_configs import config_from_meta, set_model_config
from .T5Model_sequential import (T5Cls_, T5DecoderEmbeddings_, T5DecoderPreNorm_, T5EncoderEmbeddings_, T5EncoderPreNorm_, T5ModelInfo,
                                 construct_sequential_model)
from .T5Model_tensor_parallel import T5DecoderLayer_tp, T5EncoderLayer_tp, T5Skeleton, construct_tensor_parallel_model


def get_hybrid_parallel_configs(model_config, training_args):
    return get_hybrid_parallel_configs_api(model_config, training_args, T5ModelInfo)


def construct_hybrid_parallel_model(model, model_config, training_args, hybrid_parallel_configs):
    return construct_hybrid_parallel_model_api(
        model, model_config, training_args, hybrid_parallel_configs, T5ModelInfo, construct_sequential_model,
        construct_tensor_parallel_model, wrap_block_name=[T5EncoderLayer_tp, T5DecoderLayer_tp],
        wrap_checkpoint_block_name=[T5EncoderLayer_tp, T5DecoderLayer_tp],
        wrap_other_block_name=[T5EncoderEmbeddings_, T5DecoderEmbeddings_, T5EncoderPreNorm_, T5DecoderPreNorm_, T5Cls_],
        tied_wte_attr_names=None, layernorm_name=["LayerNorm"],
        all_block_name=[T5EncoderEmbeddings_, T5DecoderEmbeddings_, T5EncoderLayer_tp, T5EncoderPreNorm_, T5DecoderLayer_tp,
                        T5DecoderPreNorm_, T5Cls_])


def get_t5_config(args, overwrite_args=True):
    return set_model_config(config_from_meta(args.model_size), args, overwrite_args)


def _refuse(config, args, hp_configs=None):
    """What the reference forbids or has no path for, refused with an error instead of changing the caller's arguments."""
    why = []
    if args.use_ulysses:
        why.append("Ulysses sequence parallelism (use_ulysses)")
    if getattr(args, "global_cp_deg", 1) > 1 or getattr(args, "vocab_cp", 1) > 1:
        why.append("context parallelism")
    if hp_configs is not None:
        if any(c > 1 for c in hp_configs["cp_sizes_enc"]) or hp_configs.get("vocab_cp", 1) > 1:
            why.append("context parallelism")
        if any(hp_configs["use_sp"]) or hp_configs.get("vocab_sp", 0):
            why.append("Ulysses sequence parallelism (use_sp / vsp)")
    if not getattr(args, "untie_embeddings_and_output_weights", True):
        why.append("tied embeddings (the reference's tied path does not synchronise the decoder embedding)")
    if getattr(args, "load", None) not in (None, "None") or getattr(args, "save", None) not in (None, "None"):
        why.append("checkpoint load / save (the reference has no T5 checkpoint format)")
    if config.dropout_rate > 0 or float(getattr(args, "hidden_dropout", 0.0)) > 0 or float(getattr(args, "attention_dropout", 0.0)) > 0:
        why.append("hidden / attention dropout (dropout_rate > 0)")
    if why:
        raise NotImplementedError("the T5 family does not support %s" % ", ".join(sorted(set(why))))


def estimate_arena_bytes(config, args, hp_configs):
    """The Llama estimate on a proxy of T5's shape: a proxy layer with the decoder layer's parameter count (self-attention, cross
    query + key_value and two output projections over the inner width d_kv x heads, the biased MLP), both vocabulary matrices of the
    embedding rows counted on every stage, and the activation staging sized for both boundary tensors (s_enc + s_dec tokens)."""
    h, f, inner = config.hidden_size, config.ffn_hidden_size, config.d_kv * config.num_attention_heads
    n = config.num_attention_heads
    dec_params = 8 * inner * h + 2 * f * h + 9 * h + 2 * inner + f
    proxy_ffn = -(-(dec_params - 4 * h * h) // (3 * h))               # Llama's layer: 4 h^2 (MHA, hn = h / n) + 3 f h + 2 h
    proxy_config = types.SimpleNamespace(hidden_size=h, intermediate_size=max(proxy_ffn, 1), num_attention_heads=n, num_key_value_heads=n,
                                         max_position_embeddings=config.n_positions + config.n_decoder_positions)
    proxy_args = types.SimpleNamespace(**dict(vars(args), padded_vocab_size=2 * args.padded_vocab_size))
    return _estimate_arena_bytes(proxy_config, proxy_args, hp_configs)


def t5_model_hp(config, args):
    _refuse(config, args)
    hybrid_parallel_configs = get_hybrid_parallel_configs(model_config=config, training_args=args)
    _refuse(config, args, hybrid_parallel_configs)
    if not getattr(args, "arena_bytes", 0):
        args.arena_bytes = estimate_arena_bytes(config, args, hybrid_parallel_configs)
    return construct_hybrid_parallel_model(model=T5Skeleton(config), model_config=config, training_args=args,
                                           hybrid_parallel_configs=hybrid_parallel_configs)

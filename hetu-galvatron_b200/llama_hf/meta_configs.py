"""Model shapes (``galvatron/models/llama_hf/meta_configs/config_utils.py:22-110`` + the shipped *.json specs).

``config_from_meta`` accepts a known name or a dict spec {dim, ffn_dim, n_heads, n_kv_heads, n_layers, norm_eps,
vocab_size, n_positions, multiple_of}; unlike HEAD it does not crash on a dict without ``ffn_dim`` (config_utils.py:34).
"""
import types

# dim, n_heads, n_kv_heads, n_layers, norm_eps, vocab, n_positions [, ffn_dim]
_SPECS = {
    "llama-0.3b": dict(dim=1024, n_heads=16, n_layers=24, norm_eps=1e-6, vocab_size=32000, n_positions=2048, multiple_of=256),
    "llama-7b": dict(dim=4096, n_heads=32, n_layers=32, norm_eps=1e-6, vocab_size=32000, n_positions=2048, multiple_of=256),
    "llama-13b": dict(dim=5120, n_heads=40, n_layers=40, norm_eps=1e-6, vocab_size=32000, n_positions=2048, multiple_of=256),
    "llama-30b": dict(dim=6656, n_heads=52, n_layers=60, norm_eps=1e-6, vocab_size=32000, n_positions=2048, multiple_of=256),
    "llama2-70b": dict(dim=8192, n_heads=64, n_kv_heads=8, n_layers=80, norm_eps=1e-5, vocab_size=32000, n_positions=4096,
                       multiple_of=4096, ffn_dim=28672),
    # BASELINE.json configs (no meta file shipped by the reference; SURVEY 8 shapes)
    "llama3-8b": dict(dim=4096, ffn_dim=14336, n_heads=32, n_kv_heads=8, n_layers=32, norm_eps=1e-5, vocab_size=128256,
                      n_positions=8192, multiple_of=256),
    # Llama-3.2-1B shapes (untied embeddings): the flagship on one 80 GB GPU, where Llama-3-8B's AdamW state alone does not fit
    "llama3.2-1b": dict(dim=2048, ffn_dim=8192, n_heads=32, n_kv_heads=8, n_layers=16, norm_eps=1e-5, vocab_size=128256,
                        n_positions=8192, multiple_of=256),
    "llama3-70b": dict(dim=8192, ffn_dim=28672, n_heads=64, n_kv_heads=8, n_layers=80, norm_eps=1e-5, vocab_size=128256,
                       n_positions=8192, multiple_of=256),
}


def config_from_meta(model_type):
    params = dict(_SPECS[model_type]) if isinstance(model_type, str) else dict(model_type)
    params.setdefault("n_kv_heads", None)
    if "ffn_dim" not in params:
        if isinstance(model_type, str) and model_type.startswith("qwen"):
            params["ffn_dim"] = int(params["dim"] * 5.5)
        else:
            mult = params.get("multiple_of", 256)
            params["ffn_dim"] = (params["dim"] * 8 // 3 + mult - 1) // mult * mult
    return types.SimpleNamespace(
        hidden_size=params["dim"], intermediate_size=int(params["ffn_dim"]), num_attention_heads=params["n_heads"],
        num_hidden_layers=params["n_layers"], rms_norm_eps=params["norm_eps"],
        num_key_value_heads=params["n_kv_heads"] or params["n_heads"], max_position_embeddings=params["n_positions"],
        vocab_size=params["vocab_size"], attention_dropout=0.0, rope_theta=params.get("rope_theta", 10000.0),
        model_name=model_type if isinstance(model_type, str) else "custom")


def set_model_config(config, args, overwrite_args=True):
    """Keep the model config and the runtime args consistent (config_utils.py:52-110)."""
    if getattr(args, "set_seqlen_manually", False) and getattr(args, "seq_length", None):
        config.max_position_embeddings = args.seq_length
    if getattr(args, "set_layernum_manually", False) and getattr(args, "num_hidden_layers", None):
        config.num_hidden_layers = args.num_hidden_layers
    if overwrite_args:
        args.hidden_size = config.hidden_size
        args.ffn_hidden_size = config.intermediate_size
        args.num_attention_heads = config.num_attention_heads
        args.num_query_groups = config.num_key_value_heads
        args.group_query_attention = config.num_key_value_heads != config.num_attention_heads
        args.num_layers = config.num_hidden_layers
        args.seq_length = config.max_position_embeddings
        args.norm_epsilon = config.rms_norm_eps
        args.vocab_size = config.vocab_size
        args.rotary_base = config.rope_theta
        mult = getattr(args, "make_vocab_size_divisible_by", 128) * max(1, getattr(args, "vocab_tp", 1))
        args.padded_vocab_size = (config.vocab_size + mult - 1) // mult * mult   # megatron _vocab_size_with_padding
    return config

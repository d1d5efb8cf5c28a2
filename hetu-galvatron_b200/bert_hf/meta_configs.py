"""BERT model shapes (``galvatron/models/bert_hf/meta_configs/*.json`` + ``config_utils.py:13-77``).  ``config_from_meta`` takes a
shipped name or a dict spec {hidden_size, num_hidden_layers, num_attention_heads, vocab_size, max_position_embeddings, ...}."""
import types

_SPECS = {
    "bert-base": dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, vocab_size=30522, max_position_embeddings=512),
    "bert-large": dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, vocab_size=30522, max_position_embeddings=512),
    "bert-huge-32": dict(hidden_size=1280, num_hidden_layers=32, num_attention_heads=16, vocab_size=30522, max_position_embeddings=512),
    "bert-huge-48": dict(hidden_size=1280, num_hidden_layers=48, num_attention_heads=16, vocab_size=30522, max_position_embeddings=512),
}


def config_from_meta(model_type):
    p = dict(_SPECS[model_type]) if isinstance(model_type, str) else dict(model_type)
    h = p["hidden_size"]
    return types.SimpleNamespace(
        hidden_size=h, num_hidden_layers=p["num_hidden_layers"], num_attention_heads=p["num_attention_heads"],
        num_key_value_heads=p["num_attention_heads"], intermediate_size=p.get("intermediate_size") or 4 * h, vocab_size=p["vocab_size"],
        max_position_embeddings=p["max_position_embeddings"], type_vocab_size=p.get("type_vocab_size", 2),
        layer_norm_eps=p.get("layer_norm_eps", 1e-12), hidden_act=p.get("hidden_act", "gelu"),
        # BertConfig's dropouts (0.1 each in HF; 0 in the shipped specs here, see arguments.hidden_dropout)
        hidden_dropout_prob=float(p.get("hidden_dropout_prob", 0.0)),
        attention_probs_dropout_prob=float(p.get("attention_probs_dropout_prob", 0.0)),
        model_name=model_type if isinstance(model_type, str) else "custom")


def set_model_config(config, args, overwrite_args=True):
    """``config_utils.py:27-77``: keep the model config and the runtime args consistent (BASELINE config 4 forces seq 8192 with
    ``set_seqlen_manually``)."""
    if getattr(args, "set_seqlen_manually", False) and getattr(args, "seq_length", None):
        config.max_position_embeddings = args.seq_length
    if getattr(args, "set_layernum_manually", False) and getattr(args, "num_hidden_layers", None):
        config.num_hidden_layers = args.num_hidden_layers
    if overwrite_args:
        args.hidden_size, args.ffn_hidden_size = config.hidden_size, config.intermediate_size
        args.num_attention_heads, args.num_query_groups, args.group_query_attention = config.num_attention_heads, config.num_attention_heads, False
        args.num_layers = args.num_hidden_layers = config.num_hidden_layers
        args.seq_length = args.max_position_embeddings = config.max_position_embeddings
        args.norm_epsilon = config.layer_norm_eps
        args.vocab_size = config.vocab_size
        mult = getattr(args, "make_vocab_size_divisible_by", 128) * max(1, getattr(args, "vocab_tp", 1))
        args.padded_vocab_size = (config.vocab_size + mult - 1) // mult * mult
        # config_utils.py:57-58,68-69 (overwrite_megatron_args)
        args.hidden_dropout, args.attention_dropout = config.hidden_dropout_prob, config.attention_probs_dropout_prob
    return config

"""T5 model shapes (``galvatron/models/T5/meta_configs/*.json`` + ``config_utils.py``).  ``config_from_meta`` takes a shipped name or a
dict spec {d_model, d_kv, d_ff, num_heads, num_layers, vocab_size, n_positions [, num_decoder_layers, n_decoder_positions,
layer_norm_epsilon, dropout_rate]}.

The inner attention width d_kv x num_heads may differ from d_model (t5-3B: 32 x 128 = 4096 against 1024).  The shipped configs
carry dropout_rate 0.1; this runtime defaults it to 0, as for GPT / BERT (``arguments.hidden_dropout``), and refuses a config that
sets it above 0 (t5/T5Model_hybrid_parallel.py)."""
import types

_SPECS = {
    "t5-small": dict(d_model=512, d_kv=64, d_ff=2048, num_heads=8, num_layers=6, vocab_size=32128, n_positions=512),
    "t5-base": dict(d_model=768, d_kv=64, d_ff=3072, num_heads=12, num_layers=12, vocab_size=32128, n_positions=512),
    "t5-large": dict(d_model=1024, d_kv=64, d_ff=4096, num_heads=16, num_layers=24, vocab_size=32128, n_positions=512),
    "t5-3B": dict(d_model=1024, d_kv=128, d_ff=16384, num_heads=32, num_layers=24, vocab_size=32128, n_positions=512),
}


def config_from_meta(model_type):
    p = dict(_SPECS[model_type]) if isinstance(model_type, str) else dict(model_type)
    return types.SimpleNamespace(
        hidden_size=p["d_model"], d_kv=p["d_kv"], ffn_hidden_size=p["d_ff"], num_attention_heads=p["num_heads"],
        num_layers=p["num_layers"], num_decoder_layers=p.get("num_decoder_layers", p["num_layers"]), vocab_size=p["vocab_size"],
        n_positions=p["n_positions"], n_decoder_positions=p.get("n_decoder_positions", p["n_positions"]),
        layer_norm_epsilon=p.get("layer_norm_epsilon", 1e-6), dropout_rate=float(p.get("dropout_rate", 0.0)),
        model_name=model_type if isinstance(model_type, str) else "custom")


def set_model_config(config, args, overwrite_args=True):
    """``config_utils.py`` set_model_config / overwrite_megatron_args: keep the model config and the runtime args consistent."""
    if getattr(args, "set_layernum_manually", False):
        config.num_layers = getattr(args, "num_encoder_layers", None) or config.num_layers
        config.num_decoder_layers = getattr(args, "num_decoder_layers", None) or config.num_decoder_layers
    if getattr(args, "set_seqlen_manually", False):
        config.n_positions = getattr(args, "encoder_seq_length", None) or config.n_positions
        config.n_decoder_positions = getattr(args, "decoder_seq_length", None) or config.n_decoder_positions
    if overwrite_args:
        args.hidden_size, args.ffn_hidden_size, args.kv_channels = config.hidden_size, config.ffn_hidden_size, config.d_kv
        args.num_attention_heads, args.num_query_groups, args.group_query_attention = config.num_attention_heads, config.num_attention_heads, False
        args.num_encoder_layers, args.num_decoder_layers = config.num_layers, config.num_decoder_layers
        args.num_layers = args.num_hidden_layers = config.num_layers + config.num_decoder_layers
        args.encoder_seq_length, args.decoder_seq_length = config.n_positions, config.n_decoder_positions
        # the larger of the two sequences: what the activation staging is sized for
        args.seq_length = args.max_position_embeddings = max(config.n_positions, config.n_decoder_positions)
        args.norm_epsilon = config.layer_norm_epsilon
        args.vocab_size = config.vocab_size
        mult = getattr(args, "make_vocab_size_divisible_by", 128) * max(1, getattr(args, "vocab_tp", 1))
        args.padded_vocab_size = (config.vocab_size + mult - 1) // mult * mult   # megatron _vocab_size_with_padding
        args.hidden_dropout = args.attention_dropout = config.dropout_rate
    return config

"""GPT model shapes (``galvatron/models/gpt_hf/meta_configs/*.json`` + ``config_utils.py:19-110``).  ``config_from_meta`` takes
a shipped name or a dict spec {n_layer, n_embd, n_head, vocab_size, n_positions [, n_inner, layer_norm_epsilon]}."""
import types

_SPECS = {
    # the shipped meta configs
    "gpt-0.3b": dict(n_layer=24, n_embd=1024, n_head=16, vocab_size=50257, n_positions=1024),
    "gpt-1.5b": dict(n_layer=48, n_embd=1600, n_head=32, vocab_size=50257, n_positions=1024),
    "gpt-2.7b": dict(n_layer=32, n_embd=2560, n_head=32, vocab_size=50257, n_positions=2048),
    "gpt-6.7b": dict(n_layer=32, n_embd=4096, n_head=32, vocab_size=50257, n_positions=2048),
    # BASELINE.json config 1: GPT-2 small (dict spec in the reference, SURVEY 8)
    "gpt2-small": dict(n_layer=12, n_embd=768, n_head=12, vocab_size=50257, n_positions=1024),
}


def config_from_meta(model_type):
    p = dict(_SPECS[model_type]) if isinstance(model_type, str) else dict(model_type)
    h = p["n_embd"]
    return types.SimpleNamespace(
        hidden_size=h, num_hidden_layers=p["n_layer"], num_attention_heads=p["n_head"], num_key_value_heads=p["n_head"],
        intermediate_size=p.get("n_inner") or 4 * h, vocab_size=p["vocab_size"], max_position_embeddings=p["n_positions"],
        layer_norm_epsilon=p.get("layer_norm_epsilon", 1e-5), attention_dropout=0.0,
        # GPT2Config's dropouts (0.1 each in HF; 0 in the shipped specs here, see arguments.hidden_dropout)
        resid_pdrop=float(p.get("resid_pdrop", 0.0)), embd_pdrop=float(p.get("embd_pdrop", p.get("resid_pdrop", 0.0))),
        attn_pdrop=float(p.get("attn_pdrop", 0.0)),
        model_name=model_type if isinstance(model_type, str) else "custom")


def set_model_config(config, args, overwrite_args=True):
    """``config_utils.py:30-82``: keep the model config and the runtime args consistent."""
    if getattr(args, "set_seqlen_manually", False) and getattr(args, "seq_length", None):
        config.max_position_embeddings = args.seq_length
    if getattr(args, "set_layernum_manually", False) and getattr(args, "num_hidden_layers", None):
        config.num_hidden_layers = args.num_hidden_layers
    if overwrite_args:
        args.hidden_size, args.ffn_hidden_size = config.hidden_size, config.intermediate_size
        args.num_attention_heads, args.num_query_groups, args.group_query_attention = config.num_attention_heads, config.num_attention_heads, False
        args.num_layers = args.num_hidden_layers = config.num_hidden_layers
        args.seq_length = args.max_position_embeddings = config.max_position_embeddings
        args.norm_epsilon = config.layer_norm_epsilon
        args.vocab_size = config.vocab_size
        mult = getattr(args, "make_vocab_size_divisible_by", 128) * max(1, getattr(args, "vocab_tp", 1))
        args.padded_vocab_size = (config.vocab_size + mult - 1) // mult * mult   # megatron _vocab_size_with_padding
        # config_utils.py:74-76 (overwrite_megatron_args): one hidden dropout for the embedding and the residual branches
        assert abs(config.resid_pdrop - config.embd_pdrop) <= 1e-3, "resid_pdrop should be equal to embd_pdrop"
        args.hidden_dropout, args.attention_dropout = config.resid_pdrop, config.attn_pdrop
    return config

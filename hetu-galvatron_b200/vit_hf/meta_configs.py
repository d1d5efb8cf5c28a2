"""ViT model shapes (``galvatron/models/vit_hf/meta_configs/vit-*-patch16-224.json`` + ``config_utils.py``).  ``config_from_meta``
takes a shipped name or a dict spec {hidden_size, num_hidden_layers, num_attention_heads, image_size, patch_size, ...}."""
import types

_COMMON = dict(image_size=224, patch_size=16, num_channels=3, num_labels=1000, layer_norm_eps=1e-12)
_SPECS = {
    "vit-base-patch16-224": dict(_COMMON, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072),
    "vit-large-patch16-224": dict(_COMMON, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096),
    "vit-huge-patch16-224": dict(_COMMON, hidden_size=1280, num_hidden_layers=32, num_attention_heads=16, intermediate_size=5120),
    "vit-xhuge-patch16-224": dict(_COMMON, hidden_size=2560, num_hidden_layers=128, num_attention_heads=32, intermediate_size=10240),
}


def config_from_meta(model_type):
    p = dict(_SPECS[model_type]) if isinstance(model_type, str) else dict(_COMMON, **model_type)
    h, img, patch = p["hidden_size"], p["image_size"], p["patch_size"]
    if img % patch:
        raise ValueError("ViT: image size %d is not a multiple of the patch size %d" % (img, patch))
    n_patches = (img // patch) ** 2
    return types.SimpleNamespace(
        hidden_size=h, num_hidden_layers=p["num_hidden_layers"], num_attention_heads=p["num_attention_heads"],
        num_key_value_heads=p["num_attention_heads"], intermediate_size=p.get("intermediate_size") or 4 * h, image_size=img,
        patch_size=patch, num_channels=p["num_channels"], num_labels=p["num_labels"], layer_norm_eps=p["layer_norm_eps"],
        hidden_act="gelu_pytorch_tanh",
        # ViTConfig's dropouts (0 in the shipped specs)
        hidden_dropout_prob=float(p.get("hidden_dropout_prob", 0.0)),
        attention_probs_dropout_prob=float(p.get("attention_probs_dropout_prob", 0.0)),
        # tokens: the patches and the CLS token; seq_run = the tokens a layer runs, padding included (vit_model_hp sets it)
        n_patches=n_patches, seq_length=n_patches + 1, seq_run=n_patches + 1,
        model_name=model_type if isinstance(model_type, str) else "custom")


def set_model_config(config, args, overwrite_args=True):
    """``config_utils.py``: keep the model config and the runtime args consistent."""
    if getattr(args, "set_layernum_manually", False) and getattr(args, "num_hidden_layers", None):
        config.num_hidden_layers = args.num_hidden_layers
    if overwrite_args:
        args.hidden_size, args.ffn_hidden_size = config.hidden_size, config.intermediate_size
        args.num_attention_heads, args.num_query_groups, args.group_query_attention = config.num_attention_heads, config.num_attention_heads, False
        args.num_layers = args.num_hidden_layers = config.num_hidden_layers
        args.seq_length = args.max_position_embeddings = config.seq_length
        args.norm_epsilon = config.layer_norm_eps
        args.num_labels = config.num_labels
        args.hidden_dropout, args.attention_dropout = config.hidden_dropout_prob, config.attention_probs_dropout_prob
    return config

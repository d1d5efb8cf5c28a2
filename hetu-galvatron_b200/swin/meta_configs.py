"""Swin model shapes (``galvatron/models/swin/meta_configs/swin-*.json`` + ``config_utils.py``).  ``config_from_meta`` takes a
shipped name or a dict spec {embed_dim, depths, num_heads, window_size, image_size, patch_size, ...}.  ``relative_position_bias``
(False in both shipped specs, the reference's model) gives every block HF's learned relative-position table."""
import types

_COMMON = dict(patch_size=4, num_channels=3, num_labels=1000, layer_norm_eps=1e-5, mlp_ratio=4, drop_path_rate=0.1,
               hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, use_absolute_embeddings=False,
               relative_position_bias=False)
_SPECS = {
    "swin-huge-patch4-window7-224": dict(_COMMON, embed_dim=320, depths=[2, 2, 42, 2], num_heads=[8, 16, 32, 64], window_size=7,
                                         image_size=224),
    "swin-large-patch4-window12-384": dict(_COMMON, embed_dim=192, depths=[2, 2, 18, 2], num_heads=[6, 12, 24, 48], window_size=12,
                                           image_size=384),
}
_ALIASES = {"swin-huge": "swin-huge-patch4-window7-224", "swin-large": "swin-large-patch4-window12-384"}


def stage_geometry(config):
    """One dict per stage: grid side ``res``, real tokens, width, heads, and the block's window / shift (HF SwinLayer: when the
    grid is no larger than the window, one window covers it and nothing is shifted)."""
    side = config.image_size // config.patch_size
    stages = []
    for k, (depth, heads) in enumerate(zip(config.depths, config.num_heads)):
        res = side >> k
        ws = min(config.window_size, res)
        shift = 0 if res <= config.window_size else config.window_size // 2
        stages.append(dict(res=res, tokens=res * res, width=config.embed_dim << k, heads=heads, depth=depth, window=ws, shift=shift))
    return stages


def config_from_meta(model_type):
    if isinstance(model_type, str):
        p = dict(_SPECS[_ALIASES.get(model_type, model_type)])
    else:
        p = dict(_COMMON, **model_type)
    if p["image_size"] % p["patch_size"]:
        raise ValueError("Swin: image size %d is not a multiple of the patch size %d" % (p["image_size"], p["patch_size"]))
    config = types.SimpleNamespace(
        embed_dim=p["embed_dim"], depths=list(p["depths"]), num_heads=list(p["num_heads"]), window_size=p["window_size"],
        image_size=p["image_size"], patch_size=p["patch_size"], num_channels=p["num_channels"], num_labels=p["num_labels"],
        layer_norm_eps=p["layer_norm_eps"], mlp_ratio=p["mlp_ratio"], drop_path_rate=float(p["drop_path_rate"]),
        hidden_dropout_prob=float(p["hidden_dropout_prob"]), attention_probs_dropout_prob=float(p["attention_probs_dropout_prob"]),
        use_absolute_embeddings=bool(p["use_absolute_embeddings"]), relative_position_bias=bool(p["relative_position_bias"]),
        hidden_act="gelu_pytorch_tanh",
        model_name=model_type if isinstance(model_type, str) else "custom")
    config.num_hidden_layers = sum(config.depths)
    config.stages = stage_geometry(config)
    # the tokens a stage's rows run, padding included (swin_model_hp sets them)
    config.tokens_run = [s["tokens"] for s in config.stages]
    return config


def set_model_config(config, args, overwrite_args=True):
    """``config_utils.py``: keep the model config and the runtime args consistent (the args describe stage 0)."""
    if overwrite_args:
        c0 = config.embed_dim
        args.hidden_size, args.ffn_hidden_size = c0, c0 * config.mlp_ratio
        args.num_attention_heads, args.num_query_groups, args.group_query_attention = config.num_heads[0], config.num_heads[0], False
        args.num_layers = args.num_hidden_layers = config.num_hidden_layers
        args.seq_length = args.max_position_embeddings = config.tokens_run[0]
        args.norm_epsilon = config.layer_norm_eps
        args.num_labels = config.num_labels
        args.hidden_dropout, args.attention_dropout = config.hidden_dropout_prob, config.attention_probs_dropout_prob
        args.drop_path_rate = config.drop_path_rate
    return config

"""Single-process restatement of the ViT model the reference runtime executes (TEST INFRASTRUCTURE ONLY).

Plain torch, no parallelism, no custom kernels -- what one rank of the reference computes when every group has size 1:
  vit_hf/ViTModel_sequential.py:33-64 (einops patchify "b c (h p1) (w p2) -> b (h w) (p1 p2 c)", the patch linear with bias, the CLS
  token prepended, + position table, [b,s,h] -> [s,b,h], hidden dropout), ViTModel_tensor_parallel.py:10-80 (PRE-LayerNorm blocks,
  bidirectional attention, biases on every projection, tanh-GeLU MLP, hidden dropout on both block outputs), ViTModel_sequential.py
  :79-180 (final LayerNorm, the pooler dense + tanh on token 0, the classifier WITHOUT its bias, per-sample vocab-parallel CE).
Layer math is oracle/gpt_bert_ref.py's (fused per-head QKV layout).  ``dtype`` = torch.bfloat16 rounds every op's output to bf16 at
the points the product rounds; float64 is exact math.  Pinned against HF ``ViTModel(add_pooling_layer=True)`` with
``hidden_act="gelu_pytorch_tanh"`` and a bias-free linear in fp64 by tests/test_vit.py.

Dropout (optional): ``drop`` has ``.hidden`` (the probability) and ``.apply(x, bias, residual, p, site, dtype)`` -> residual + keep *
scale * (x + bias) rounded to dtype, with the masks of include/bg_galvatron.h (tests/_dropout_ref.Drop)."""
import torch

from . import gpt_bert_ref as ref


def patchify(pixels, patch):
    """[b, C, H, W] -> [b, P, p*p*C] in (p1 p2 c) order"""
    b, c, hgt, wid = pixels.shape
    x = pixels.reshape(b, c, hgt // patch, patch, wid // patch, patch).permute(0, 2, 4, 3, 5, 1)
    return x.reshape(b, (hgt // patch) * (wid // patch), patch * patch * c)


def _site(row, kind):
    return 3 * row + kind


def _no_bias(p, key):
    return dict(p, **{key: torch.zeros_like(p[key])})


def forward_loss(weights, pixels, labels, cfg, dtype=torch.float32, drop=None):
    """pixels [b, C, H, W], labels [b] -> (per-sample loss [b], scalar mean).  weights: patch [h, p*p*C], patch_b [h], cls [h],
    pos [S, h], layers [{ln1, ln1_b, qkv, qkv_b, dense, dense_b, ln2, ln2_b, h_to_4h, h_to_4h_b, 4h_to_h, 4h_to_h_b}], norm, norm_b,
    pooler [h, h], pooler_b [h], classifier [num_labels, h].  cfg: hidden, ffn, n_heads, head_dim, eps, patch."""
    wd = lambda t: ref._r(t, dtype) if t.dtype != torch.float64 else t  # noqa: E731
    hd = drop is not None and drop.hidden > 0
    x = ref._r(patchify(pixels, cfg["patch"]), dtype)
    e = ref._r(x @ wd(weights["patch"]).t(), dtype)                                   # [b, P, h]
    pos = wd(weights["pos"])
    rows = e + (pos[1:] + wd(weights["patch_b"]))[None]
    first = (pos[0] + wd(weights["cls"])).expand(e.shape[0], 1, -1)
    h = torch.cat([first, rows], dim=1).transpose(0, 1)                                # [S, b, h], unrounded sums
    h = drop.apply(h, None, None, drop.hidden, _site(0, 0), dtype) if hd else ref._r(h, dtype)
    for i, lw in enumerate(weights["layers"]):
        p = {k: wd(v) for k, v in lw.items()}
        y = ref.layer_norm(h, p["ln1"], p["ln1_b"], cfg["eps"], dtype)
        if hd:
            h = drop.apply(ref.attention(y, _no_bias(p, "dense_b"), cfg, dtype, False, None), p["dense_b"], h, drop.hidden,
                           _site(i + 1, 1), dtype)
        else:
            h = ref._r(ref.attention(y, p, cfg, dtype, False, None) + h, dtype)
        y = ref.layer_norm(h, p["ln2"], p["ln2_b"], cfg["eps"], dtype)
        if hd:
            h = drop.apply(ref.mlp(y, _no_bias(p, "4h_to_h_b"), cfg, dtype), p["4h_to_h_b"], h, drop.hidden, _site(i + 1, 2), dtype)
        else:
            h = ref._r(ref.mlp(y, p, cfg, dtype) + h, dtype)
    h = ref.layer_norm(h, wd(weights["norm"]), wd(weights["norm_b"]), cfg["eps"], dtype)
    pooled = ref._r(torch.tanh(ref._r(h[0] @ wd(weights["pooler"]).t(), dtype) + wd(weights["pooler_b"])), dtype)
    logits = ref._r(pooled @ wd(weights["classifier"]).t(), dtype)                      # [b, num_labels]
    loss = ref._token_loss(logits.unsqueeze(0), labels.unsqueeze(0), dtype)[0]
    return loss, loss.mean()


def init_weights(cfg, seed=0, std=0.02, dtype=torch.float32):
    """cfg: hidden, ffn, n_heads, head_dim, n_layers, patch, channels, seq, num_labels"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    rnd = lambda *shape: (torch.randn(*shape, generator=g) * std).to(dtype)  # noqa: E731
    h, k = cfg["hidden"], cfg["patch"] * cfg["patch"] * cfg["channels"]
    layers = [ref._layer(cfg, rnd, dtype) for _ in range(cfg["n_layers"])]
    return dict(patch=rnd(h, k), patch_b=rnd(h), cls=rnd(h), pos=rnd(cfg["seq"], h), layers=layers, norm=torch.ones(h, dtype=dtype),
                norm_b=torch.zeros(h, dtype=dtype), pooler=rnd(h, h), pooler_b=rnd(h), classifier=rnd(cfg["num_labels"], h))


def to_hf_state_dict(w, cfg):
    """oracle weights -> the HF ``ViTModel(add_pooling_layer=True)`` state dict (the mapping tests/test_vit.py pins) and the
    classifier weight.  HF's patch projection is a Conv2d [h, C, p, p]: the linear weight [h, p*p*C] is its permute(0, 2, 3, 1)."""
    p, c, h = cfg["patch"], cfg["channels"], cfg["hidden"]
    sd = {"embeddings.cls_token": w["cls"].view(1, 1, h), "embeddings.position_embeddings": w["pos"].unsqueeze(0),
          "embeddings.patch_embeddings.projection.weight": w["patch"].view(h, p, p, c).permute(0, 3, 1, 2).contiguous(),
          "embeddings.patch_embeddings.projection.bias": w["patch_b"], "layernorm.weight": w["norm"], "layernorm.bias": w["norm_b"],
          "pooler.dense.weight": w["pooler"], "pooler.dense.bias": w["pooler_b"]}
    for i, lw in enumerate(w["layers"]):
        (q, k, v), (qb, kb, vb) = ref.split_qkv(lw, cfg)
        pre = "encoder.layer.%d." % i
        sd.update({pre + "attention.attention.query.weight": q, pre + "attention.attention.query.bias": qb,
                   pre + "attention.attention.key.weight": k, pre + "attention.attention.key.bias": kb,
                   pre + "attention.attention.value.weight": v, pre + "attention.attention.value.bias": vb,
                   pre + "attention.output.dense.weight": lw["dense"], pre + "attention.output.dense.bias": lw["dense_b"],
                   pre + "intermediate.dense.weight": lw["h_to_4h"], pre + "intermediate.dense.bias": lw["h_to_4h_b"],
                   pre + "output.dense.weight": lw["4h_to_h"], pre + "output.dense.bias": lw["4h_to_h_b"],
                   pre + "layernorm_before.weight": lw["ln1"], pre + "layernorm_before.bias": lw["ln1_b"],
                   pre + "layernorm_after.weight": lw["ln2"], pre + "layernorm_after.bias": lw["ln2_b"]})
    return sd, w["classifier"]

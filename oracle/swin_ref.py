"""Single-process restatement of the Swin model this repository runs for the reference's ``models/swin`` (TEST INFRASTRUCTURE ONLY).

Plain torch, no parallelism, no custom kernels, written on the [b, H, W, C] grid the way HF ``SwinForImageClassification`` is: the
einops patchify + patch linear with bias + LayerNorm; per stage, pre-LN blocks with attention inside ws x ws windows after
``roll(-s, -s)`` on every odd block (HF's windows and HF's shift mask, window w with window w's mask), biases on every projection,
tanh-GeLU MLP, per-sample drop path on the attention branch; patch merging (x0 = [0::2, 0::2], x1 = [1::2, 0::2], x2 = [0::2, 1::2],
x3 = [1::2, 1::2]) + LayerNorm(4C) + bias-free 4C -> 2C reduction between stages; final LayerNorm, mean over tokens, bias-free
classifier, per-sample cross entropy.  What the reference differs in and this follows instead is in DESIGN.md section 5: no
relative-position bias (the reference's attention has none), HF's windows (the reference's are strided across the image) and a
per-sample drop path at one uniform rate.

``dtype`` = torch.bfloat16 rounds every op's output at the points the product rounds; float64 is exact math.  Pinned in fp64 to HF
``SwinForImageClassification`` with zeroed relative-position tables and a zero classifier bias by tests/test_swin.py.

Drop path (optional): ``drop`` has ``.rate`` and ``.keep(site, b)`` -> bool [b], the per-sample masks of include/bg_galvatron.h
(tests/_swin_backend.DropPath)."""
import torch
import torch.nn.functional as F


def _r(t, dtype):
    return t if dtype == torch.float64 else t.to(dtype).float()


def patchify(pixels, patch):
    """[b, C, H, W] -> [b, H/p, W/p, p*p*C] in (p1 p2 c) order"""
    b, c, hgt, wid = pixels.shape
    return pixels.reshape(b, c, hgt // patch, patch, wid // patch, patch).permute(0, 2, 4, 3, 5, 1).reshape(
        b, hgt // patch, wid // patch, patch * patch * c)


def layer_norm(x, w, b, eps, dtype):
    comp = torch.float64 if dtype == torch.float64 else torch.float32
    xf = x.to(comp)
    mean = xf.mean(-1, keepdim=True)
    var = (xf - mean).pow(2).mean(-1, keepdim=True)
    return _r((xf - mean) / torch.sqrt(var + eps) * w.to(comp) + b.to(comp), dtype)


def hf_shift_mask(res, window, shift):
    """HF SwinLayer.get_attn_mask(...) != 0 -> bool [nW, L, L]"""
    img = torch.zeros(1, res, res, 1)
    cnt = 0
    for hs in (slice(0, -window), slice(-window, -shift), slice(-shift, None)):
        for ws in (slice(0, -window), slice(-window, -shift), slice(-shift, None)):
            img[:, hs, ws, :] = cnt
            cnt += 1
    mw = window_partition(img, window).reshape(-1, window * window)
    return (mw.unsqueeze(1) - mw.unsqueeze(2)) != 0


def window_partition(x, window):
    """[b, H, W, C] -> [b * nW, ws * ws, C] (HF window_partition)"""
    b, hgt, wid, c = x.shape
    x = x.view(b, hgt // window, window, wid // window, window, c).permute(0, 1, 3, 2, 4, 5)
    return x.reshape(-1, window * window, c)


def window_reverse(x, window, hgt, wid):
    c = x.shape[-1]
    b = x.shape[0] // ((hgt // window) * (wid // window))
    x = x.view(b, hgt // window, wid // window, window, window, c).permute(0, 1, 3, 2, 4, 5)
    return x.reshape(b, hgt, wid, c)


def stages_of(cfg):
    side, out = cfg["image"] // cfg["patch"], []
    for k, (depth, heads) in enumerate(zip(cfg["depths"], cfg["heads"])):
        res = side >> k
        out.append(dict(res=res, width=cfg["embed_dim"] << k, heads=heads, depth=depth, window=min(cfg["window"], res),
                        shift=0 if res <= cfg["window"] else cfg["window"] // 2))
    return out


def block(h, p, st, shifted, cfg, dtype, drop=None, site_id=0):
    """h [b, H, W, C] -> the block's output (same shape)"""
    b, res, _, c = h.shape
    heads, ws = st["heads"], st["window"]
    hn, s = c // heads, (st["shift"] if shifted else 0)
    comp = torch.float64 if dtype == torch.float64 else torch.float32
    y = layer_norm(h, p["ln1"], p["ln1_b"], cfg["eps"], dtype)
    qkv = _r(_r(y @ p["qkv"].t(), dtype) + p["qkv_b"], dtype)                          # per head q | k | v
    if s:
        qkv = torch.roll(qkv, shifts=(-s, -s), dims=(1, 2))
    win = window_partition(qkv, ws).view(-1, ws * ws, heads, 3, hn).to(comp)         # [b * nW, L, heads, 3, hn]
    q, k, v = [win[:, :, :, i].transpose(1, 2) for i in range(3)]                    # [b * nW, heads, L, hn]
    scores = q @ k.transpose(-1, -2) * hn ** -0.5
    if s:
        mask = hf_shift_mask(res, ws, s).repeat(b, 1, 1)[:, None]
        scores = scores.masked_fill(mask, float("-inf"))
    ctx = _r(torch.softmax(scores, -1) @ v, dtype).transpose(1, 2).reshape(-1, ws * ws, c)
    ctx = window_reverse(ctx, ws, res, res)
    if s:
        ctx = torch.roll(ctx, shifts=(s, s), dims=(1, 2))
    if drop is not None and drop.rate > 0:
        keep = drop.keep(site_id, b).view(b, 1, 1, 1)
        scale = torch.tensor(1.0 / (1.0 - drop.rate), dtype=torch.float32).to(comp)
        out = _r(ctx @ p["dense"].t(), dtype)
        h = _r(h + torch.where(keep, (out + p["dense_b"]) * scale, torch.zeros((), dtype=comp)), dtype)
    else:
        h = _r(_r(ctx @ p["dense"].t() + h, dtype) + p["dense_b"], dtype)
    y = layer_norm(h, p["ln2"], p["ln2_b"], cfg["eps"], dtype)
    a = _r(y @ p["h_to_4h"].t(), dtype)
    g = _r(F.gelu(a + p["h_to_4h_b"], approximate="tanh"), dtype)
    return _r(_r(g @ p["4h_to_h"].t() + h, dtype) + p["4h_to_h_b"], dtype)


def merge(h, p, cfg, dtype):
    x = torch.cat([h[:, 0::2, 0::2], h[:, 1::2, 0::2], h[:, 0::2, 1::2], h[:, 1::2, 1::2]], dim=-1)
    return _r(layer_norm(x, p["norm"], p["norm_b"], cfg["eps"], dtype) @ p["reduction"].t(), dtype)


def forward_loss(weights, pixels, labels, cfg, dtype=torch.float32, drop=None):
    """pixels [b, C, H, W], labels [b] -> (per-sample loss [b], scalar mean).  weights: patch [C0, p*p*ch], patch_b, emb_ln, emb_ln_b,
    stages [{blocks: [{ln1, ln1_b, qkv, qkv_b, dense, dense_b, ln2, ln2_b, h_to_4h, h_to_4h_b, 4h_to_h, 4h_to_h_b}], merge: {norm,
    norm_b, reduction} or None}], norm, norm_b, classifier [num_labels, C_last].  cfg: embed_dim, depths, heads, window, patch, image,
    eps.  Drop path sites: site(layer + 1, 1) with layer the block's index over the whole model."""
    comp = torch.float64 if dtype == torch.float64 else torch.float32
    wd = lambda t: t if dtype == torch.float64 else _r(t, dtype)  # noqa: E731
    x = _r(patchify(pixels.to(comp), cfg["patch"]), dtype)
    h = layer_norm(_r(x @ wd(weights["patch"]).t(), dtype) + wd(weights["patch_b"]), wd(weights["emb_ln"]), wd(weights["emb_ln_b"]),
                   cfg["eps"], dtype)
    layer = 0
    for st, sw in zip(stages_of(cfg), weights["stages"]):
        for j, bw in enumerate(sw["blocks"]):
            h = block(h, {k: wd(v) for k, v in bw.items()}, st, j % 2 == 1, cfg, dtype, drop, 3 * (layer + 1) + 1)
            layer += 1
        if sw["merge"] is not None:
            h = merge(h, {k: wd(v) for k, v in sw["merge"].items()}, cfg, dtype)
    h = layer_norm(h, wd(weights["norm"]), wd(weights["norm_b"]), cfg["eps"], dtype)
    pooled = _r(h.reshape(h.shape[0], -1, h.shape[-1]).mean(1), dtype)
    logits = _r(pooled @ wd(weights["classifier"]).t(), dtype)
    loss = F.cross_entropy(logits.to(comp), labels, reduction="none")
    return loss, loss.mean()


def init_weights(cfg, num_labels, seed=0, std=0.02, dtype=torch.float32):
    g = torch.Generator(device="cpu").manual_seed(seed)
    rnd = lambda *shape: (torch.randn(*shape, generator=g) * std).to(dtype)  # noqa: E731
    ones = lambda n: torch.ones(n, dtype=dtype)  # noqa: E731
    zeros = lambda n: torch.zeros(n, dtype=dtype)  # noqa: E731
    c0, k = cfg["embed_dim"], cfg["patch"] * cfg["patch"] * cfg.get("channels", 3)
    stages = []
    sts = stages_of(cfg)
    for i, st in enumerate(sts):
        c = st["width"]
        blocks = [dict(ln1=ones(c), ln1_b=zeros(c), qkv=rnd(3 * c, c), qkv_b=rnd(3 * c), dense=rnd(c, c), dense_b=rnd(c), ln2=ones(c),
                       ln2_b=zeros(c), h_to_4h=rnd(4 * c, c), h_to_4h_b=rnd(4 * c), **{"4h_to_h": rnd(c, 4 * c), "4h_to_h_b": rnd(c)})
                  for _ in range(st["depth"])]
        mg = dict(norm=ones(4 * c), norm_b=zeros(4 * c), reduction=rnd(2 * c, 4 * c)) if i + 1 < len(sts) else None
        stages.append(dict(blocks=blocks, merge=mg))
    cl = sts[-1]["width"]
    return dict(patch=rnd(c0, k), patch_b=rnd(c0), emb_ln=ones(c0), emb_ln_b=zeros(c0), stages=stages, norm=ones(cl), norm_b=zeros(cl),
                classifier=rnd(num_labels, cl))


def to_hf_state_dict(w, cfg):
    """oracle weights -> HF ``SwinForImageClassification`` tensors (the mapping tests/test_swin.py pins): the conv patch weight
    [C, ch, p, p] is the linear weight [C, p*p*ch] through permute(0, 3, 1, 2) of its [C, p, p, ch] view; the fused per-head QKV rows
    split into query / key / value."""
    p, c0 = cfg["patch"], cfg["embed_dim"]
    ch = w["patch"].shape[1] // (p * p)
    sd = {"swin.embeddings.patch_embeddings.projection.weight": w["patch"].view(c0, p, p, ch).permute(0, 3, 1, 2).contiguous(),
          "swin.embeddings.patch_embeddings.projection.bias": w["patch_b"], "swin.embeddings.norm.weight": w["emb_ln"],
          "swin.embeddings.norm.bias": w["emb_ln_b"], "swin.layernorm.weight": w["norm"], "swin.layernorm.bias": w["norm_b"],
          "classifier.weight": w["classifier"], "classifier.bias": torch.zeros(w["classifier"].shape[0], dtype=w["classifier"].dtype)}
    for k, (st, sw) in enumerate(zip(stages_of(cfg), w["stages"])):
        heads, c = st["heads"], st["width"]
        for j, bw in enumerate(sw["blocks"]):
            pre = "swin.encoder.layers.%d.blocks.%d." % (k, j)
            qkv, qkv_b = bw["qkv"].view(heads, 3, c // heads, c), bw["qkv_b"].view(heads, 3, c // heads)
            for i, name in enumerate(("query", "key", "value")):
                sd[pre + "attention.self.%s.weight" % name] = qkv[:, i].reshape(c, c)
                sd[pre + "attention.self.%s.bias" % name] = qkv_b[:, i].reshape(c)
            sd.update({pre + "attention.output.dense.weight": bw["dense"], pre + "attention.output.dense.bias": bw["dense_b"],
                       pre + "layernorm_before.weight": bw["ln1"], pre + "layernorm_before.bias": bw["ln1_b"],
                       pre + "layernorm_after.weight": bw["ln2"], pre + "layernorm_after.bias": bw["ln2_b"],
                       pre + "intermediate.dense.weight": bw["h_to_4h"], pre + "intermediate.dense.bias": bw["h_to_4h_b"],
                       pre + "output.dense.weight": bw["4h_to_h"], pre + "output.dense.bias": bw["4h_to_h_b"]})
        if sw["merge"] is not None:
            pre = "swin.encoder.layers.%d.downsample." % k
            sd.update({pre + "reduction.weight": sw["merge"]["reduction"], pre + "norm.weight": sw["merge"]["norm"],
                       pre + "norm.bias": sw["merge"]["norm_b"]})
    return sd

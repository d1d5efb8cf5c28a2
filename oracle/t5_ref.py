"""Single-process restatement of the T5 model this repository runs for the reference's ``models/T5`` (TEST INFRASTRUCTURE ONLY).

Plain torch, no parallelism, no custom kernels.  Encoder: per layer x + Attn(RMSNorm(x)), then x + MLP(RMSNorm(x)), attention over
all tokens; final RMSNorm.  Decoder: causal self-attention, cross-attention (queries from the decoder, keys / values from the
encoder output), MLP, each pre-norm with a residual; final RMSNorm; bias-free lm_head; per-token cross entropy.  The reference's
Megatron blocks: biases on every projection, scale 1 / sqrt(d_kv) over the inner width d_kv x heads, tanh-GeLU MLP, no
relative-position bias, no positions, three untied vocabulary matrices (``shared``, ``dec_shared``, ``lm_head``).  A label -1 is
scored as Megatron's vocab-parallel cross entropy scores it (target logit = the row's maximum, i.e. 0 after the max is taken off).

Weights: shared, dec_shared [V, h]; enc_norm, dec_norm [h]; lm_head [V, h]; enc: [{ln1, qkv [3 inner, h] per head q | k | v, qkv_b,
dense [h, inner], dense_b, ln2, h_to_4h [f, h], h_to_4h_b, 4h_to_h [h, f], 4h_to_h_b}]; dec: the same plus lnx, q [inner, h], q_b,
kv [2 inner, h] per head k | v, kv_b, xdense [h, inner], xdense_b.

``dtype`` = torch.bfloat16 rounds every op's output at the points the product rounds; float64 is exact math.  Pinned in fp64 to HF
``T5ForConditionalGeneration`` (gelu_new, untied, relative-attention tables and biases zero, q pre-scaled by 1 / sqrt(d_kv),
shared = dec_shared) by tests/test_t5.py."""
import torch
import torch.nn.functional as F


def _r(t, dtype):
    return t if dtype == torch.float64 else t.to(dtype).float()


def rms_norm(x, w, eps, dtype):
    comp = torch.float64 if dtype == torch.float64 else torch.float32
    xf = x.to(comp)
    return _r(xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps) * w.to(comp), dtype)


def _attend(q, k, v, heads, causal):
    """q [b, sq, inner], k / v [b, sk, inner] -> [b, sq, inner] (softmax over keys, scale 1 / sqrt(hn))"""
    b, sq, inner = q.shape
    hn = inner // heads
    q, k, v = [t.view(b, -1, heads, hn).transpose(1, 2) for t in (q, k, v)]
    scores = q @ k.transpose(-1, -2) * hn ** -0.5
    if causal:
        s = scores.shape[-1]
        scores = scores.masked_fill(torch.triu(torch.ones(s, s, dtype=torch.bool), 1), float("-inf"))
    return (torch.softmax(scores, -1) @ v).transpose(1, 2).reshape(b, sq, inner)


def _self_attention(h, p, heads, eps, causal, dtype, ln="ln1", qkv="qkv", dense="dense"):
    y = rms_norm(h, p[ln], eps, dtype)
    m = _r(_r(y @ p[qkv].t(), dtype) + p[qkv + "_b"], dtype)
    b, s, _ = m.shape
    m = m.view(b, s, heads, 3, -1)
    q, k, v = [m[:, :, :, i].reshape(b, s, -1) for i in range(3)]
    ctx = _r(_attend(q, k, v, heads, causal), dtype)
    return _r(_r(ctx @ p[dense].t() + h, dtype) + p[dense + "_b"], dtype)


def _cross_attention(h, enc, p, heads, eps, dtype):
    y = rms_norm(h, p["lnx"], eps, dtype)
    q = _r(_r(y @ p["q"].t(), dtype) + p["q_b"], dtype)
    kv = _r(_r(enc @ p["kv"].t(), dtype) + p["kv_b"], dtype)
    b, s, _ = kv.shape
    kv = kv.view(b, s, heads, 2, -1)
    k, v = kv[:, :, :, 0].reshape(b, s, -1), kv[:, :, :, 1].reshape(b, s, -1)
    ctx = _r(_attend(q, k, v, heads, False), dtype)
    return _r(_r(ctx @ p["xdense"].t() + h, dtype) + p["xdense_b"], dtype)


def _mlp(h, p, eps, dtype):
    y = rms_norm(h, p["ln2"], eps, dtype)
    a = _r(y @ p["h_to_4h"].t(), dtype)
    g = _r(F.gelu(a + p["h_to_4h_b"], approximate="tanh"), dtype)
    return _r(_r(g @ p["4h_to_h"].t() + h, dtype) + p["4h_to_h_b"], dtype)


def token_loss(logits, labels):
    """per-token cross entropy [b, s] of logits [b, s, V]; label -1 -> logsumexp - max (Megatron's target logit 0 after the max)"""
    lf = logits.to(torch.float64 if logits.dtype == torch.float64 else torch.float32)
    lse = torch.logsumexp(lf, -1)
    picked = lf.gather(-1, labels.clamp(min=0).unsqueeze(-1)).squeeze(-1)
    return lse - torch.where(labels >= 0, picked, lf.max(-1).values)


def forward_logits(w, enc_tokens, dec_tokens, cfg, dtype=torch.float32):
    """-> logits [b, s_dec, V].  cfg: heads, eps."""
    comp = torch.float64 if dtype == torch.float64 else torch.float32
    wd = (lambda t: t) if dtype == torch.float64 else (lambda t: _r(t, dtype))
    heads, eps = cfg["heads"], cfg["eps"]
    cast = lambda p: {k: wd(t).to(comp) for k, t in p.items()}  # noqa: E731
    h = wd(w["shared"]).to(comp)[enc_tokens]
    for p in w["enc"]:
        p = cast(p)
        h = _mlp(_self_attention(h, p, heads, eps, False, dtype), p, eps, dtype)
    enc = rms_norm(h, wd(w["enc_norm"]), eps, dtype)
    d = wd(w["dec_shared"]).to(comp)[dec_tokens]
    for p in w["dec"]:
        p = cast(p)
        d = _self_attention(d, p, heads, eps, True, dtype)
        d = _cross_attention(d, enc, p, heads, eps, dtype)
        d = _mlp(d, p, eps, dtype)
    d = rms_norm(d, wd(w["dec_norm"]), eps, dtype)
    return _r(d @ wd(w["lm_head"]).to(comp).t(), dtype)


def forward_loss(w, enc_tokens, dec_tokens, labels, cfg, dtype=torch.float32, loss_mask=None):
    """-> (per-token loss [b, s_dec], scalar): the mean over all tokens, or with ``loss_mask`` the reference's masked mean
    sum(loss * mask) / sum(mask)."""
    loss = token_loss(forward_logits(w, enc_tokens, dec_tokens, cfg, dtype), labels)
    if loss_mask is None:
        return loss, loss.mean()
    m = loss_mask.to(loss.dtype)
    return loss, (loss * m).sum() / m.sum()


def init_weights(h, inner, ffn, vocab, n_enc, n_dec, seed=0, std=0.05, dtype=torch.float32):
    """random weights of the layout above (biases and norm weights random too, so that every path is exercised)"""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=g, dtype=dtype) * std  # noqa: E731
    one = lambda: 1 + rnd(h)  # noqa: E731

    def layer(cross):
        p = dict(ln1=one(), qkv=rnd(3 * inner, h), qkv_b=rnd(3 * inner), dense=rnd(h, inner), dense_b=rnd(h), ln2=one(),
                 h_to_4h=rnd(ffn, h), h_to_4h_b=rnd(ffn), **{"4h_to_h": rnd(h, ffn), "4h_to_h_b": rnd(h)})
        if cross:
            p.update(lnx=one(), q=rnd(inner, h), q_b=rnd(inner), kv=rnd(2 * inner, h), kv_b=rnd(2 * inner), xdense=rnd(h, inner),
                     xdense_b=rnd(h))
        return p
    return dict(shared=rnd(vocab, h), dec_shared=rnd(vocab, h), enc_norm=one(), dec_norm=one(), lm_head=rnd(vocab, h),
                enc=[layer(False) for _ in range(n_enc)], dec=[layer(True) for _ in range(n_dec)])


def to_hf_state_dict(w, heads):
    """HF T5ForConditionalGeneration names; q weights pre-scaled by 1 / sqrt(d_kv) (HF's attention does not scale).  HF has no
    biases and one shared embedding: the caller zeroes the biases and sets dec_shared = shared."""
    sd = {"shared.weight": w["shared"], "encoder.final_layer_norm.weight": w["enc_norm"], "decoder.final_layer_norm.weight": w["dec_norm"],
          "lm_head.weight": w["lm_head"]}
    sd["encoder.embed_tokens.weight"] = sd["decoder.embed_tokens.weight"] = w["shared"]

    def split(m, parts):            # per head [part 0 | part 1 | ...] -> one head-major matrix per part
        return [t.reshape(-1, m.shape[1]) for t in m.view(heads, parts, -1, m.shape[1]).unbind(1)]

    for stack, layers in (("encoder", w["enc"]), ("decoder", w["dec"])):
        for i, p in enumerate(layers):
            pre = "%s.block.%d.layer." % (stack, i)
            q, k, v = split(p["qkv"], 3)
            hn = q.shape[0] // heads
            sd.update({pre + "0.SelfAttention.q.weight": q * hn ** -0.5, pre + "0.SelfAttention.k.weight": k,
                       pre + "0.SelfAttention.v.weight": v, pre + "0.SelfAttention.o.weight": p["dense"],
                       pre + "0.layer_norm.weight": p["ln1"]})
            ff = "2" if stack == "decoder" else "1"
            sd.update({pre + ff + ".DenseReluDense.wi.weight": p["h_to_4h"], pre + ff + ".DenseReluDense.wo.weight": p["4h_to_h"],
                       pre + ff + ".layer_norm.weight": p["ln2"]})
            if stack == "decoder":
                k2, v2 = split(p["kv"], 2)
                sd.update({pre + "1.EncDecAttention.q.weight": p["q"] * hn ** -0.5, pre + "1.EncDecAttention.k.weight": k2,
                           pre + "1.EncDecAttention.v.weight": v2, pre + "1.EncDecAttention.o.weight": p["xdense"],
                           pre + "1.layer_norm.weight": p["lnx"]})
    return sd

"""Single-process restatement of the Llama layer math the reference runtime executes (TEST INFRASTRUCTURE ONLY).

Plain torch, no parallelism, no custom kernels: what one rank of the reference computes when every group has size 1,
which is also what the reference's own GPU tests compare against (an HF model on one rank fed the global batch,
tests/core/test_tp.py:60-121).  Follows, line by line:
  * LlamaModel_sequential.py:45-63   embedding, [b,s,h] -> [s,b,h]
  * LlamaModel_tensor_parallel.py:56-83,95-100   pre-norm residual blocks (flash-attn RMSNorm: fp32 math, one rounding)
  * tensor_parallel/transformer.py:731-767   fused QKV in per-group layout [ng, (np/ng + 2) * hn], split
  * transformer.py:842-848   K/V repeat_interleave to the full head count
  * megatron rotary_pos_embedding.py apply_rotary_pos_emb: t*cos + rotate_half(t)*sin, cos/sin cast to the activation dtype
  * transformer.py:453-509   causal softmax attention (flash-attn there, exact softmax here), scale 1/sqrt(hn)
  * transformer.py:122-124,150-166   swiglu MLP: silu(x[..., :ffn]) * x[..., ffn:]
  * LlamaModel_sequential.py:142-186 + cross_entropy.py:14-100   lm_head, per-token cross entropy
  * hybrid_parallel_model.py:75-79, pipeline.py:919-920   loss = mean over the microbatch's tokens, / real_chunks

``dtype`` = torch.bfloat16 rounds every op's output to bf16 (the reference's mixed-precision numerics: bf16 storage, fp32
accumulate); torch.float32/float64 gives the exact-math answer.  Parity status: PINNED.  The reference ships no golden tensors
(SURVEY 8c), so the pins are outputs of the reference run here: (1) HF ``LlamaForCausalLM`` in fp64 -- the model the reference's own
tests compare with (tests/test_oracle_llama.py: per-token loss 2e-6, gradients 1e-5); (2) the unmodified reference RUNTIME executed on
GPUs under 7 strategies (oracle/ref_runtime/run_ref.py -> tests/golden/ref_runtime/*.json): the host runtime, whose every strategy is
checked against this file, reproduces the reference's losses over 3 Adam steps to 4e-5 and its all-rank gradient norm to 6e-4
(tests/test_ref_runtime_parity.py).
"""
import math

import torch
import torch.nn.functional as F


def _r(x, dtype):
    """Round to the storage dtype, keep computing in fp32/fp64."""
    if dtype in (torch.float32, torch.float64):
        return x.to(dtype)
    return x.to(dtype).float()


def rms_norm(x, w, eps, dtype):
    xf = x.double() if dtype == torch.float64 else x.float()
    y = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps) * w
    return _r(y, dtype)


def rotate_half(x):
    x1, x2 = torch.chunk(x, 2, dim=-1)
    return torch.cat((-x2, x1), dim=-1)


def rope_tables(seq, hn, base, dtype, device):
    inv_freq = 1.0 / (base ** (torch.arange(0, hn, 2, dtype=torch.float32, device=device) / hn))
    freqs = torch.outer(torch.arange(seq, dtype=torch.float32, device=device), inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    cos, sin = torch.cos(emb), torch.sin(emb)
    if dtype not in (torch.float32, torch.float64):
        cos, sin = cos.to(dtype).float(), sin.to(dtype).float()
    return cos[:, None, None, :], sin[:, None, None, :]   # [s, 1, 1, hn]


def attention_block(h, p, cfg, dtype):
    """h [s, b, hidden] -> [s, b, hidden] (pre-norm + attention + residual)."""
    s, b, _ = h.shape
    n_heads, n_groups, hn = cfg["n_heads"], cfg["n_kv_heads"], cfg["head_dim"]
    r = n_heads // n_groups
    x = rms_norm(h, p["ln1"], cfg["eps"], dtype)
    mixed = _r(x @ p["qkv"].t(), dtype).view(s, b, n_groups, (r + 2) * hn)
    q, k, v = torch.split(mixed, [r * hn, hn, hn], dim=3)
    q = q.reshape(s, b, n_heads, hn)
    k = k.repeat_interleave(r, dim=2)
    v = v.repeat_interleave(r, dim=2)
    cos, sin = rope_tables(s, hn, cfg["rope_base"], dtype, h.device)
    q = _r(q * cos + rotate_half(q) * sin, dtype)
    k = _r(k * cos + rotate_half(k) * sin, dtype)
    qb, kb, vb = [t.permute(1, 2, 0, 3) for t in (q, k, v)]               # [b, n, s, hn]
    scores = (qb @ kb.transpose(-1, -2)) / math.sqrt(hn)
    mask = torch.triu(torch.ones(s, s, dtype=torch.bool, device=h.device), diagonal=1)
    scores = scores.masked_fill(mask, float("-inf"))
    ctxt = _r(torch.softmax(scores, dim=-1) @ vb, dtype)                   # [b, n, s, hn]
    ctxt = ctxt.permute(2, 0, 1, 3).reshape(s, b, n_heads * hn)
    out = _r(ctxt @ p["dense"].t(), dtype)
    return _r(out + h, dtype)


def mlp_block(h, p, cfg, dtype):
    x = rms_norm(h, p["ln2"], cfg["eps"], dtype)
    inter = _r(x @ p["h_to_4h"].t(), dtype)
    gate, up = torch.chunk(inter, 2, dim=-1)
    act = _r(F.silu(gate) * up, dtype)
    out = _r(act @ p["4h_to_h"].t(), dtype)
    return _r(out + h, dtype)


def forward_loss(weights, tokens, labels, cfg, dtype=torch.float32):
    """tokens, labels [b, s] -> (per-token loss [b, s], scalar mean).  ``weights``: dict of fp32/fp64 tensors:
    embed [V,h]; layers: list of {ln1, qkv, dense, ln2, h_to_4h, 4h_to_h}; norm [h]; lm_head [V,h]."""
    wd = lambda t: _r(t, dtype) if t.dtype != torch.float64 else t  # noqa: E731  (bf16 copy of the fp32 master)
    h = wd(weights["embed"])[tokens].transpose(0, 1)                        # [s, b, h]
    for p in weights["layers"]:
        p = {k: wd(v) for k, v in p.items()}
        h = attention_block(h, p, cfg, dtype)
        h = mlp_block(h, p, cfg, dtype)
    h = rms_norm(h, wd(weights["norm"]), cfg["eps"], dtype)
    logits = _r(h @ wd(weights["lm_head"]).t(), dtype)                      # [s, b, V]
    tgt = labels.transpose(0, 1)
    loss = F.cross_entropy(logits.reshape(-1, logits.shape[-1]).float() if dtype != torch.float64 else
                           logits.reshape(-1, logits.shape[-1]), tgt.reshape(-1), reduction="none").view(tgt.shape)
    loss = loss.transpose(0, 1)                                             # [b, s]
    return loss, loss.mean()


def init_weights(cfg, seed=0, std=0.02, dtype=torch.float32, device="cpu"):
    g = torch.Generator(device="cpu").manual_seed(seed)
    h, ffn, hn = cfg["hidden"], cfg["ffn"], cfg["head_dim"]
    qkv_rows = (cfg["n_heads"] + 2 * cfg["n_kv_heads"]) * hn
    rnd = lambda *shape: (torch.randn(*shape, generator=g) * std).to(dtype).to(device)  # noqa: E731
    layers = [dict(ln1=torch.ones(h, dtype=dtype, device=device), qkv=rnd(qkv_rows, h), dense=rnd(h, cfg["n_heads"] * hn),
                   ln2=torch.ones(h, dtype=dtype, device=device), h_to_4h=rnd(2 * ffn, h), **{"4h_to_h": rnd(h, ffn)})
              for _ in range(cfg["n_layers"])]
    return dict(embed=rnd(cfg["vocab"], h), layers=layers, norm=torch.ones(h, dtype=dtype, device=device),
                lm_head=rnd(cfg["vocab"], h))


def to_hf_state_dict(weights, cfg):
    """Megatron-layout weights -> HF LlamaForCausalLM state dict (inverse of galvatron/tools/checkpoint_convert_h2g.py:43-82):
    fused per-group QKV -> q/k/v_proj with HF's rotary layout (same half-split convention, no permutation needed), gate|up split."""
    hn, ng, r = cfg["head_dim"], cfg["n_kv_heads"], cfg["n_heads"] // cfg["n_kv_heads"]
    sd = {"model.embed_tokens.weight": weights["embed"], "model.norm.weight": weights["norm"], "lm_head.weight": weights["lm_head"]}
    for i, p in enumerate(weights["layers"]):
        qkv = p["qkv"].view(ng, (r + 2) * hn, -1)
        pre = "model.layers.%d." % i
        sd[pre + "self_attn.q_proj.weight"] = qkv[:, :r * hn].reshape(ng * r * hn, -1)
        sd[pre + "self_attn.k_proj.weight"] = qkv[:, r * hn:(r + 1) * hn].reshape(ng * hn, -1)
        sd[pre + "self_attn.v_proj.weight"] = qkv[:, (r + 1) * hn:].reshape(ng * hn, -1)
        sd[pre + "self_attn.o_proj.weight"] = p["dense"]
        gate, up = torch.chunk(p["h_to_4h"], 2, dim=0)
        sd[pre + "mlp.gate_proj.weight"], sd[pre + "mlp.up_proj.weight"] = gate, up
        sd[pre + "mlp.down_proj.weight"] = p["4h_to_h"]
        sd[pre + "input_layernorm.weight"], sd[pre + "post_attention_layernorm.weight"] = p["ln1"], p["ln2"]
    return sd

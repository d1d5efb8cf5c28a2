"""Restatement of the dropout of the GPT / BERT families (TEST INFRASTRUCTURE ONLY).

* ``philox4x32_10``: Philox4x32-10 in numpy (Salmon et al., SC'11; the generator of curand_philox4x32_x.h).
* ``keep_mask``: the mask definition of include/bg_galvatron.h -- element (token t, sample b, column j) of (seed, iteration, site) is
  kept iff Philox(counter = (j / 4, t, b, iteration), key = (seed, site)).word[j % 4] >= floor(p * 2^32).
* ``dropout_add_ref`` / ``dropout_bwd_ref``: the row kernels' math in torch fp32, in the kernels' operation order (bit-exact).
* ``DropoutOracleBackend``: the CPU (gloo) backend plus the two dropout methods and attention-probability dropout.
* ``gpt_forward_loss`` / ``bert_forward_loss``: the single-process oracle of oracle/gpt_bert_ref.py with the same dropout sites
  (embedding; attention-block output with attention_dropout; MLP-block output; attention probabilities with an explicit mask).
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gpt_bert_ref as ref  # noqa: E402
from oracle.gloo_backend import OracleBackend  # noqa: E402

_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: 4 uint32 arrays (broadcastable), key: 2 uint32 arrays -> 4 uint32 arrays."""
    c0, c1, c2, c3 = [np.asarray(c, dtype=np.uint64) for c in ctr]
    k0, k1 = [np.asarray(k, dtype=np.uint64) for k in key]
    for i in range(10):
        if i:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
    return [c.astype(np.uint32) for c in (c0, c1, c2, c3)]


def threshold(p):
    return int(np.floor(float(p) * 4294967296.0))


def scale(p):
    return np.float32(1.0 / (1.0 - float(p)))


def words(seed, iteration, site, tokens, samples, h):
    """Philox words u [len(tokens), len(samples), h] (uint32) of the given global token positions and sample indices."""
    assert h % 4 == 0
    t = np.asarray(tokens, dtype=np.uint64)[:, None, None]
    b = np.asarray(samples, dtype=np.uint64)[None, :, None]
    j4 = np.arange(h // 4, dtype=np.uint64)[None, None, :]
    out = philox4x32_10((j4, t, b, np.uint64(iteration)), (np.uint64(seed), np.uint64(site)))
    return np.stack(out, axis=-1).reshape(len(tokens), len(samples), h)


def keep_mask(seed, iteration, site, tokens, samples, h, p):
    """bool [T, B, h] (SBH): which elements dropout keeps."""
    return torch.from_numpy(words(seed, iteration, site, tokens, samples, h) >= np.uint32(threshold(p)))


def _f32(v):
    return torch.tensor(float(v), dtype=torch.float32)


def dropout_add_ref(x, bias, residual, keep, p, dtype=torch.bfloat16):
    """residual + keep * scale * (x + bias), fp32 steps in the kernel's order, one rounding each (bias / residual None = 0)."""
    v = x.float() + (bias.float() if bias is not None else torch.zeros((), dtype=torch.float32))
    v = torch.where(keep, v * _f32(scale(p)), torch.zeros((), dtype=torch.float32))
    y = (residual.float() if residual is not None else torch.zeros((), dtype=torch.float32)) + v
    return y.to(dtype) if dtype is not None else y


def dropout_bwd_ref(dy, keep, p):
    """(dx bf16, dbias fp32 column sums of keep * scale * dy)"""
    g = torch.where(keep, dy.float() * _f32(scale(p)), torch.zeros((), dtype=torch.float32))
    return g.to(dy.dtype), g.reshape(-1, g.shape[-1]).sum(0)


class DropoutOracleBackend(OracleBackend):
    """The gloo backend with the dropout methods of ``CudaBackend`` restated on the CPU."""

    def dropout_add_fwd(self, x, bias, residual, p, seed, iteration, site, seq_base, sample_base):
        s, b, h = x.shape
        keep = keep_mask(seed, iteration, site, seq_base + np.arange(s), sample_base + np.arange(b), h, p)
        return dropout_add_ref(x, bias, residual, keep, p, dtype=x.dtype)

    def dropout_bwd(self, dy, p, seed, iteration, site, seq_base, sample_base, with_bias):
        s, b, h = dy.shape
        keep = keep_mask(seed, iteration, site, seq_base + np.arange(s), sample_base + np.arange(b), h, p)
        dx, db = dropout_bwd_ref(dy, keep, p)
        return dx, (db if with_bias else None)

    # attention-probability dropout: a mask from torch's (forked) CPU generator, kept for backward with the probabilities
    def attention_fwd(self, q, k, v, causal, softmax_scale, key_mask=None, dropout_p=0.0):
        out, probs, rng = super().attention_fwd(q, k, v, causal, softmax_scale, key_mask)
        if dropout_p <= 0.0:
            return out, probs, rng
        keep = (torch.rand(probs.shape) >= dropout_p).float() / (1.0 - dropout_p)
        rep = q.shape[2] // k.shape[2]
        vf = v.float().repeat_interleave(rep, 2).transpose(1, 2)
        out = ((probs * keep) @ vf).transpose(1, 2).contiguous().to(q.dtype)
        return out, torch.stack([probs, keep]), rng

    def attention_bwd(self, dout, q, k, v, out, p, causal, softmax_scale, rng, dropout_p=0.0):
        if dropout_p <= 0.0:
            return super().attention_bwd(dout, q, k, v, out, p, causal, softmax_scale, rng)
        probs, keep = p[0], p[1]
        rep = q.shape[2] // k.shape[2]
        b, s, ng, d = k.shape
        qf, kf, vf = q.float(), k.float().repeat_interleave(rep, 2), v.float().repeat_interleave(rep, 2)
        qf, kf, vf, do = [t.transpose(1, 2) for t in (qf, kf, vf, dout.float())]
        dv = (probs * keep).transpose(-1, -2) @ do
        dp = (do @ vf.transpose(-1, -2)) * keep
        ds = probs * (dp - (dp * probs).sum(-1, keepdim=True)) * softmax_scale
        dq = (ds @ kf).transpose(1, 2)
        dk = (ds.transpose(-1, -2) @ qf).transpose(1, 2).reshape(b, s, ng, rep, d).sum(3)
        dv = dv.transpose(1, 2).reshape(b, s, ng, rep, d).sum(3)
        return dq.contiguous().to(q.dtype), dk.contiguous().to(k.dtype), dv.contiguous().to(v.dtype)


# ---- the single-process oracle with dropout ----------------------------------------------------------------------------------
def _site(row, kind):
    return 3 * row + kind


class Drop:
    """Dropout settings of one oracle forward: probabilities, seed, iteration and the global index of the batch's first sample."""

    def __init__(self, hidden=0.0, attention=0.0, seed=1234, iteration=0, sample_base=0, position_shift=0):
        self.hidden, self.attention, self.seed, self.iteration = hidden, attention, seed, iteration
        self.sample_base, self.position_shift = sample_base, position_shift      # (shift: deliberately wrong positions, for tests)

    def apply(self, x, bias, residual, p, site_id, dtype):
        """x [s, b, h] float (bf16 values) -> residual + keep * scale * (x + bias), rounded to ``dtype``."""
        s, b, h = x.shape
        keep = keep_mask(self.seed, self.iteration, site_id, self.position_shift + np.arange(s), self.sample_base + np.arange(b), h, p)
        zero = torch.zeros((), dtype=x.dtype)
        v = torch.where(keep, (x + (bias if bias is not None else zero)) * float(scale(p)), zero)
        return ref._r((residual if residual is not None else zero) + v, dtype)


def _no_bias(p, key):
    return dict(p, **{key: torch.zeros_like(p[key])})


def gpt_forward_loss(weights, tokens, labels, cfg, drop, dtype=torch.bfloat16):
    """oracle/gpt_bert_ref.gpt_forward_loss with dropout at the embedding, attention-block and MLP-block outputs."""
    wd = lambda t: ref._r(t, dtype) if t.dtype != torch.float64 else t  # noqa: E731
    s = tokens.shape[1]
    h = ref._r(wd(weights["wte"])[tokens] + wd(weights["wpe"])[torch.arange(s)][None], dtype).transpose(0, 1)
    if drop.hidden > 0:
        h = drop.apply(h, None, None, drop.hidden, _site(0, 0), dtype)
    for i, lw in enumerate(weights["layers"]):
        p = {k: wd(v) for k, v in lw.items()}
        x = ref.layer_norm(h, p["ln1"], p["ln1_b"], cfg["eps"], dtype)
        if drop.attention > 0:
            h = drop.apply(ref.attention(x, _no_bias(p, "dense_b"), cfg, dtype, True, None), p["dense_b"], h, drop.attention, _site(i + 1, 1), dtype)
        else:
            h = ref._r(ref.attention(x, p, cfg, dtype, True, None) + h, dtype)
        x = ref.layer_norm(h, p["ln2"], p["ln2_b"], cfg["eps"], dtype)
        if drop.hidden > 0:
            h = drop.apply(ref.mlp(x, _no_bias(p, "4h_to_h_b"), cfg, dtype), p["4h_to_h_b"], h, drop.hidden, _site(i + 1, 2), dtype)
        else:
            h = ref._r(ref.mlp(x, p, cfg, dtype) + h, dtype)
    h = ref.layer_norm(h, wd(weights["norm"]), wd(weights["norm_b"]), cfg["eps"], dtype)
    logits = ref._r(h @ wd(weights["lm_head"]).t(), dtype)
    loss = ref._token_loss(logits, labels.transpose(0, 1), dtype).transpose(0, 1)
    return loss, loss.mean()


def bert_forward_loss(weights, tokens, labels, cfg, drop, dtype=torch.bfloat16, attention_mask=None, token_type_ids=None):
    """oracle/gpt_bert_ref.bert_forward_loss with dropout after the embedding LayerNorm and on both sublayer outputs."""
    wd = lambda t: ref._r(t, dtype) if t.dtype != torch.float64 else t  # noqa: E731
    s = tokens.shape[1]
    tt = torch.zeros_like(tokens) if token_type_ids is None else token_type_ids
    e = wd(weights["word"])[tokens] + wd(weights["pos"])[torch.arange(s)][None] + wd(weights["type"])[tt]
    h = ref.layer_norm(ref._r(e, dtype), wd(weights["emb_ln"]), wd(weights["emb_ln_b"]), cfg["eps"], dtype).transpose(0, 1)
    if drop.hidden > 0:
        h = drop.apply(h, None, None, drop.hidden, _site(0, 0), dtype)
    for i, lw in enumerate(weights["layers"]):
        p = {k: wd(v) for k, v in lw.items()}
        if drop.attention > 0:
            a = drop.apply(ref.attention(h, _no_bias(p, "dense_b"), cfg, dtype, False, attention_mask), p["dense_b"], h, drop.attention,
                           _site(i + 1, 1), dtype)
        else:
            a = ref._r(ref.attention(h, p, cfg, dtype, False, attention_mask) + h, dtype)
        h = ref.layer_norm(a, p["ln1"], p["ln1_b"], cfg["eps"], dtype)
        if drop.hidden > 0:
            m = drop.apply(ref.mlp(h, _no_bias(p, "4h_to_h_b"), cfg, dtype), p["4h_to_h_b"], h, drop.hidden, _site(i + 1, 2), dtype)
        else:
            m = ref._r(ref.mlp(h, p, cfg, dtype) + h, dtype)
        h = ref.layer_norm(m, p["ln2"], p["ln2_b"], cfg["eps"], dtype)
    t = ref._r(ref.gelu(ref._r(h @ wd(weights["transform"]).t(), dtype) + wd(weights["transform_b"]), cfg.get("gelu_tanh", True)), dtype)
    t = ref.layer_norm(t, wd(weights["transform_ln"]), wd(weights["transform_ln_b"]), cfg["eps"], dtype)
    logits = ref._r(ref._r(t @ wd(weights["decoder"]).t(), dtype) + wd(weights["decoder_b"]), dtype)
    loss = ref._token_loss(logits, labels.transpose(0, 1), dtype).transpose(0, 1)
    return loss, loss.mean()

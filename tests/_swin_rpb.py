"""The Swin relative-position bias restated for tests (TEST INFRASTRUCTURE ONLY): the oracle model with per-block tables and the CPU
(gloo) backend with the two bias kernels in torch.

Oracle: oracle/swin_ref.py's model, each block optionally with HF's ``relative_position_bias_table`` (weights key ``rpb``,
[(2w-1)^2, heads]): scores = q k^T / sqrt(hn) + table[relative_position_index], then the shift mask, in HF ``SwinSelfAttention``'s
order.  Without ``rpb`` keys the block is swin_ref.block's arithmetic.  Pinned in fp64 to HF ``SwinForImageClassification`` with
non-zero tables by tests/test_swin_rel_bias.py.

Backend: ``SwinRelBiasOracleBackend`` = tests/_swin_backend.SwinOracleBackend (its attention also taking the bias as ``window_bias``)
+ ``swin_rel_bias_fwd`` (the table gathered through the index, rounded to bf16, -inf where the shift mask separates, repeated over
the mb * nW windows) and ``swin_rel_bias_bwd`` (the fp32 sum over windows, added into the table rows through the cell lists)."""
import torch
import torch.nn.functional as F

from _swin_backend import SwinOracleBackend
from oracle import swin_ref as ref
from oracle.swin_ref import _r


def relative_position_index(window):
    """long [L, L], as HF SwinSelfAttention.create_relative_position_index"""
    c = torch.stack(torch.meshgrid(torch.arange(window), torch.arange(window), indexing="ij")).flatten(1)
    rel = (c[:, :, None] - c[:, None, :]).permute(1, 2, 0) + (window - 1)
    return rel[..., 0] * (2 * window - 1) + rel[..., 1]


def block(h, p, st, shifted, cfg, dtype):
    """swin_ref.block (no drop path) with the relative-position bias of p["rpb"] when present"""
    b, res, _, c = h.shape
    heads, ws = st["heads"], st["window"]
    hn, s = c // heads, (st["shift"] if shifted else 0)
    comp = torch.float64 if dtype == torch.float64 else torch.float32
    y = ref.layer_norm(h, p["ln1"], p["ln1_b"], cfg["eps"], dtype)
    qkv = _r(_r(y @ p["qkv"].t(), dtype) + p["qkv_b"], dtype)
    if s:
        qkv = torch.roll(qkv, shifts=(-s, -s), dims=(1, 2))
    win = ref.window_partition(qkv, ws).view(-1, ws * ws, heads, 3, hn).to(comp)
    q, k, v = [win[:, :, :, i].transpose(1, 2) for i in range(3)]
    scores = q @ k.transpose(-1, -2) * hn ** -0.5
    if "rpb" in p:
        idx = relative_position_index(ws).reshape(-1)
        scores = scores + p["rpb"][idx].to(comp).view(ws * ws, ws * ws, heads).permute(2, 0, 1)
    if s:
        mask = ref.hf_shift_mask(res, ws, s).repeat(b, 1, 1)[:, None]
        scores = scores.masked_fill(mask, float("-inf"))
    ctx = _r(torch.softmax(scores, -1) @ v, dtype).transpose(1, 2).reshape(-1, ws * ws, c)
    ctx = ref.window_reverse(ctx, ws, res, res)
    if s:
        ctx = torch.roll(ctx, shifts=(s, s), dims=(1, 2))
    h = _r(_r(ctx @ p["dense"].t() + h, dtype) + p["dense_b"], dtype)
    y = ref.layer_norm(h, p["ln2"], p["ln2_b"], cfg["eps"], dtype)
    a = _r(y @ p["h_to_4h"].t(), dtype)
    g = _r(F.gelu(a + p["h_to_4h_b"], approximate="tanh"), dtype)
    return _r(_r(g @ p["4h_to_h"].t() + h, dtype) + p["4h_to_h_b"], dtype)


def forward_loss(weights, pixels, labels, cfg, dtype=torch.float32):
    """swin_ref.forward_loss (no drop path) through ``block`` above"""
    comp = torch.float64 if dtype == torch.float64 else torch.float32
    wd = lambda t: t if dtype == torch.float64 else _r(t, dtype)  # noqa: E731
    x = _r(ref.patchify(pixels.to(comp), cfg["patch"]), dtype)
    h = ref.layer_norm(_r(x @ wd(weights["patch"]).t(), dtype) + wd(weights["patch_b"]), wd(weights["emb_ln"]), wd(weights["emb_ln_b"]),
                       cfg["eps"], dtype)
    for st, sw in zip(ref.stages_of(cfg), weights["stages"]):
        for j, bw in enumerate(sw["blocks"]):
            h = block(h, {k: wd(v) for k, v in bw.items()}, st, j % 2 == 1, cfg, dtype)
        if sw["merge"] is not None:
            h = ref.merge(h, {k: wd(v) for k, v in sw["merge"].items()}, cfg, dtype)
    h = ref.layer_norm(h, wd(weights["norm"]), wd(weights["norm_b"]), cfg["eps"], dtype)
    pooled = _r(h.reshape(h.shape[0], -1, h.shape[-1]).mean(1), dtype)
    logits = _r(pooled @ wd(weights["classifier"]).t(), dtype)
    loss = F.cross_entropy(logits.to(comp), labels, reduction="none")
    return loss, loss.mean()


def add_tables(w, cfg, seed=0, std=0.02):
    """random non-zero tables [(2w-1)^2, heads] in every block of oracle weights ``w``"""
    g = torch.Generator().manual_seed(seed)
    for st, sw in zip(ref.stages_of(cfg), w["stages"]):
        for bw in sw["blocks"]:
            bw["rpb"] = (torch.randn((2 * st["window"] - 1) ** 2, st["heads"], generator=g) * std).to(bw["qkv"].dtype)
    return w


def to_hf_state_dict(w, cfg):
    """swin_ref.to_hf_state_dict + every block's table"""
    sd = ref.to_hf_state_dict(w, cfg)
    for k, sw in enumerate(w["stages"]):
        for j, bw in enumerate(sw["blocks"]):
            sd["swin.encoder.layers.%d.blocks.%d.attention.self.relative_position_bias_table" % (k, j)] = bw["rpb"]
    return sd


class SwinRelBiasOracleBackend(SwinOracleBackend):
    def attention(self, q, k, v, causal, softmax_scale, key_mask=None, dropout_p=0.0, window_mask=None, window_bias=None):
        mask = window_bias if window_bias is not None else window_mask
        return super().attention(q, k, v, causal, softmax_scale, key_mask, dropout_p, mask)

    def swin_rel_bias_fwd(self, table, index, shift_mask, mb, n_windows, window):
        L = window * window
        b = table[index.long()].to(torch.bfloat16).t().reshape(1, -1, L, L).repeat(n_windows, 1, 1, 1)     # [nW, heads, L, L]
        if shift_mask is not None:
            b = b.masked_fill(shift_mask.bool()[:, None], float("-inf"))
        return b.repeat(mb, 1, 1, 1)

    def swin_rel_bias_bwd(self, dbias, cells, offsets, n_windows, window):
        heads, L = dbias.shape[1], dbias.shape[2]
        g = dbias.float().sum(0).reshape(heads, L * L).t()                                                 # [L * L, heads]
        n_table = offsets.numel() - 1
        entry = torch.repeat_interleave(torch.arange(n_table, device=g.device), (offsets[1:] - offsets[:-1]).long())
        return torch.zeros(n_table, heads, dtype=torch.float32, device=g.device).index_add_(0, entry, g[cells.long()])

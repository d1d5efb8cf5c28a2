"""The CPU (gloo) backend with the Swin methods of ``CudaBackend`` restated in torch (TEST INFRASTRUCTURE ONLY).

``SwinOracleBackend`` extends tests/_vit_backend.ViTOracleBackend (the gloo backend + dropout + the ViT kernels, for the patchify).
Every relayout goes through the same int32 token maps the kernels read, with ``index_select`` / indexing:
  * ``swin_window_qkv_*`` / ``swin_window_merge_*``: SBH rows <-> window rows through map / inv, bias added in fp32, one rounding;
  * ``swin_merge_ln_*``: the r x r gather, + bias, LayerNorm in fp32 (OracleBackend.layernorm_fwd's formula), scattered backward;
  * ``swin_mean_pool_*``: the fp32 mean of the real tokens, and dy / T;
  * ``drop_path_add_*``: the per-sample mask of include/bg_galvatron.h (``drop_path_keep``) in the kernels' operation order;
  * ``attention``: fp32 softmax attention with the additive window mask, differentiable.
"""
import numpy as np
import torch
import torch.nn.functional as F

import _dropout_ref as dref
from _vit_backend import ViTOracleBackend


def drop_path_keep(seed, iteration, site, samples, p):
    """bool [len(samples)]: word 0 of Philox4x32-10((0, 0xffffffff, sample, iteration), (seed, site)) >= floor(p * 2^32)."""
    s = np.asarray(samples, dtype=np.uint64)
    w = dref.philox4x32_10((np.uint64(0), np.uint64(0xFFFFFFFF), s, np.uint64(iteration)), (np.uint64(seed), np.uint64(site)))[0]
    return torch.from_numpy(w >= np.uint32(dref.threshold(p)))


class DropPath:
    """The oracle's drop path: rate, and the masks of one forward at (seed, iteration) for the global batch from sample_base."""

    def __init__(self, rate, seed, iteration=0, sample_base=0):
        self.rate, self.seed, self.iteration, self.sample_base = rate, seed, iteration, sample_base

    def keep(self, site, b):
        return drop_path_keep(self.seed, self.iteration, site, self.sample_base + np.arange(b), self.rate)


def merge_sources(mb, height, width, r, in_bsh):
    """long [T_out, mb, r * r]: the input row of every gathered piece (HF's x0, x1, x2, x3 order for r = 2)."""
    wo = width // r
    to = torch.arange((height // r) * wo)
    io, jo = to // wo, to % wo
    q = torch.arange(r * r)
    ts = (r * io[:, None] + (q & 1)[None]) * width + r * jo[:, None] + (q >> 1)[None]          # [T_out, r*r]
    b = torch.arange(mb)[None, :, None]
    return b * (height * width) + ts[:, None] if in_bsh else ts[:, None] * mb + b


class SwinOracleBackend(ViTOracleBackend):
    def swin_window_qkv_fwd(self, mixed, bias, tmap, inv, n_windows, mb, heads, hn):
        L = tmap.numel() // n_windows
        m = mixed.reshape(-1, mb, heads * 3 * hn).index_select(0, tmap.long())                # [nW * L, mb, 3C] in window order
        m = (m.float() + bias.float()).to(mixed.dtype)
        m = m.view(n_windows, L, mb, heads, 3, hn).permute(2, 0, 1, 3, 4, 5).reshape(mb * n_windows, L, heads, 3, hn)
        return [m[:, :, :, i].contiguous() for i in range(3)]

    def swin_window_qkv_bwd(self, dq, dk, dv, tmap, inv, n_windows, mb, t_run):
        heads, hn = dq.shape[2], dq.shape[3]
        g = torch.stack([dq, dk, dv], dim=3).reshape(mb, -1, heads * 3 * hn).index_select(1, inv.long()).transpose(0, 1)
        db = g.float().reshape(-1, g.shape[-1]).sum(0)
        return F.pad(g, (0, 0, 0, 0, 0, t_run - g.shape[0])).reshape(t_run * mb, -1).contiguous(), db

    def swin_window_merge_fwd(self, windows, tmap, inv, n_windows, mb, t_run):
        c = windows.shape[2] * windows.shape[3]
        rows = windows.reshape(mb, -1, c).index_select(1, inv.long()).transpose(0, 1)
        return F.pad(rows, (0, 0, 0, 0, 0, t_run - rows.shape[0])).contiguous()

    def swin_window_merge_bwd(self, drows, tmap, inv, n_windows, mb, heads, hn):
        g = drows.reshape(-1, mb, heads * hn).index_select(0, tmap.long()).transpose(0, 1)
        return g.reshape(mb * n_windows, -1, heads, hn).contiguous()

    @staticmethod
    def _gathered(x, add_bias, mb, height, width, r, in_bsh):
        idx = merge_sources(mb, height, width, r, in_bsh)
        c = x.shape[-1]
        v = x.reshape(-1, c)[idx.reshape(-1)].reshape(idx.shape[0], mb, r * r * c).float()
        return idx, (v + add_bias.float() if add_bias is not None else v)

    def swin_merge_ln_fwd(self, x, add_bias, weight, bias, eps, mb, height, width, r, in_bsh, t_out_run):
        _, v = self._gathered(x, add_bias, mb, height, width, r, in_bsh)
        mean = v.mean(-1, keepdim=True)
        rstd = torch.rsqrt((v - mean).pow(2).mean(-1, keepdim=True) + eps)
        y = ((v - mean) * rstd * weight.float() + bias.float()).to(x.dtype)
        pad = t_out_run - v.shape[0]
        return (F.pad(y, (0, 0, 0, 0, 0, pad)), F.pad(mean.reshape(-1), (0, pad * mb)), F.pad(rstd.reshape(-1), (0, pad * mb)))

    def swin_merge_ln_bwd(self, dy, x, add_bias, weight, mean, rstd, mb, height, width, r, in_bsh):
        idx, v = self._gathered(x, add_bias, mb, height, width, r, in_bsh)
        n = v.shape[0] * mb
        m, rs = mean[:n].view(v.shape[0], mb, 1), rstd[:n].view(v.shape[0], mb, 1)
        xh = (v - m) * rs
        g = dy.reshape(-1, mb, v.shape[-1])[:v.shape[0]].float()
        gw = g * weight.float()
        dv = rs * (gw - gw.mean(-1, keepdim=True) - xh * (gw * xh).mean(-1, keepdim=True))
        c = x.shape[-1]
        dx = torch.zeros(x.numel() // c, c, dtype=torch.float32)
        dx[idx.reshape(-1)] = dv.reshape(-1, c)
        dab = dv.reshape(-1, dv.shape[-1]).sum(0) if add_bias is not None else None
        return (dx.to(x.dtype).view_as(x), (g * xh).reshape(-1, v.shape[-1]).sum(0).to(weight.dtype),
                g.reshape(-1, v.shape[-1]).sum(0).to(weight.dtype), dab)

    def swin_mean_pool_fwd(self, x, tokens, rows_out):
        y = x[:tokens].float().sum(0) / tokens
        return F.pad(y, (0, 0, 0, rows_out - y.shape[0])).to(x.dtype)

    def swin_mean_pool_bwd(self, dy, tokens, t_run, mb):
        g = (dy[:mb].float() / tokens).to(dy.dtype)
        return F.pad(g.unsqueeze(0).expand(tokens, mb, -1), (0, 0, 0, 0, 0, t_run - tokens)).contiguous()

    def drop_path_add_fwd(self, x, bias, residual, p, seed, iteration, site, sample_base):
        s, b, h = x.shape
        keep = drop_path_keep(seed, iteration, site, sample_base + np.arange(b), p).view(1, b, 1)
        v = x.float() + (bias.float() if bias is not None else 0.0)
        v = torch.where(keep, v * dref._f32(dref.scale(p)), torch.zeros((), dtype=torch.float32))
        return (residual.float() + v).to(x.dtype)

    def drop_path_add_bwd(self, dy, p, seed, iteration, site, sample_base, with_bias):
        s, b, h = dy.shape
        keep = drop_path_keep(seed, iteration, site, sample_base + np.arange(b), p).view(1, b, 1)
        g = torch.where(keep, dy.float() * dref._f32(dref.scale(p)), torch.zeros((), dtype=torch.float32))
        return g.to(dy.dtype), (g.reshape(-1, h).sum(0) if with_bias else None)

    def attention(self, q, k, v, causal, softmax_scale, key_mask=None, dropout_p=0.0, window_mask=None):
        assert not causal and key_mask is None and dropout_p == 0.0
        qf, kf, vf = [t.float().transpose(1, 2) for t in (q, k, v)]
        scores = qf @ kf.transpose(-1, -2) * softmax_scale
        if window_mask is not None:
            scores = scores + window_mask.float()
        return (torch.softmax(scores, -1) @ vf).transpose(1, 2).to(q.dtype)

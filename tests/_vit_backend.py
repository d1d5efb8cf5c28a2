"""The CPU (gloo) backend with the ViT methods of ``CudaBackend`` restated in torch (TEST INFRASTRUCTURE ONLY).

``ViTOracleBackend`` extends tests/_dropout_ref.DropoutOracleBackend (the gloo backend plus the dropout methods), so the embedding's
fused dropout is restated through those dropout methods with the same masks and operation order as the kernels:
  * ``vit_patchify``: einops "b c (h p1) (w p2) -> b (h w) (p1 p2 c)", rounded to bf16, zero rows up to rows_pad;
  * ``vit_embed_fwd`` / ``vit_embed_bwd``: bg_vit_embed_fwd / bg_vit_embed_bwd of include/bg_galvatron.h in fp32;
  * ``bias_tanh_fwd`` / ``bias_tanh_bwd``: tanh(x + b) and dy * (1 - tanh(x + b)^2) in fp32, one rounding.
"""
import torch
import torch.nn.functional as F

from _dropout_ref import DropoutOracleBackend


class ViTOracleBackend(DropoutOracleBackend):
    def bias_tanh_fwd(self, x, bias):
        v = x.float() if bias is None else x.float() + bias.float()
        return torch.tanh(v).to(x.dtype)

    def bias_tanh_bwd(self, dy, x, bias):
        t = torch.tanh(x.float() if bias is None else x.float() + bias.float())
        return (dy.float() * (1 - t * t)).to(x.dtype)

    def vit_patchify(self, pixels, patch, rows_pad):
        b, c, hgt, wid = pixels.shape
        rows = pixels.reshape(b, c, hgt // patch, patch, wid // patch, patch).permute(0, 2, 4, 3, 5, 1)
        rows = rows.reshape(b * (hgt // patch) * (wid // patch), patch * patch * c).to(torch.bfloat16)
        return F.pad(rows, (0, 0, 0, rows_pad - rows.shape[0]))

    def vit_embed_fwd(self, patch_out, bias, cls, pos, batch, s_run, p, seed, iteration, site, sample_base):
        n_patches, h = pos.shape[0] - 1, pos.shape[1]
        y = torch.zeros(s_run, batch, h, dtype=torch.float32)
        posf = pos.float()
        y[0] = posf[0] + cls.float()
        patches = patch_out[:batch * n_patches].float().view(batch, n_patches, h).transpose(0, 1)
        y[1:n_patches + 1] = patches + (posf[1:] + bias.float())[:, None]
        if p > 0.0:         # dropout of the fp32 sums, one rounding after it (dropout_add_fwd keeps an fp32 input in fp32)
            y = self.dropout_add_fwd(y, None, None, p, seed, iteration, site, 0, sample_base)
        return y.to(torch.bfloat16)

    def vit_embed_bwd(self, dy, n_patches, rows_pad, p, seed, iteration, site, sample_base):
        s_run, batch, h = dy.shape
        g = dy.float()
        if p > 0.0:
            g = self.dropout_bwd(g, p, seed, iteration, site, 0, sample_base, False)[0]
        dpos = g[:n_patches + 1].sum(1)
        dpatch = g[1:n_patches + 1].transpose(0, 1).reshape(batch * n_patches, h).to(torch.bfloat16)
        return F.pad(dpatch, (0, 0, 0, rows_pad - dpatch.shape[0])), dpos[0], dpos, dpos[1:].sum(0)

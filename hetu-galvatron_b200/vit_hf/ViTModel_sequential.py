"""Sequential (pipeline-able) view of the ViT model (``galvatron/models/vit_hf/ViTModel_sequential.py``): rows
``['embed'] + ['vit_enc'] * L + ['prenorm', 'cls']``.

The embedding row takes the pixels [B, C, H, W] (fp32 or bf16) as the pipeline's first-stage input and runs three kernels around the
patch GEMM: the patchify relayout, the GEMM (TN; column-parallel over the row's group with the output gathered, as the reference),
and one pass that adds the patch bias, prepends the CLS token, adds the position table, writes the SBH activation with its padding
tokens and applies the embedding dropout.  Backward keeps the pixels, not the patch rows, and patchifies them again for the wgrad GEMM.
The head runs the pooler (GEMM + bias-tanh on the CLS row), the bias-free classifier and the vocabulary-parallel cross entropy."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ..core.runtime.arguments import get_args
from ..core.runtime.backend import get_backend
from ..core.runtime.hybrid_parallel_config import ModelInfo, mixed_precision_dtype
from ..core.runtime.pipeline import PipeSequential
from ..core.runtime.tensor_parallel import linear_with_grad_accumulation_and_async_allreduce, vocab_parallel_cross_entropy
from ..core.runtime.tensor_parallel import random as dropout_random
from ..core.runtime.tensor_parallel.layers import _write_wgrad
from ..core.runtime.tensor_parallel.random import SITE_EMBEDDING, check_probability, site
from .ViTModel_tensor_parallel import ceil8


def _size(g):
    return 1 if g is None else g.size


class _ViTEmbedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pixels, weight, bias, cls, pos, patch, s_run, p, coords, tp_group):
        be = get_backend()
        b, n_patches = pixels.shape[0], pos.shape[0] - 1
        rows_pad = ceil8(b * n_patches)
        seed, iteration, site_id, sample_base = coords
        out = be.gemm(be.vit_patchify(pixels, patch, rows_pad), weight, "tn")            # [rows_pad, h / t]
        if _size(tp_group) > 1:                                                             # gather_output=True
            out = be.all_gather_last_dim(out, tp_group)
            bias = be.all_gather_last_dim(bias.view(1, -1), tp_group).view(-1)
        ctx.save_for_backward(pixels, weight)
        ctx.dims = (patch, n_patches, rows_pad, p, coords, tp_group)
        ctx.dtypes = (bias.dtype, cls.dtype, pos.dtype)
        return be.vit_embed_fwd(out, bias, cls, pos, b, s_run, p, seed, iteration, site_id, sample_base)

    @staticmethod
    def backward(ctx, dy):
        be = get_backend()
        pixels, weight = ctx.saved_tensors
        patch, n_patches, rows_pad, p, (seed, iteration, site_id, sample_base), tp_group = ctx.dims
        dpatch, dcls, dpos, dbias = be.vit_embed_bwd(dy, n_patches, rows_pad, p, seed, iteration, site_id, sample_base)
        if _size(tp_group) > 1:        # this rank's output columns (dy is the whole gradient on every rank of the group)
            n, r = weight.shape[0], tp_group.rank_in_group()
            dpatch, dbias = dpatch[:, r * n:(r + 1) * n].contiguous(), dbias[r * n:(r + 1) * n]
        dw = _write_wgrad(weight, dpatch, be.vit_patchify(pixels, patch, rows_pad))
        bias_dt, cls_dt, pos_dt = ctx.dtypes
        return None, dw, dbias.to(bias_dt), dcls.to(cls_dt), dpos.to(pos_dt), None, None, None, None, None


class ViTEmbeddings_(nn.Module):
    def __init__(self, model):
        super().__init__()
        args, config = get_args(), model.config
        self.embeddings = model.vit.embeddings
        self.tp_group = self.embeddings.tp_group
        self.patch_size, self.seq_run = config.patch_size, config.seq_run
        self.dropout_p = check_probability(getattr(args, "hidden_dropout", 0.0), "hidden_dropout")     # :65

    def forward(self, pixel_values, labels=None, position_ids=None, attention_mask=None):
        e = self.embeddings
        p = self.dropout_p if self.training else 0.0
        ctx = dropout_random.get_context()
        if p > 0.0 and ctx.batch is not None and pixel_values.shape[0] != ctx.batch:
            raise NotImplementedError("dropout: the embedding sees %d samples of a %d-sample microbatch" % (pixel_values.shape[0], ctx.batch))
        coords = (ctx.seed, ctx.iteration, site(0, SITE_EMBEDDING), ctx.sample_base)
        return _ViTEmbedFn.apply(pixel_values, e.weight, e.bias, e.cls_token, e.position_embeddings, self.patch_size, self.seq_run, p,
                                 coords, self.tp_group)


class ViTLayers_(nn.Module):
    def __init__(self, model, layer_idx):
        super().__init__()
        self.layer = model.vit.encoder.layer[layer_idx]

    def forward(self, hidden_states, labels=None, position_ids=None, attention_mask=None):
        # (the key mask of the padding tokens is the layer's own: it depends on the token counts only)
        return self.layer(hidden_states)


class ViTPreNorm_(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.LayerNorm = model.vit.layernorm

    def forward(self, hidden_states, labels=None, position_ids=None, attention_mask=None):
        return self.LayerNorm(hidden_states)


class _BiasTanhFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, bias):
        x = x.contiguous()
        ctx.save_for_backward(x, bias)
        return get_backend().bias_tanh_fwd(x, bias)

    @staticmethod
    def backward(ctx, dy):
        x, bias = ctx.saved_tensors
        dx = get_backend().bias_tanh_bwd(dy.contiguous(), x, bias)
        return dx, dx.reshape(-1, dx.shape[-1]).float().sum(0).to(bias.dtype)


class ViTCls_(nn.Module):
    def __init__(self, model, parallel_loss=True, half_entropy=True):
        super().__init__()
        args = get_args()
        self.pooler, self.classifier = model.vit.pooler, model.classifier
        self.tp_group = self.classifier.tp_group
        self.half_entropy = half_entropy and not args.entropy_in_fp32
        n, n_pad = self.classifier.labels_per_rank, self.classifier.output_size_per_partition
        self.labels_per_rank, self.padded_per_rank = n, n_pad
        self.pad_columns = (torch.arange(n_pad) >= n) if n_pad > n else None

    def forward(self, hidden_states, labels=None, position_ids=None, attention_mask=None):
        b = hidden_states.shape[1]
        x = hidden_states[0]                                                     # the CLS token, [b, h]
        if b % 8:                                                                # GEMM rows: zero tail up to a multiple of 8
            x = F.pad(x, (0, 0, 0, ceil8(b) - b))
        pooled = _BiasTanhFn.apply(linear_with_grad_accumulation_and_async_allreduce(x, self.pooler.weight), self.pooler.bias)
        # the classifier's dgrad is all-reduced over its group inside the linear, so the replicated pooler sees the whole gradient
        logits = linear_with_grad_accumulation_and_async_allreduce(pooled, self.classifier.weight, async_grad_allreduce=True,
                                                                   tp_group=self.tp_group)[:b]
        if self.pad_columns is not None:     # padding classes: -inf, so the softmax runs over the real num_labels classes only
            self.pad_columns = self.pad_columns.to(logits.device)
            logits = logits.masked_fill(self.pad_columns, float("-inf"))
        # class l lives on rank l // n at column l % n of that rank's padded slice
        target = (labels // self.labels_per_rank) * self.padded_per_rank + labels % self.labels_per_rank
        logits_in = logits if self.half_entropy else logits.float()
        loss = vocab_parallel_cross_entropy(logits_in.unsqueeze(0), target.view(1, b), tp_group=self.tp_group)   # [1, b]
        return loss.transpose(0, 1).contiguous()                                 # per-sample loss [b, 1]


def construct_sequential_model(model, config):
    model_ = PipeSequential()
    model_.add_module("embeddings", ViTEmbeddings_(model))
    for i in range(config.num_hidden_layers):
        model_.add_module("layer_%d" % i, ViTLayers_(model, i))
    model_.add_module("prenorm", ViTPreNorm_(model))
    model_.add_module("cls", ViTCls_(model))
    return model_


class ViTModelInfo(ModelInfo):
    def __init__(self, config, args):
        super().__init__()
        seq_len, hidden = config.seq_run, config.hidden_size
        dt = mixed_precision_dtype(args.mixed_precision)
        shape = [[seq_len, -1, hidden]] if args.shape_order == "SBH" else [[-1, seq_len, hidden]]
        self.set_layernums([config.num_hidden_layers])
        self.set_shapes([shape])
        self.set_dtypes([[dt]])
        self.set_module_types(["embed"] + ["vit_enc"] * config.num_hidden_layers + ["prenorm", "cls"])

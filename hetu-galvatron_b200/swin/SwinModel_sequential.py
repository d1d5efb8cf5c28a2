"""Sequential (pipeline-able) view of the Swin model (``galvatron/models/swin/SwinModel_sequential.py``): rows
``['embed'] + per stage (['swin_enc'] * depth + ['swin_downsample'], no downsample after the last) + ['pooler', 'cls']``.

The embedding row takes the pixels [B, C, H, W] (fp32 or bf16): ViT's patchify kernel, the patch GEMM (column-parallel over the
row's group, output gathered), then one pass that adds the patch bias, applies the embedding LayerNorm and writes the SBH activation
with its padding tokens (``bg_swin_merge_ln_fwd`` with r = 1).  Backward keeps the pixels and patchifies them again for the wgrad.
The head runs the final LayerNorm (the ``pooler`` row), the mean over the real tokens, the bias-free classifier and the
vocabulary-parallel cross entropy."""
import torch
import torch.nn as nn

from ..core.runtime.arguments import get_args
from ..core.runtime.backend import get_backend
from ..core.runtime.hybrid_parallel_config import ModelInfo, mixed_precision_dtype
from ..core.runtime.pipeline import PipeSequential
from ..core.runtime.tensor_parallel import linear_with_grad_accumulation_and_async_allreduce, vocab_parallel_cross_entropy
from ..core.runtime.tensor_parallel.layers import _write_wgrad
from .SwinModel_tensor_parallel import ceil8


def _size(g):
    return 1 if g is None else g.size


class _SwinEmbedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pixels, weight, bias, ln_w, ln_b, patch, eps, t_run, tp_group):
        be = get_backend()
        b, side = pixels.shape[0], pixels.shape[2] // patch
        rows_pad = ceil8(b * side * side)
        out = be.gemm(be.vit_patchify(pixels, patch, rows_pad), weight, "tn")             # [rows_pad, C / t], (sample, patch) rows
        if _size(tp_group) > 1:                                                             # gather_output=True
            out = be.all_gather_last_dim(out, tp_group)
            bias = be.all_gather_last_dim(bias.view(1, -1), tp_group).view(-1)
        y, mean, rstd = be.swin_merge_ln_fwd(out, bias, ln_w, ln_b, eps, b, side, side, 1, True, t_run)
        ctx.save_for_backward(pixels, weight, out, bias, ln_w, mean, rstd)
        ctx.dims = (patch, side, rows_pad, tp_group)
        return y

    @staticmethod
    def backward(ctx, dy):
        be = get_backend()
        pixels, weight, out, bias, ln_w, mean, rstd = ctx.saved_tensors
        patch, side, rows_pad, tp_group = ctx.dims
        dout, dln_w, dln_b, dbias = be.swin_merge_ln_bwd(dy, out, bias, ln_w, mean, rstd, pixels.shape[0], side, side, 1, True)
        if _size(tp_group) > 1:        # this rank's output columns (dy is the whole gradient on every rank of the group)
            n, r = weight.shape[0], tp_group.rank_in_group()
            dout, dbias = dout[:, r * n:(r + 1) * n].contiguous(), dbias[r * n:(r + 1) * n]
        dw = _write_wgrad(weight, dout, be.vit_patchify(pixels, patch, rows_pad))
        return None, dw, dbias.to(weight.dtype), dln_w, dln_b, None, None, None, None


class SwinEmbeddings_(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.embeddings = model.swin.embeddings
        self.tp_group = self.embeddings.tp_group
        self.patch_size, self.tokens_run = model.config.patch_size, model.config.tokens_run[0]

    def forward(self, pixel_values, labels=None, position_ids=None, attention_mask=None):
        e = self.embeddings
        return _SwinEmbedFn.apply(pixel_values, e.weight, e.bias, e.norm.weight, e.norm.bias, self.patch_size, e.norm.eps,
                                  self.tokens_run, self.tp_group)


class SwinLayers_(nn.Module):
    def __init__(self, model, stage, block):
        super().__init__()
        self.layer = model.swin.encoder.layers[stage].blocks[block]

    def forward(self, hidden_states, labels=None, position_ids=None, attention_mask=None):
        return self.layer(hidden_states)


class SwinDownsample_(nn.Module):
    def __init__(self, model, stage):
        super().__init__()
        self.downsample = model.swin.encoder.layers[stage].downsample

    def forward(self, hidden_states, labels=None, position_ids=None, attention_mask=None):
        return self.downsample(hidden_states)


class SwinPreNorm_(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.LayerNorm = model.swin.layernorm

    def forward(self, hidden_states, labels=None, position_ids=None, attention_mask=None):
        return self.LayerNorm(hidden_states)


class _MeanPoolFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, tokens, rows_out):
        ctx.dims = (tokens, x.shape[0], x.shape[1])
        return get_backend().swin_mean_pool_fwd(x, tokens, rows_out)

    @staticmethod
    def backward(ctx, dy):
        tokens, t_run, mb = ctx.dims
        return get_backend().swin_mean_pool_bwd(dy, tokens, t_run, mb), None, None


class SwinCls_(nn.Module):
    def __init__(self, model, half_entropy=True):
        super().__init__()
        args = get_args()
        self.classifier = model.classifier
        self.tp_group = self.classifier.tp_group
        self.tokens = model.config.stages[-1]["tokens"]
        self.half_entropy = half_entropy and not args.entropy_in_fp32
        n, n_pad = self.classifier.labels_per_rank, self.classifier.output_size_per_partition
        self.labels_per_rank, self.padded_per_rank = n, n_pad
        self.pad_columns = (torch.arange(n_pad) >= n) if n_pad > n else None

    def forward(self, hidden_states, labels=None, position_ids=None, attention_mask=None):
        b = hidden_states.shape[1]
        pooled = _MeanPoolFn.apply(hidden_states, self.tokens, ceil8(b))        # [ceil8(b), C]: GEMM rows padded with zeros
        logits = linear_with_grad_accumulation_and_async_allreduce(pooled, self.classifier.weight, async_grad_allreduce=True,
                                                                   tp_group=self.tp_group)[:b]
        if self.pad_columns is not None:     # padding classes: -inf, so the softmax runs over the real num_labels classes only
            self.pad_columns = self.pad_columns.to(logits.device)
            logits = logits.masked_fill(self.pad_columns, float("-inf"))
        target = (labels // self.labels_per_rank) * self.padded_per_rank + labels % self.labels_per_rank
        logits_in = logits if self.half_entropy else logits.float()
        loss = vocab_parallel_cross_entropy(logits_in.unsqueeze(0), target.view(1, b), tp_group=self.tp_group)   # [1, b]
        return loss.transpose(0, 1).contiguous()                                 # per-sample loss [b, 1]


def construct_sequential_model(model, config):
    model_ = PipeSequential()
    model_.add_module("embeddings", SwinEmbeddings_(model))
    for k, stage in enumerate(config.stages):
        for j in range(stage["depth"]):
            model_.add_module("encoder_%d_%d" % (k, j), SwinLayers_(model, k, j))
        if k + 1 < len(config.stages):
            model_.add_module("downsample_%d" % k, SwinDownsample_(model, k))
    model_.add_module("pre_norm", SwinPreNorm_(model))
    model_.add_module("cls", SwinCls_(model))
    return model_


class SwinModelInfo(ModelInfo):
    """Four layer types, one per stage: [[tokens_run_k, -1, C_k]] (a downsample row's boundary shape is the next stage's)."""

    def __init__(self, config, args):
        super().__init__()
        dt = mixed_precision_dtype(args.mixed_precision)
        shapes = []
        for stage, t_run in zip(config.stages, config.tokens_run):
            shapes.append([[t_run, -1, stage["width"]]] if args.shape_order == "SBH" else [[-1, t_run, stage["width"]]])
        types_ = ["embed"]
        for k, stage in enumerate(config.stages):
            types_ += ["swin_enc"] * stage["depth"] + (["swin_downsample"] if k + 1 < len(config.stages) else [])
        self.set_layernums([s["depth"] for s in config.stages])
        self.set_shapes(shapes)
        self.set_dtypes([[dt] for _ in config.stages])
        self.set_module_types(types_ + ["pooler", "cls"])

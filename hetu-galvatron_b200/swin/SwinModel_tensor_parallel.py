"""Swin layer classes over the group-explicit parallel ops (``galvatron/models/swin/SwinModel_tensor_parallel.py``): pre-LayerNorm
blocks whose attention runs inside windows (cyclically shifted on every odd block), biases on every projection, tanh-GeLU MLP,
per-sample drop path on the attention branch; a patch-merging row between stages (2x2 neighbourhood -> LayerNorm(4C) -> bias-free
4C -> 2C reduction, column-parallel with the output gathered); the patch embedding with its LayerNorm.

Windows are HF ``SwinLayer``'s: ``roll(-s, -s)`` then contiguous ws x ws windows, window w with window w's shift mask.  Shift,
partition and token padding are one int32 token map per layer shape (``token_map``): the QKV relayout writes q, k, v straight into
window order and the merge kernel writes the attention output back into token rows, so no activation is rolled, permuted or copied
in torch.  There is no relative-position bias by default (the reference's attention has none); the ``relative_position_bias``
spec key gives every block HF's learned table (``SwinAttention_tp``), turned into the attention's additive mask by
``bg_swin_rel_bias_fwd`` and its gradient folded back into the table by ``bg_swin_rel_bias_bwd``.

Token padding: stage k runs ``config.tokens_run[k]`` tokens, the real ones followed by rows no kernel reads as input (the window
relayout, the patch merge and the mean-pool address real tokens only), so their gradient is exactly zero
(``SwinModel_hybrid_parallel``)."""
import functools
import types

import torch
from torch import nn

from ..core.runtime.arguments import get_args
from ..core.runtime.backend import get_backend
from ..core.runtime.tensor_parallel import ColumnParallelLinear, LayerNorm, ParallelMLP
from ..core.runtime.tensor_parallel import random as dropout_random
from ..core.runtime.tensor_parallel.layers import RowParallelLinear, mark_tensor_parallel
from ..core.runtime.tensor_parallel.random import SITE_DROP_PATH, check_probability, site
from ..core.runtime.tensor_parallel.transformer import _attention
from ..gpt_hf.GPTModel_tensor_parallel import core_transformer_config_from_args


def _size(g):
    return 1 if g is None else g.size


def ceil8(n):
    return (int(n) + 7) // 8 * 8


def token_map(res, window, shift):
    """int64 [nW * ws * ws]: entry w * ws^2 + i is the token (row-major on the res x res grid) at position i of window w after
    HF's roll(-shift, -shift) and window partition."""
    nw = res // window
    wh, ww, ih, iw = torch.meshgrid(torch.arange(nw), torch.arange(nw), torch.arange(window), torch.arange(window), indexing="ij")
    return (((wh * window + ih + shift) % res) * res + (ww * window + iw + shift) % res).reshape(-1)


def shift_mask(res, window, shift):
    """bool [nW, ws^2, ws^2], True where HF ``SwinLayer.get_attn_mask`` is non-zero (query and key come from different regions of
    the rolled grid); None when nothing is shifted."""
    if shift == 0:
        return None
    nw = res // window
    y = torch.arange(res)
    region = torch.where(y < res - window, 0, torch.where(y < res - shift, 1, 2))
    label = (region[:, None] * 3 + region[None, :]).reshape(nw, window, nw, window).permute(0, 2, 1, 3).reshape(nw * nw, -1)
    return label[:, :, None] != label[:, None, :]


def relative_position_index(window):
    """int64 [L * L]: HF ``SwinSelfAttention.create_relative_position_index`` flattened -- entry i * L + j is the table row of query
    i and key j, (dy + w - 1) * (2w - 1) + dx + w - 1 for their offset (dy, dx) in the window."""
    c = torch.stack(torch.meshgrid(torch.arange(window), torch.arange(window), indexing="ij")).flatten(1)
    rel = c[:, :, None] - c[:, None, :] + (window - 1)
    return (rel[0] * (2 * window - 1) + rel[1]).reshape(-1)


class WindowLayout:
    """The token map of one (resolution, window, shift), its inverse and the additive shift mask, on each device once; the mask is
    expanded to mb * nW windows and cached per (mb, device, dtype), as ``_KeyMask`` caches.  One instance per layer shape, shared by
    every block of that shape (``window_layout``).  The expanded mask is materialised: its window axis is b * nW + w, which no
    broadcast view of the [nW, L, L] mask expresses.  With the relative-position bias, ``rel_maps`` holds what its kernels read:
    the index, the shift mask as bytes, and the index's cells grouped by table entry (cells, offsets)."""

    def __init__(self, res, window, shift):
        self.res, self.window, self.shift = res, window, shift
        self.n_windows = (res // window) ** 2
        self.tokens = res * res
        m = token_map(res, window, shift)
        self._map, self._inv = m.to(torch.int32), torch.argsort(m).to(torch.int32)
        self._mask = shift_mask(res, window, shift)
        self._dev, self._masks, self._rel = {}, {}, {}

    def maps(self, device):
        key = str(device)
        if key not in self._dev:
            self._dev[key] = (self._map.to(device), self._inv.to(device))
        return self._dev[key]

    def rel_maps(self, device):
        """(index int32 [L * L], shift mask uint8 [nW, L, L] or None, cells int32 [L * L] = the stable argsort of the index,
        offsets int32 [(2w-1)^2 + 1]: entry t's cells are cells[offsets[t]:offsets[t + 1]], ascending) on ``device``."""
        key = str(device)
        if key not in self._rel:
            index = relative_position_index(self.window)
            counts = torch.bincount(index, minlength=(2 * self.window - 1) ** 2)
            offsets = torch.cat([torch.zeros(1, dtype=torch.int64), counts.cumsum(0)])
            cells = torch.argsort(index, stable=True)
            mask = self._mask.to(torch.uint8) if self._mask is not None else None
            self._rel[key] = tuple(t.to(device) if t is not None else None for t in
                                   (index.to(torch.int32), mask, cells.to(torch.int32), offsets.to(torch.int32)))
        return self._rel[key]

    def attn_mask(self, mb, device, dtype):
        if self._mask is None:
            return None
        key = (mb, str(device), dtype)
        if key not in self._masks:
            bias = torch.zeros(self._mask.shape, dtype=dtype).masked_fill_(self._mask, float("-inf"))
            self._masks[key] = bias.to(device).unsqueeze(1).repeat(mb, 1, 1, 1)          # [mb * nW, 1, L, L], window b * nW + w
        return self._masks[key]


@functools.lru_cache(maxsize=None)
def window_layout(res, window, shift):
    return WindowLayout(res, window, shift)


class _WindowQkvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mixed, bias, layout, heads, hn):
        t_run, mb = mixed.shape[0], mixed.shape[1]
        tmap, inv = layout.maps(mixed.device)
        ctx.dims = (layout, mb, t_run, bias.dtype)
        return tuple(get_backend().swin_window_qkv_fwd(mixed.contiguous(), bias, tmap, inv, layout.n_windows, mb, heads, hn))

    @staticmethod
    def backward(ctx, dq, dk, dv):
        layout, mb, t_run, bias_dt = ctx.dims
        tmap, inv = layout.maps(dq.device)
        dmixed, dbias = get_backend().swin_window_qkv_bwd(dq, dk, dv, tmap, inv, layout.n_windows, mb, t_run)
        return dmixed.view(t_run, mb, -1), dbias.to(bias_dt), None, None, None


class _WindowMergeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, windows, layout, mb, t_run):
        tmap, inv = layout.maps(windows.device)
        ctx.dims = (layout, mb, windows.shape[2], windows.shape[3])
        return get_backend().swin_window_merge_fwd(windows, tmap, inv, layout.n_windows, mb, t_run)

    @staticmethod
    def backward(ctx, drows):
        layout, mb, heads, hn = ctx.dims
        tmap, inv = layout.maps(drows.device)
        return get_backend().swin_window_merge_bwd(drows, tmap, inv, layout.n_windows, mb, heads, hn), None, None, None


class _RelBiasFn(torch.autograd.Function):
    """The block's relative-position table -> its additive attention mask [mb * nW, heads, L, L] (bias + shift mask), and the
    mask's gradient -> the table's."""

    @staticmethod
    def forward(ctx, table, layout, mb):
        index, mask, _, _ = layout.rel_maps(table.device)
        ctx.dims = (layout, table.dtype)
        return get_backend().swin_rel_bias_fwd(table, index, mask, mb, layout.n_windows, layout.window)

    @staticmethod
    def backward(ctx, dbias):
        layout, dt = ctx.dims
        _, _, cells, offsets = layout.rel_maps(dbias.device)
        return get_backend().swin_rel_bias_bwd(dbias, cells, offsets, layout.n_windows, layout.window).to(dt), None, None


class _MergeLnFn(torch.autograd.Function):
    """Gather r x r neighbourhoods (r = 2: patch merging; r = 1: identity) + optional bias, then LayerNorm, into SBH rows."""

    @staticmethod
    def forward(ctx, x, add_bias, weight, bias, eps, mb, res, r, in_bsh, t_out_run):
        y, mean, rstd = get_backend().swin_merge_ln_fwd(x, add_bias, weight, bias, eps, mb, res, res, r, in_bsh, t_out_run)
        ctx.save_for_backward(x, add_bias, weight, mean, rstd)
        ctx.dims = (mb, res, r, in_bsh, add_bias is not None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, add_bias, weight, mean, rstd = ctx.saved_tensors
        mb, res, r, in_bsh, has_bias = ctx.dims
        dx, dw, db, dab = get_backend().swin_merge_ln_bwd(dy, x, add_bias if has_bias else None, weight, mean, rstd, mb, res, res, r,
                                                          in_bsh)
        return dx, (dab.to(add_bias.dtype) if has_bias else None), dw, db, None, None, None, None, None, None


class _DropPathFn(torch.autograd.Function):
    """y = residual + keep_b * scale * (x + bias), the per-sample mask regenerated in backward from (seed, site, iteration, sample)."""

    @staticmethod
    def forward(ctx, x, bias, residual, p, site_id):
        c = dropout_random.get_context()
        ctx.coords = (p, c.seed, c.iteration, site_id, c.sample_base)
        ctx.bias_dtype = bias.dtype
        return get_backend().drop_path_add_fwd(x, bias, residual, p, c.seed, c.iteration, site_id, c.sample_base)

    @staticmethod
    def backward(ctx, dy):
        p, seed, iteration, site_id, sample_base = ctx.coords
        dx, dbias = get_backend().drop_path_add_bwd(dy, p, seed, iteration, site_id, sample_base, True)
        return dx, dbias.to(ctx.bias_dtype), dy, None, None


def stage_config(mconf, stage):
    """The block config of one stage: width C_k, heads, 4 C_k MLP."""
    c, heads = stage["width"], stage["heads"]
    return types.SimpleNamespace(**dict(vars(mconf), hidden_size=c, ffn_hidden_size=4 * c, num_attention_heads=heads,
                                        num_query_groups=heads, kv_channels=c // heads))


class SwinAttention_tp(nn.Module):
    """QKV (column-parallel, bias added by the window relayout) -> window attention -> merge to token rows -> projection
    (row-parallel; + residual in its epilogue, or the drop path kernel).

    With ``window`` (the relative-position bias): HF's ``relative_position_bias_table`` [(2w-1)^2, heads], split by heads over the
    tensor-parallel group as the QKV projection is.  Its init is the original Swin's, truncated normal with std 0.02, drawn for the
    whole table from a generator seeded by (seed, layer) so that every tensor-parallel layout holds slices of one table."""

    def __init__(self, mconf, tp_group, window=None, layer_number=0):
        super().__init__()
        t = _size(tp_group)
        heads, c = mconf.num_attention_heads, mconf.hidden_size
        if heads % t:
            raise ValueError("Swin: %d heads are not divisible by the tensor-parallel degree %d" % (heads, t))
        self.heads_local, self.hn = heads // t, c // heads
        self.query_key_value = ColumnParallelLinear(c, 3 * c, config=mconf, bias=True, gather_output=False, skip_bias_add=True,
                                                    tp_group=tp_group, device="meta")
        self.dense = RowParallelLinear(c, c, config=mconf, bias=True, skip_bias_add=True, input_is_parallel=True, tp_group=tp_group,
                                       device="meta")
        self.scale = self.hn ** -0.5
        self.tp_group, self.layer_number = tp_group, layer_number
        if window is not None:
            self.relative_position_bias_table = nn.Parameter(torch.empty((2 * window - 1) ** 2, self.heads_local, device="meta"))
        else:
            self.relative_position_bias_table = None

    def reset_parameters(self):
        table = self.relative_position_bias_table
        if table is None:
            return
        heads = table.shape[1] * _size(self.tp_group)
        g = torch.Generator().manual_seed(get_args().seed * 1000003 + self.layer_number)
        full = nn.init.trunc_normal_(torch.empty(table.shape[0], heads), std=0.02, generator=g)
        r = self.tp_group.rank_in_group() if _size(self.tp_group) > 1 else 0
        with torch.no_grad():
            table.copy_(full[:, r * table.shape[1]:(r + 1) * table.shape[1]])
        mark_tensor_parallel(table)


class SwinBlock_tp(nn.Module):
    def __init__(self, config, stage, layer_number, shifted, tp_group=None):
        super().__init__()
        args = get_args()
        mconf = stage_config(core_transformer_config_from_args(args), stage)
        self.tp_group = tp_group.group if tp_group is not None else None
        c = stage["width"]
        self.layernorm_before = LayerNorm(c, eps=config.layer_norm_eps, device="meta")
        self.attention = SwinAttention_tp(mconf, self.tp_group, stage["window"] if config.relative_position_bias else None,
                                          layer_number)
        self.layernorm_after = LayerNorm(c, eps=config.layer_norm_eps, device="meta")
        self.mlp = ParallelMLP(mconf, tp_group=self.tp_group, device="meta")
        self.layout = window_layout(stage["res"], stage["window"], stage["shift"] if shifted else 0)
        self.drop_path = check_probability(getattr(args, "drop_path_rate", 0.0), "drop_path_rate")
        self.site = site(layer_number + 1, SITE_DROP_PATH)
        self.idx = layer_number

    def forward(self, hidden_states, attention_mask=None):
        a, mb = self.attention, hidden_states.shape[1]
        residual = hidden_states
        mixed, qkv_bias = a.query_key_value(self.layernorm_before(hidden_states))              # [t_run, mb, 3 C / t]
        q, k, v = _WindowQkvFn.apply(mixed, qkv_bias, self.layout, a.heads_local, a.hn)       # [mb * nW, L, heads / t, hn]
        if a.relative_position_bias_table is not None:
            bias = _RelBiasFn.apply(a.relative_position_bias_table, self.layout, mb)    # [mb * nW, heads / t, L, L]
            ctxt = get_backend().attention(q, k, v, False, a.scale, window_bias=bias)
        else:
            mask = self.layout.attn_mask(mb, q.device, q.dtype)
            if mask is None:
                ctxt = _attention(q, k, v, False, a.scale)
            else:
                ctxt = get_backend().attention(q, k, v, False, a.scale, window_mask=mask)
        ctxt = _WindowMergeFn.apply(ctxt, self.layout, mb, hidden_states.shape[0])            # [t_run, mb, C / t]
        if self.drop_path > 0.0 and self.training:
            batch = dropout_random.get_context().batch
            if batch is not None and mb != batch:       # (swin_model_hp refuses such strategies; this guards the sample coordinates)
                raise NotImplementedError("drop path: a block sees %d samples of a %d-sample microbatch (a relocation that re-splits "
                                          "the batch is not supported with drop path)" % (mb, batch))
            out, bias = a.dense(ctxt)
            hidden_states = _DropPathFn.apply(out, bias, residual, self.drop_path, self.site)
        else:
            out, bias = a.dense(ctxt, residual=residual)                                      # + residual in the GEMM epilogue
            hidden_states = out + bias
        out, bias = self.mlp(self.layernorm_after(hidden_states), residual=hidden_states)
        return out + bias


class SwinDownsample_tp(nn.Module):
    """Patch merging (HF ``SwinPatchMerging``): 2x2 neighbourhood -> LayerNorm(4C) -> bias-free 4C -> 2C reduction, column-parallel
    over the row's group with the output gathered (the reference's ``ColumnParallelLinear(gather_output=True)``)."""

    def __init__(self, config, stage, next_tokens_run, tp_group=None):
        super().__init__()
        mconf = core_transformer_config_from_args(get_args())
        c = stage["width"]
        self.res, self.tokens_out_run = stage["res"], next_tokens_run
        self.layernorm = LayerNorm(4 * c, eps=config.layer_norm_eps, device="meta")
        self.reduction = ColumnParallelLinear(4 * c, 2 * c, config=mconf, bias=False, gather_output=True,
                                              tp_group=tp_group.group if tp_group is not None else None, device="meta")

    def forward(self, hidden_states):
        ln = self.layernorm
        y = _MergeLnFn.apply(hidden_states, None, ln.weight, ln.bias, ln.eps, hidden_states.shape[1], self.res, 2, False,
                             self.tokens_out_run)
        return self.reduction(y)[0]


class SwinPatchEmbedding(nn.Module):
    """The embedding row's parameters: the patch projection (column-parallel with gathered output, as the reference) and its
    LayerNorm (HF ``SwinEmbeddings.norm``)."""

    def __init__(self, config, tp_group):
        super().__init__()
        t = _size(tp_group)
        c, k = config.embed_dim, config.patch_size * config.patch_size * config.num_channels
        if c % t:
            raise ValueError("Swin: embed_dim %d is not divisible by the embedding's tensor-parallel degree %d" % (c, t))
        self.tp_group = tp_group
        self.weight = nn.Parameter(torch.empty(c // t, k, device="meta"))
        self.bias = nn.Parameter(torch.empty(c // t, device="meta"))
        self.norm = LayerNorm(c, eps=config.layer_norm_eps, device="meta")
        self.init_std = get_args().init_method_std

    def reset_parameters(self):
        nn.init.normal_(self.weight, mean=0.0, std=self.init_std)
        nn.init.zeros_(self.bias)
        mark_tensor_parallel(self.weight)
        mark_tensor_parallel(self.bias)


class SwinClassifier(ColumnParallelLinear):
    """The classifier, column-parallel over the classes with no bias (the reference creates one and never adds it).  Each rank's
    slice of num_labels / t classes is padded to a multiple of 8 rows that stay zero."""

    def __init__(self, config, mconf, tp_group):
        t = _size(tp_group)
        if config.num_labels % t:
            raise ValueError("Swin: num_labels %d is not divisible by the classifier's tensor-parallel degree %d" % (config.num_labels, t))
        width = config.stages[-1]["width"]
        super().__init__(width, t * ceil8(config.num_labels // t), config=mconf, bias=False, tp_group=tp_group, device="meta")
        self.labels_per_rank = config.num_labels // t

    def reset_parameters(self):
        super().reset_parameters()
        with torch.no_grad():
            self.weight[self.labels_per_rank:].zero_()


class SwinSkeleton(nn.Module):
    """Container with the attribute layout of HF ``SwinForImageClassification`` (``.swin.embeddings``, ``.swin.encoder.layers[k]
    .blocks`` / ``.downsample``, ``.swin.layernorm``, ``.classifier``); created empty -- ``construct_tensor_parallel_model`` builds
    every layer."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.swin = nn.Module()
        self.swin.encoder = nn.Module()
        self.swin.encoder.layers = nn.ModuleList()
        self.swin.embeddings = self.swin.layernorm = self.classifier = None


def construct_tensor_parallel_model(model, config, tp_groups_whole, sp_groups_whole):
    """Whole-model rows: [embed, (swin_enc x depth_k, swin_downsample) per stage (no downsample after the last), pooler, cls]."""
    mconf = core_transformer_config_from_args(get_args())
    row, layer_number = 1, 0
    stages = nn.ModuleList()
    for k, stage in enumerate(config.stages):
        st = nn.Module()
        blocks = []
        for j in range(stage["depth"]):
            blocks.append(SwinBlock_tp(config, stage, layer_number, j % 2 == 1, tp_group=tp_groups_whole[row]))
            row, layer_number = row + 1, layer_number + 1
        st.blocks = nn.ModuleList(blocks)
        st.downsample = None
        if k + 1 < len(config.stages):
            st.downsample = SwinDownsample_tp(config, stage, config.tokens_run[k + 1], tp_group=tp_groups_whole[row])
            row += 1
        stages.append(st)
    model.swin.encoder.layers = stages
    model.swin.embeddings = SwinPatchEmbedding(config, tp_groups_whole[0].group)
    model.swin.layernorm = LayerNorm(config.stages[-1]["width"], eps=config.layer_norm_eps, device="meta")
    model.classifier = SwinClassifier(config, mconf, tp_groups_whole[-1].group)
    return model

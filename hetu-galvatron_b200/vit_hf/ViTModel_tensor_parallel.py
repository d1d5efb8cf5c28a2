"""ViT layer classes over the group-explicit parallel ops (``galvatron/models/vit_hf/ViTModel_tensor_parallel.py``): PRE-LayerNorm
encoder blocks, bidirectional attention (``AttnMaskType.padding``), biases on every projection, tanh-GeLU MLP, hidden dropout on
both block outputs.

Token padding: a layer runs ``config.seq_run`` tokens, the image's P + 1 real ones followed by zero rows when the real count times a
micro-batch is not a multiple of 8 (the GEMMs' granule; ``ViTModel_hybrid_parallel.token_rows``).  The padding tokens are masked out as
KEYS, so no real token ever reads them; as queries they compute rows nothing downstream reads, so their gradient is exactly zero."""
import torch
from torch import nn

from ..core.runtime.arguments import get_args
from ..core.runtime.tensor_parallel import AttnMaskType, AttnType, ColumnParallelLinear, LayerNorm, ParallelAttention, ParallelMLP
from ..core.runtime.tensor_parallel.layers import mark_tensor_parallel
from ..core.runtime.tensor_parallel.random import SITE_ATTENTION, SITE_MLP, bias_dropout_add, site
from ..gpt_hf.GPTModel_tensor_parallel import core_transformer_config_from_args


def _size(g):
    return 1 if g is None else g.size


def ceil8(n):
    return (int(n) + 7) // 8 * 8


class _KeyMask:
    """[b, seq_run] bool key mask, True for the real tokens; None when the layer runs no padding tokens."""

    def __init__(self, config):
        self.real, self.run = config.seq_length, config.seq_run
        self._cache = {}

    def __call__(self, hidden_states):
        if self.run == self.real:
            return None
        b, dev = hidden_states.shape[1], hidden_states.device
        key = (b, str(dev))
        if key not in self._cache:
            self._cache[key] = (torch.arange(self.run, device=dev) < self.real).unsqueeze(0).expand(b, self.run).contiguous()
        return self._cache[key]


class ViTAttention_tp(nn.Module):
    def __init__(self, config, layer_number, tp_group=None, sp_group=None):
        super().__init__()
        mconf = core_transformer_config_from_args(get_args())
        self.tp_group = tp_group.group if tp_group is not None else None
        self.attention = ParallelAttention(mconf, layer_number, attention_type=AttnType.self_attn, attn_mask_type=AttnMaskType.padding,
                                           tp_group=self.tp_group, device="meta")
        self.LayerNorm = LayerNorm(config.hidden_size, eps=config.layer_norm_eps, device="meta")
        # the reference drops the attention-block output with hidden_dropout_prob (:43-50)
        self.dropout_p, self.site = mconf.hidden_dropout, site(layer_number + 1, SITE_ATTENTION)
        self.key_mask = _KeyMask(config)

    def forward(self, hidden_states, attention_mask=None):
        residual = hidden_states
        x = self.LayerNorm(hidden_states)
        mask = self.key_mask(hidden_states)
        if self.dropout_p > 0.0 and self.training:
            out, bias = self.attention(x, mask)
            return bias_dropout_add(out, bias, residual, self.dropout_p, self.site)
        out, bias = self.attention(x, mask, residual=residual)            # + residual in the projection GEMM's epilogue
        return out if bias is None else out + bias


class ViTMLP_tp(nn.Module):
    def __init__(self, config, tp_group=None, layer_number=0):
        super().__init__()
        mconf = core_transformer_config_from_args(get_args())
        self.tp_group = tp_group.group if tp_group is not None else None
        self.mlp = ParallelMLP(mconf, tp_group=self.tp_group, device="meta")
        self.LayerNorm = LayerNorm(config.hidden_size, eps=config.layer_norm_eps, device="meta")
        self.dropout_p, self.site = mconf.hidden_dropout, site(layer_number + 1, SITE_MLP)      # :61-69

    def forward(self, hidden_states):
        residual = hidden_states
        x = self.LayerNorm(hidden_states)
        if self.dropout_p > 0.0 and self.training:
            out, bias = self.mlp(x)
            return bias_dropout_add(out, bias, residual, self.dropout_p, self.site)
        out, bias = self.mlp(x, residual=residual)
        return out if bias is None else out + bias


class ViTLayer_tp(nn.Module):
    def __init__(self, config, layer_number, tp_group=None, sp_group=None):
        super().__init__()
        self.attention = ViTAttention_tp(config, layer_number, tp_group, sp_group)
        self.mlp = ViTMLP_tp(config, tp_group, layer_number)
        self.idx = layer_number

    def forward(self, hidden_states, attention_mask=None):
        return self.mlp(self.attention(hidden_states, attention_mask))


class ViTPatchEmbedding(nn.Module):
    """The embedding row's parameters: the patch projection (column-parallel over the row's tensor-parallel group, gathered
    output, as the reference's ``ColumnParallelLinear(p*p*C -> h, gather_output=True)``), the CLS token and the position table."""

    def __init__(self, config, tp_group):
        super().__init__()
        t = _size(tp_group)
        h, k = config.hidden_size, config.patch_size * config.patch_size * config.num_channels
        if h % t:
            raise ValueError("ViT: hidden size %d is not divisible by the embedding's tensor-parallel degree %d" % (h, t))
        self.tp_group = tp_group
        self.weight = nn.Parameter(torch.empty(h // t, k, device="meta"))
        self.bias = nn.Parameter(torch.empty(h // t, device="meta"))
        self.cls_token = nn.Parameter(torch.empty(h, device="meta"))
        self.position_embeddings = nn.Parameter(torch.empty(config.seq_length, h, device="meta"))
        self.init_std = get_args().init_method_std

    def reset_parameters(self):
        for p in (self.weight, self.cls_token, self.position_embeddings):
            nn.init.normal_(p, mean=0.0, std=self.init_std)
        nn.init.zeros_(self.bias)
        mark_tensor_parallel(self.weight)
        mark_tensor_parallel(self.bias)


class ViTPooler(nn.Module):
    """The pooler the reference adds to HF's ViT (``vit_model_hp``): dense + tanh on the CLS token, replicated."""

    def __init__(self, config):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(config.hidden_size, config.hidden_size, device="meta"))
        self.bias = nn.Parameter(torch.empty(config.hidden_size, device="meta"))
        self.init_std = get_args().init_method_std

    def reset_parameters(self):
        nn.init.normal_(self.weight, mean=0.0, std=self.init_std)
        nn.init.zeros_(self.bias)


class ViTClassifier(ColumnParallelLinear):
    """The classifier, column-parallel over the classes with no bias (the reference creates one and never adds it, ViTLoss_).  Each
    rank's slice of num_labels / t classes is padded to a multiple of 8 rows; the padding rows stay zero (they get no gradient)."""

    def __init__(self, config, mconf, tp_group):
        t = _size(tp_group)
        if config.num_labels % t:
            raise ValueError("ViT: num_labels %d is not divisible by the classifier's tensor-parallel degree %d" % (config.num_labels, t))
        super().__init__(config.hidden_size, t * ceil8(config.num_labels // t), config=mconf, bias=False, tp_group=tp_group, device="meta")
        self.labels_per_rank = config.num_labels // t

    def reset_parameters(self):
        super().reset_parameters()
        with torch.no_grad():
            self.weight[self.labels_per_rank:].zero_()


class ViTSkeleton(nn.Module):
    """Container with the attribute layout of HF ``ViTForImageClassification`` plus the reference's pooler (``.vit.embeddings``,
    ``.vit.encoder.layer``, ``.vit.layernorm``, ``.vit.pooler``, ``.classifier``); created empty -- every real layer is built by
    ``construct_tensor_parallel_model``."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.vit = nn.Module()
        self.vit.encoder = nn.Module()
        self.vit.encoder.layer = nn.ModuleList()
        self.vit.embeddings = self.vit.layernorm = self.vit.pooler = self.classifier = None


def construct_tensor_parallel_model(model, config, tp_groups_enc, sp_groups_enc):
    """Whole-model rows: [embed, layer_0..L-1, prenorm, cls] (ViTModel_tensor_parallel.py:90-145; 4-argument callback)."""
    mconf = core_transformer_config_from_args(get_args())
    model.vit.encoder.layer = nn.ModuleList([ViTLayer_tp(config, i, tp_group=tp_groups_enc[i + 1], sp_group=sp_groups_enc[i + 1])
                                             for i in range(config.num_hidden_layers)])
    model.vit.embeddings = ViTPatchEmbedding(config, tp_groups_enc[0].group)
    model.vit.layernorm = LayerNorm(config.hidden_size, eps=config.layer_norm_eps, device="meta")
    model.vit.pooler = ViTPooler(config)
    model.classifier = ViTClassifier(config, mconf, tp_groups_enc[-1].group)
    return model

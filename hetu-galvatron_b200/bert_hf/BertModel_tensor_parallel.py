"""BERT layer classes over the group-explicit parallel ops (``galvatron/models/bert_hf/BertModel_tensor_parallel.py``):
POST-LayerNorm encoder blocks, bidirectional attention under a key padding mask, biases on every projection, GeLU MLP."""
import torch
from torch import nn

from ..core.runtime.arguments import get_args
from ..core.runtime.tensor_parallel import (AttnMaskType, AttnType, ColumnParallelLinear, LayerNorm, ParallelAttention, ParallelMLP,
                                            VocabParallelEmbedding)
from ..core.runtime.tensor_parallel.random import SITE_ATTENTION, SITE_MLP, bias_dropout_add, site
from ..gpt_hf.GPTModel_tensor_parallel import _megatron_sp, _seq_rank, core_transformer_config_from_args


class BertAttention_tp(nn.Module):
    def __init__(self, config, layer_number, tp_group=None, sp_group=None):
        super().__init__()
        args = get_args()
        self.use_ulysses = sp_group is not None and sp_group.size > 1
        mconf = core_transformer_config_from_args(args)
        self.tp_group = tp_group.group if tp_group is not None else None
        self.sp_group = sp_group.group if sp_group is not None else None
        self.attention = ParallelAttention(mconf, layer_number, attention_type=AttnType.self_attn, attn_mask_type=AttnMaskType.padding,
                                           tp_group=self.tp_group, sp_group=self.sp_group, use_ulysses=self.use_ulysses, device="meta")
        self.LayerNorm = LayerNorm(config.hidden_size, eps=config.layer_norm_eps, device="meta",
                                   sequence_parallel=_megatron_sp(args, tp_group))
        # attention_dropout on the attention-block output, as the reference (:29-36)
        self.dropout_p, self.site = mconf.attention_dropout, site(layer_number + 1, SITE_ATTENTION)
        self.seq_rank = _seq_rank(args, tp_group, sp_group)

    def forward(self, hidden_states, attention_mask):
        residual = hidden_states
        if self.dropout_p > 0.0 and self.training:
            out, bias = self.attention(hidden_states, attention_mask)
            return self.LayerNorm(bias_dropout_add(out, bias, residual, self.dropout_p, self.site, self.seq_rank * out.shape[0]))
        hidden_states, bias = self.attention(hidden_states, attention_mask, residual=residual)   # + residual in the GEMM epilogue
        if bias is not None:
            hidden_states = hidden_states + bias
        return self.LayerNorm(hidden_states)                             # post-LN (:31-39)


class BertMLP_tp(nn.Module):
    def __init__(self, config, tp_group=None, layer_number=0, sp_group=None):
        super().__init__()
        args = get_args()
        mconf = core_transformer_config_from_args(args)
        self.tp_group = tp_group.group if tp_group is not None else None
        self.mlp = ParallelMLP(mconf, tp_group=self.tp_group, device="meta")
        self.LayerNorm = LayerNorm(config.hidden_size, eps=config.layer_norm_eps, device="meta",
                                   sequence_parallel=_megatron_sp(args, tp_group))
        self.dropout_p, self.site = mconf.hidden_dropout, site(layer_number + 1, SITE_MLP)       # :48-55
        self.seq_rank = _seq_rank(args, tp_group, sp_group)

    def forward(self, hidden_states):
        residual = hidden_states
        if self.dropout_p > 0.0 and self.training:
            out, bias = self.mlp(hidden_states)
            return self.LayerNorm(bias_dropout_add(out, bias, residual, self.dropout_p, self.site, self.seq_rank * out.shape[0]))
        hidden_states, bias = self.mlp(hidden_states, residual=residual)
        if bias is not None:
            hidden_states = hidden_states + bias
        return self.LayerNorm(hidden_states)


class BertLayer_tp(nn.Module):
    def __init__(self, config, layer_number, tp_group=None, sp_group=None):
        super().__init__()
        self.attention = BertAttention_tp(config, layer_number, tp_group, sp_group)
        self.mlp = BertMLP_tp(config, tp_group, layer_number, sp_group)
        self.idx = layer_number

    def forward(self, hidden_states, attention_mask=None):
        return self.mlp(self.attention(hidden_states, attention_mask))


class _Transform(nn.Module):
    """HF ``BertPredictionHeadTransform``: dense + GeLU + LayerNorm, replicated over the tensor-parallel group."""

    def __init__(self, config, sequence_parallel):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(config.hidden_size, config.hidden_size, device="meta"))
        self.bias = nn.Parameter(torch.empty(config.hidden_size, device="meta"))
        self.LayerNorm = LayerNorm(config.hidden_size, eps=config.layer_norm_eps, device="meta", sequence_parallel=sequence_parallel)
        self._sequence_parallel = bool(sequence_parallel)
        self.init_std = get_args().init_method_std

    def reset_parameters(self):
        nn.init.normal_(self.weight, mean=0.0, std=self.init_std)
        nn.init.zeros_(self.bias)
        for p in (self.weight, self.bias):    # under Megatron-SP the head sees its sequence slice only: summed over the TP group
            setattr(p, "sequence_parallel", self._sequence_parallel)

    def forward(self, hidden_states):
        x = torch.nn.functional.linear(hidden_states, self.weight.to(hidden_states.dtype), self.bias.to(hidden_states.dtype))
        return self.LayerNorm(torch.nn.functional.gelu(x, approximate="tanh"))


class _TypeEmbedding(nn.Module):
    """Token-type (segment) embedding, replicated (the reference keeps HF's ``nn.Embedding``, :121-130)."""

    def __init__(self, config):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(config.type_vocab_size, config.hidden_size, device="meta"))
        self.init_std = get_args().init_method_std

    def reset_parameters(self):
        nn.init.normal_(self.weight, mean=0.0, std=self.init_std)

    def forward(self, token_type_ids):
        return torch.nn.functional.embedding(token_type_ids, self.weight)


class BertSkeleton(nn.Module):
    """Container with the attribute layout of HF ``BertForMaskedLM`` (``.bert.embeddings/.encoder.layer``, ``.cls.predictions``) that
    the reference's callbacks mutate; created empty -- every real layer is built by ``construct_tensor_parallel_model``."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.bert = nn.Module()
        self.bert.embeddings = nn.Module()
        self.bert.encoder = nn.Module()
        self.bert.encoder.layer = nn.ModuleList()
        self.cls = nn.Module()
        self.cls.predictions = nn.Module()


def construct_tensor_parallel_model(model, config, tp_groups_enc, sp_groups_enc):
    """Whole-model rows: [embed, layer_0..L-1, mlm_head] (BertModel_tensor_parallel.py:74-133; 4-argument callback)."""
    args = get_args()
    mconf = core_transformer_config_from_args(args)
    model.bert.encoder.layer = nn.ModuleList([BertLayer_tp(config, i, tp_group=tp_groups_enc[i + 1], sp_group=sp_groups_enc[i + 1])
                                              for i in range(config.num_hidden_layers)])
    emb = model.bert.embeddings
    for name, rows in (("word_embeddings", args.padded_vocab_size), ("position_embeddings", config.max_position_embeddings)):
        setattr(emb, name, VocabParallelEmbedding(rows, mconf.hidden_size, config=mconf, tp_group=tp_groups_enc[0].group,
                                                  sp_group=sp_groups_enc[0].group, device="meta"))
    emb.token_type_embeddings = _TypeEmbedding(config)
    vocab_msp = bool(args.sequence_parallel) and args.vocab_tp > 1 and not args.vocab_sp
    emb.LayerNorm = LayerNorm(config.hidden_size, eps=config.layer_norm_eps, device="meta")
    model.cls.predictions.transform = _Transform(config, sequence_parallel=vocab_msp)
    model.cls.predictions.decoder = ColumnParallelLinear(config.hidden_size, args.padded_vocab_size, config=mconf, bias=True,
                                                         tp_group=tp_groups_enc[-1].group, sp_group=sp_groups_enc[-1].group, device="meta")
    return model

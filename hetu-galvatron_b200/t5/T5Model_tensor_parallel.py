"""T5 layer classes over the group-explicit parallel ops (``galvatron/models/T5/T5Model_tensor_parallel.py``): pre-RMSNorm blocks
(T5LayerNorm: weight only), Megatron attention with biases and scale 1/sqrt(d_kv) over an inner width d_kv x heads, bias-GeLU (tanh
form) MLP with biases.  The encoder attends to everything, the decoder's self-attention is causal and its cross-attention sees the
whole encoder output -- the reference's flash-attention path, on which the batch's masks are not used.  No relative-position bias
and no positions (the reference has neither)."""
import types

from torch import nn

from ..core.runtime.arguments import get_args
from ..core.runtime.tensor_parallel import (AttnMaskType, AttnType, ColumnParallelLinear, ParallelAttention, ParallelMLP, RMSNorm,
                                            VocabParallelEmbedding)


def t5_transformer_config(args):
    """The ``TransformerConfig`` fields the layer code reads for a T5 block: biases on, tanh-GeLU, no gating, kv_channels = d_kv."""
    return types.SimpleNamespace(
        hidden_size=args.hidden_size, ffn_hidden_size=args.ffn_hidden_size, num_attention_heads=args.num_attention_heads,
        num_query_groups=args.num_attention_heads, kv_channels=args.kv_channels, layernorm_epsilon=args.norm_epsilon,
        init_method_std=args.init_method_std, sequence_parallel=args.sequence_parallel, gated_linear_unit=False, add_bias_linear=True,
        gelu_tanh=True, hidden_dropout=0.0, attention_dropout=0.0)


def _megatron_sp(args, tp_group):
    return bool(args.sequence_parallel) and tp_group is not None and tp_group.size > 1


class T5Attention_tp(nn.Module):
    """RMSNorm -> self- or cross-attention -> + residual (the residual rides in the output projection's GEMM epilogue)."""

    def __init__(self, config, layer_number, attention_type, attn_mask_type, tp_group=None):
        super().__init__()
        args = get_args()
        self.tp_group = tp_group.group if tp_group is not None else None
        self.cross = attention_type == AttnType.cross_attn
        self.attention = ParallelAttention(t5_transformer_config(args), layer_number, attention_type=attention_type,
                                           attn_mask_type=attn_mask_type, tp_group=self.tp_group, device="meta")
        self.LayerNorm = RMSNorm(config.hidden_size, eps=config.layer_norm_epsilon, device="meta",
                                 sequence_parallel=_megatron_sp(args, tp_group))

    def forward(self, hidden_states, encoder_output=None):
        """-> the block's output; for cross-attention (output, encoder_output pass-through)"""
        residual = hidden_states
        normed = self.LayerNorm(hidden_states)
        if self.cross:
            out, bias, enc = self.attention(normed, None, encoder_output, residual=residual)
            return (out if bias is None else out + bias), enc
        out, bias = self.attention(normed, None, residual=residual)
        return out if bias is None else out + bias


class T5MLP_tp(nn.Module):
    def __init__(self, config, tp_group=None):
        super().__init__()
        args = get_args()
        self.tp_group = tp_group.group if tp_group is not None else None
        self.mlp = ParallelMLP(t5_transformer_config(args), tp_group=self.tp_group, device="meta")
        self.LayerNorm = RMSNorm(config.hidden_size, eps=config.layer_norm_epsilon, device="meta",
                                 sequence_parallel=_megatron_sp(args, tp_group))

    def forward(self, hidden_states):
        out, bias = self.mlp(self.LayerNorm(hidden_states), residual=hidden_states)
        return out if bias is None else out + bias


class T5EncoderLayer_tp(nn.Module):
    def __init__(self, config, layer_number, tp_group=None):
        super().__init__()
        self.attention = T5Attention_tp(config, layer_number, AttnType.self_attn, AttnMaskType.padding, tp_group)
        self.mlp = T5MLP_tp(config, tp_group)
        self.idx = layer_number

    def forward(self, hidden_states):
        return self.mlp(self.attention(hidden_states))


class T5DecoderLayer_tp(nn.Module):
    """(encoder output, decoder hidden states) -> (the same encoder output, the layer's output)"""

    def __init__(self, config, layer_number, tp_group=None):
        super().__init__()
        self.attention = T5Attention_tp(config, layer_number, AttnType.self_attn, AttnMaskType.causal, tp_group)
        self.cross_attention = T5Attention_tp(config, layer_number, AttnType.cross_attn, AttnMaskType.padding, tp_group)
        self.mlp = T5MLP_tp(config, tp_group)
        self.idx = layer_number

    def forward(self, enc_hidden_states, dec_hidden_states):
        hidden = self.attention(dec_hidden_states)
        hidden, enc_hidden_states = self.cross_attention(hidden, enc_hidden_states)
        return enc_hidden_states, self.mlp(hidden)


class T5Skeleton(nn.Module):
    """Container with the attributes the sequential rows read (``shared``, ``dec_shared``, ``encoder``, ``decoder``, the two final
    norms, ``lm_head``); created empty -- every real layer is built by ``construct_tensor_parallel_model``."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.encoder, self.decoder = nn.ModuleList(), nn.ModuleList()
        self.shared = self.dec_shared = self.lm_head = self.enc_final_norm = self.dec_final_norm = None


def row_index(config):
    """whole-model row of each part: embed_1, t5_enc x L_enc, pre_norm_1, embed_2, t5_dec x L_dec, pre_norm_2, cls"""
    le, ld = config.num_layers, config.num_decoder_layers
    return dict(embed_1=0, enc=1, pre_norm_1=le + 1, embed_2=le + 2, dec=le + 3, pre_norm_2=le + ld + 3, cls=le + ld + 4)


def construct_tensor_parallel_model(model, config, tp_groups_enc, sp_groups_enc, cp_groups_enc):
    """Whole-model rows as ``row_index``; the vocabulary rows take their own row's tensor-parallel group."""
    args = get_args()
    mconf = t5_transformer_config(args)
    rows = row_index(config)
    model.encoder = nn.ModuleList([T5EncoderLayer_tp(config, i, tp_group=tp_groups_enc[rows["enc"] + i]) for i in range(config.num_layers)])
    model.decoder = nn.ModuleList([T5DecoderLayer_tp(config, config.num_layers + i, tp_group=tp_groups_enc[rows["dec"] + i])
                                   for i in range(config.num_decoder_layers)])
    for name, row in (("shared", rows["embed_1"]), ("dec_shared", rows["embed_2"])):
        setattr(model, name, VocabParallelEmbedding(args.padded_vocab_size, mconf.hidden_size, config=mconf,
                                                    tp_group=tp_groups_enc[row].group, device="meta"))
    # the final norms sit in the vocabulary-degree rows pre_norm_1 / pre_norm_2
    sp_norm = bool(args.sequence_parallel) and args.vocab_tp > 1
    model.enc_final_norm = RMSNorm(config.hidden_size, eps=config.layer_norm_epsilon, device="meta", sequence_parallel=sp_norm)
    model.dec_final_norm = RMSNorm(config.hidden_size, eps=config.layer_norm_epsilon, device="meta", sequence_parallel=sp_norm)
    model.lm_head = ColumnParallelLinear(mconf.hidden_size, args.padded_vocab_size, config=mconf, bias=False,
                                         tp_group=tp_groups_enc[rows["cls"]].group, device="meta")
    return model

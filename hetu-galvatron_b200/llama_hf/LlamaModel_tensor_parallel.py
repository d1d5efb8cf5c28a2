"""Llama layer classes over the group-explicit parallel ops (``galvatron/models/llama_hf/LlamaModel_tensor_parallel.py``)."""
import types

import torch
from torch import nn

from ..core.runtime.arguments import get_args
from ..core.runtime.backend import get_backend
from ..core.runtime.redistribute import local_positions
from ..core.runtime.tensor_parallel import (AttnMaskType, AttnType, ColumnParallelLinear, ParallelAttention, ParallelMLP,
                                            RMSNorm, VocabParallelEmbedding)


def core_transformer_config_from_args(args):
    """The handful of ``TransformerConfig`` fields the layer code reads (megatron ``core_transformer_config_from_args``)."""
    return types.SimpleNamespace(
        hidden_size=args.hidden_size, ffn_hidden_size=args.ffn_hidden_size, num_attention_heads=args.num_attention_heads,
        num_query_groups=args.num_query_groups or args.num_attention_heads, kv_channels=args.hidden_size // args.num_attention_heads,
        layernorm_epsilon=args.norm_epsilon, init_method_std=args.init_method_std, sequence_parallel=args.sequence_parallel,
        gated_linear_unit=True, add_bias_linear=False, rotary_base=getattr(args, "rotary_base", 10000.0))


class LlamaAttention_tp(nn.Module):
    def __init__(self, config, layer_number, tp_group=None, sp_group=None, cp_group=None):
        super().__init__()
        args = get_args()
        self.sequence_parallel = args.sequence_parallel
        self.sp_size = sp_group.size if sp_group is not None else 1
        self.cp_size = cp_group.size if cp_group is not None else 1
        self.use_ulysses = self.sp_size > 1
        self.use_zigzag_cp = self.cp_size > 1
        mconf = core_transformer_config_from_args(args)
        self.tp_group = tp_group.group if tp_group is not None else None
        self.sp_group = sp_group.group if sp_group is not None else None
        self.cp_group = cp_group.group if cp_group is not None else None
        self.attention = ParallelAttention(mconf, layer_number, attention_type=AttnType.self_attn,
                                           attn_mask_type=AttnMaskType.causal, tp_group=self.tp_group, sp_group=self.sp_group,
                                           cp_group=self.cp_group, cp_ranks=cp_group.ranks if cp_group is not None else None,
                                           use_ulysses=self.use_ulysses, use_zigzag_cp=self.use_zigzag_cp, device="meta")
        self.hidden_size, self.num_heads = config.hidden_size, config.num_attention_heads
        self.head_dim = self.hidden_size // self.num_heads
        self.layer_idx = layer_number
        megatron_sp = bool(self.sequence_parallel) and (tp_group is not None and tp_group.size > 1)
        self.LayerNorm = RMSNorm(config.hidden_size, eps=config.rms_norm_eps, device="meta", sequence_parallel=megatron_sp)
        self.rotary_base = mconf.rotary_base
        self._rope_cache = {}
        self.recompute_activations = bool(getattr(get_args(), "recompute_activations", False))

    def _rope(self, local_seq, offset, device):
        key = (local_seq, offset)
        if key not in self._rope_cache:
            self._rope_cache[key] = get_backend().rope_tables(local_seq, self.head_dim, self.rotary_base, offset,
                                                              torch.bfloat16 if get_args().mixed_precision == "bf16" else torch.float32, device)
        return self._rope_cache[key]

    def _rope_zigzag(self, local_seq, device):
        """RoPE rows of the ``local_seq`` tokens this rank holds under zigzag context parallelism, Ulysses or not: the positions
        of redistribute.local_positions (the reference builds them in get_pos_emb_on_this_cp_sp_rank_galvatron)"""
        key = ("zigzag", local_seq)
        if key not in self._rope_cache:
            c, r = self.cp_size, self.cp_group.rank_in_group()
            p, j = (self.sp_size, self.sp_group.rank_in_group()) if self.use_ulysses else (1, 0)
            cos, sin = self._rope(local_seq * c * p, 0, device)
            idx = local_positions(local_seq * c * p, c, r, p, j).to(device)
            self._rope_cache[key] = (cos[idx].contiguous(), sin[idx].contiguous())
        return self._rope_cache[key]

    def forward(self, hidden_states, attention_mask):
        residual = hidden_states
        hidden_states = self.LayerNorm(hidden_states)
        s_local = hidden_states.shape[0]
        # position offset rules of LlamaModel_tensor_parallel.py:58-79: Ulysses ranks hold consecutive sequence slices
        # (offset = local_seq * sp_rank); Megatron-SP gathers the sequence before QKV, so RoPE sees tp * local positions
        if self.use_ulysses:
            seq, offset = s_local, s_local * self.sp_group.rank_in_group()
        elif self.sequence_parallel and self.tp_group is not None and self.tp_group.size > 1:
            seq, offset = s_local * self.tp_group.size, 0
        else:
            seq, offset = s_local, 0
        if self.use_zigzag_cp:
            # zigzag context parallelism: this rank's `seq` tokens are chunks (r, 2c-1-r) of the sequence, or under Ulysses the sp
            # rank's slice of them; RoPE takes their global positions (the reference lets Megatron's RotaryEmbedding pick them,
            # LlamaModel_tensor_parallel.py:58-63)
            rope = self._rope_zigzag(seq, hidden_states.device)
        else:
            rope = self._rope(seq, offset, hidden_states.device)
        recipe = ("rmsnorm", residual, self.LayerNorm.weight, self.LayerNorm.eps) if self.recompute_activations else None
        # `out + residual` (:83) rides in the o-proj GEMM's epilogue (or follows its collective)
        out, _ = self.attention(hidden_states, attention_mask, rotary_pos_emb=rope, input_recipe=recipe, residual=residual)
        return out


class LlamaMLP_tp(nn.Module):
    def __init__(self, config, tp_group=None):
        super().__init__()
        args = get_args()
        mconf = core_transformer_config_from_args(args)
        self.tp_group = tp_group.group if tp_group is not None else None
        self.mlp = ParallelMLP(mconf, tp_group=self.tp_group, device="meta")
        self.recompute_activations = bool(getattr(args, "recompute_activations", False))
        megatron_sp = bool(args.sequence_parallel) and (tp_group is not None and tp_group.size > 1)
        self.LayerNorm = RMSNorm(config.hidden_size, eps=config.rms_norm_eps, device="meta", sequence_parallel=megatron_sp)

    def forward(self, hidden_states):
        residual = hidden_states
        hidden_states = self.LayerNorm(hidden_states)
        recipe = ("rmsnorm", residual, self.LayerNorm.weight, self.LayerNorm.eps) if self.recompute_activations else None
        out, _ = self.mlp(hidden_states, input_recipe=recipe, residual=residual)      # `out + residual` (:100) in the GEMM epilogue
        return out


class LlamaLayer_tp(nn.Module):
    def __init__(self, config, layer_number, tp_group=None, sp_group=None, cp_group=None):
        super().__init__()
        self.attention = LlamaAttention_tp(config, layer_number, tp_group, sp_group, cp_group)
        self.mlp = LlamaMLP_tp(config, tp_group)
        self.idx = layer_number

    def forward(self, hidden_states, attention_mask=None):
        return self.mlp(self.attention(hidden_states, attention_mask))


class LlamaSkeleton(nn.Module):
    """Container with the attribute layout of HF ``LlamaForCausalLM`` (``.model.layers/.embed_tokens``, ``.lm_head``) that
    the reference's callbacks mutate; created empty -- every real layer is built by ``construct_tensor_parallel_model``."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.model = nn.Module()
        self.model.layers = nn.ModuleList()
        self.model.embed_tokens = None
        self.lm_head = None


def construct_tensor_parallel_model(model, config, tp_groups_whole, sp_groups_whole, cp_groups_whole):
    """Whole-model rows: [embed, layer_0..L-1, norm, cls] (LlamaModel_tensor_parallel.py:121-160)."""
    args = get_args()
    mconf = core_transformer_config_from_args(args)
    layers = nn.ModuleList([LlamaLayer_tp(config, i, tp_group=tp_groups_whole[i + 1], sp_group=sp_groups_whole[i + 1],
                                          cp_group=cp_groups_whole[i + 1]) for i in range(config.num_hidden_layers)])
    setattr(model.model, "layers", layers)
    setattr(model.model, "embed_tokens", VocabParallelEmbedding(
        args.padded_vocab_size, mconf.hidden_size, config=mconf, tp_group=tp_groups_whole[0].group,
        sp_group=sp_groups_whole[0].group, cp_group=cp_groups_whole[0].group, device="meta"))
    setattr(model, "lm_head", ColumnParallelLinear(
        mconf.hidden_size, args.padded_vocab_size, config=mconf, bias=False, tp_group=tp_groups_whole[-1].group,
        sp_group=sp_groups_whole[-1].group, cp_group=cp_groups_whole[-1].group, device="meta"))
    return model

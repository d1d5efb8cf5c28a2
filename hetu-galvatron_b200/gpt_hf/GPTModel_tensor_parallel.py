"""GPT layer classes over the group-explicit parallel ops (``galvatron/models/gpt_hf/GPTModel_tensor_parallel.py``):
pre-LayerNorm blocks with biases on every projection, GeLU MLP, learned absolute positions (no RoPE)."""
import types

from torch import nn

from ..core.runtime.arguments import get_args
from ..core.runtime.redistribute import local_positions, token_runs
from ..core.runtime.tensor_parallel import (AttnMaskType, AttnType, ColumnParallelLinear, LayerNorm, ParallelAttention, ParallelMLP,
                                            VocabParallelEmbedding)
from ..core.runtime.tensor_parallel.random import SITE_ATTENTION, SITE_MLP, bias_dropout_add, check_probability, site


def core_transformer_config_from_args(args):
    """The ``TransformerConfig`` fields the layer code reads (megatron ``core_transformer_config_from_args``) for a GPT / BERT style
    block: biases on, GeLU (tanh form: ``bias_gelu_fusion``), no gating, no rotary embedding."""
    return types.SimpleNamespace(
        hidden_size=args.hidden_size, ffn_hidden_size=args.ffn_hidden_size, num_attention_heads=args.num_attention_heads,
        num_query_groups=args.num_attention_heads, kv_channels=args.hidden_size // args.num_attention_heads,
        layernorm_epsilon=args.norm_epsilon, init_method_std=args.init_method_std, sequence_parallel=args.sequence_parallel,
        gated_linear_unit=False, add_bias_linear=True, gelu_tanh=True,
        hidden_dropout=check_probability(getattr(args, "hidden_dropout", 0.0), "hidden_dropout"),
        attention_dropout=check_probability(getattr(args, "attention_dropout", 0.0), "attention_dropout"))


def _megatron_sp(args, tp_group):
    return bool(args.sequence_parallel) and tp_group is not None and tp_group.size > 1


def _seq_rank(args, tp_group, sp_group):
    """Index of the sequence slice a block's [s/p, b, h] activations hold: the Ulysses rank, the Megatron-SP (tensor-parallel) rank,
    or 0 when the block sees the whole sequence.  Dropout masks are drawn at global token positions seq_rank * s/p + local row."""
    if sp_group is not None and sp_group.size > 1:
        return sp_group.rank_in_group()
    if _megatron_sp(args, tp_group):
        return tp_group.rank_in_group()
    return 0


def _size(g):
    return 1 if g is None else g.size


def row_runs(rows, cp_group=None, sp_group=None, tp_group=None):
    """Runs of consecutive global tokens, ((first row, rows, first token), ...), held by the ``rows`` local rows of an SBH activation
    of a rank in these groups: the cp rank's zigzag chunks, of those the Ulysses (``sp_group``) rank's slice, of that the
    Megatron-SP (``tp_group``) rank's slice (redistribute.local_positions).  Dropout masks are drawn at these positions."""
    c, p, t = _size(cp_group), _size(sp_group), _size(tp_group)
    pos = local_positions(rows * c * p * t, c, cp_group.rank_in_group() if c > 1 else 0, p, sp_group.rank_in_group() if p > 1 else 0)
    k = tp_group.rank_in_group() if t > 1 else 0
    return token_runs(pos[k * rows:(k + 1) * rows])


class _Dropout:
    """hidden-state dropout of one block output: the site and the token runs of this rank's rows (per local row count)"""

    def __init__(self, p, site_id, args, tp_group, sp_group, cp_group):
        self.p, self.site = p, site_id
        ulysses = sp_group is not None and sp_group.size > 1
        self.groups = (cp_group, sp_group if ulysses else None, tp_group if not ulysses and _megatron_sp(args, tp_group) else None)
        self._runs = {}

    def __call__(self, out, bias, residual):
        rows = out.shape[0]
        if rows not in self._runs:
            self._runs[rows] = row_runs(rows, *self.groups)
        return bias_dropout_add(out, bias, residual, self.p, self.site, self._runs[rows])


def _check_cp(args, mconf, cp_group, sp_group):
    """Construction-time limits of a GPT layer under context parallelism (degree c, Ulysses degree p)."""
    c, p = _size(cp_group), _size(sp_group)
    if c == 1:
        return
    if mconf.attention_dropout > 0.0:
        raise NotImplementedError(
            "GPT with context parallelism (cp %d) needs attn_pdrop = 0: GPT's attention_dropout (%g) also drops the attention-block "
            "output, as in the reference, and attention-probability dropout is not supported with context parallelism "
            "(hidden dropout, resid_pdrop / embd_pdrop, is)" % (c, mconf.attention_dropout))
    if args.seq_length % (2 * c * p):
        raise ValueError("GPT with context parallelism: sequence length %d must be a multiple of 2 x cp%s = %d"
                         % (args.seq_length, " x sp" if p > 1 else "", 2 * c * p))


class GPTAttention_tp(nn.Module):
    def __init__(self, config, layer_number, tp_group=None, sp_group=None, cp_group=None):
        super().__init__()
        args = get_args()
        self.use_ulysses = sp_group is not None and sp_group.size > 1
        self.use_zigzag_cp = cp_group is not None and cp_group.size > 1
        mconf = core_transformer_config_from_args(args)
        _check_cp(args, mconf, cp_group, sp_group)
        self.tp_group = tp_group.group if tp_group is not None else None
        self.sp_group = sp_group.group if sp_group is not None else None
        self.cp_group = cp_group.group if cp_group is not None else None
        self.attention = ParallelAttention(mconf, layer_number, attention_type=AttnType.self_attn, attn_mask_type=AttnMaskType.causal,
                                           tp_group=self.tp_group, sp_group=self.sp_group, cp_group=self.cp_group,
                                           cp_ranks=cp_group.ranks if cp_group is not None else None, use_ulysses=self.use_ulysses,
                                           use_zigzag_cp=self.use_zigzag_cp, device="meta")
        self.LayerNorm = LayerNorm(config.hidden_size, eps=config.layer_norm_epsilon, device="meta",
                                   sequence_parallel=_megatron_sp(args, tp_group))
        # the reference drops the attention-block output with attention_dropout, not hidden_dropout (:31-39): kept on purpose
        self.dropout_p = mconf.attention_dropout
        self.dropout = _Dropout(self.dropout_p, site(layer_number + 1, SITE_ATTENTION), args, tp_group, sp_group, cp_group)

    def forward(self, hidden_states, attention_mask):
        residual = hidden_states
        hidden_states = self.LayerNorm(hidden_states)
        if self.dropout_p > 0.0 and self.training:
            # after the projection's reduction (all-reduce / reduce-scatter): one row kernel for bias + dropout + residual
            out, bias = self.attention(hidden_states, None)
            return self.dropout(out, bias, residual)
        # causal: the mask is implied (flash path, :36-41); the residual add (:42) rides in the projection GEMM's epilogue
        hidden_states, bias = self.attention(hidden_states, None, residual=residual)
        return hidden_states if bias is None else hidden_states + bias


class GPTMLP_tp(nn.Module):
    def __init__(self, config, tp_group=None, layer_number=0, sp_group=None, cp_group=None):
        super().__init__()
        args = get_args()
        mconf = core_transformer_config_from_args(args)
        self.tp_group = tp_group.group if tp_group is not None else None
        self.mlp = ParallelMLP(mconf, tp_group=self.tp_group, device="meta")
        self.LayerNorm = LayerNorm(config.hidden_size, eps=config.layer_norm_epsilon, device="meta",
                                   sequence_parallel=_megatron_sp(args, tp_group))
        self.dropout_p = mconf.hidden_dropout                                                      # :51-59
        self.dropout = _Dropout(self.dropout_p, site(layer_number + 1, SITE_MLP), args, tp_group, sp_group, cp_group)

    def forward(self, hidden_states):
        residual = hidden_states
        hidden_states = self.LayerNorm(hidden_states)
        if self.dropout_p > 0.0 and self.training:
            out, bias = self.mlp(hidden_states)
            return self.dropout(out, bias, residual)
        hidden_states, bias = self.mlp(hidden_states, residual=residual)
        return hidden_states if bias is None else hidden_states + bias


class GPTLayer_tp(nn.Module):
    def __init__(self, config, layer_number, tp_group=None, sp_group=None, cp_group=None):
        super().__init__()
        self.attention = GPTAttention_tp(config, layer_number, tp_group, sp_group, cp_group)
        self.mlp = GPTMLP_tp(config, tp_group, layer_number, sp_group, cp_group)
        self.idx = layer_number

    def forward(self, hidden_states, attention_mask=None):
        return self.mlp(self.attention(hidden_states, attention_mask))


class GPTSkeleton(nn.Module):
    """Container with the attribute layout of HF ``GPT2LMHeadModel`` (``.transformer.h/.wte/.wpe/.ln_f``, ``.lm_head``) that the
    reference's callbacks mutate; created empty -- every real layer is built by ``construct_tensor_parallel_model``."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.transformer = nn.Module()
        self.transformer.h = nn.ModuleList()
        self.transformer.wte = self.transformer.wpe = None
        self.transformer.ln_f = LayerNorm(config.hidden_size, eps=config.layer_norm_epsilon, device="meta")
        self.lm_head = None


def construct_tensor_parallel_model(model, config, tp_groups_enc, sp_groups_enc, cp_groups_enc):
    """Whole-model rows: [embed, layer_0..L-1, norm, cls] (GPTModel_tensor_parallel.py:84-132); the 5-argument callback, as the
    Llama family's: the embeddings and the head take the cp group of their row, the layers that of theirs."""
    args = get_args()
    mconf = core_transformer_config_from_args(args)
    layers = nn.ModuleList([GPTLayer_tp(config, i, tp_group=tp_groups_enc[i + 1], sp_group=sp_groups_enc[i + 1],
                                        cp_group=cp_groups_enc[i + 1]) for i in range(config.num_hidden_layers)])
    setattr(model.transformer, "h", layers)
    for name, rows in (("wte", args.padded_vocab_size), ("wpe", args.seq_length)):
        setattr(model.transformer, name, VocabParallelEmbedding(rows, mconf.hidden_size, config=mconf, tp_group=tp_groups_enc[0].group,
                                                                sp_group=sp_groups_enc[0].group, cp_group=cp_groups_enc[0].group,
                                                                device="meta"))
    # the final norm sits in the "norm" row, whose degrees are the vocabulary's
    model.transformer.ln_f = LayerNorm(config.hidden_size, eps=config.layer_norm_epsilon, device="meta",
                                       sequence_parallel=bool(args.sequence_parallel) and args.vocab_tp > 1 and not args.vocab_sp)
    setattr(model, "lm_head", ColumnParallelLinear(mconf.hidden_size, args.padded_vocab_size, config=mconf, bias=False,
                                                   tp_group=tp_groups_enc[-1].group, sp_group=sp_groups_enc[-1].group,
                                                   cp_group=cp_groups_enc[-1].group, device="meta"))
    return model

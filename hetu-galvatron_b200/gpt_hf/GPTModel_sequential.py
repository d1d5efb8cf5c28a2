"""Sequential (pipeline-able) view of the GPT model (``galvatron/models/gpt_hf/GPTModel_sequential.py``)."""
import torch
import torch.nn as nn

from ..core.runtime.arguments import get_args
from ..core.runtime.hybrid_parallel_config import ModelInfo, mixed_precision_dtype
from ..core.runtime.pipeline import PipeSequential
from ..core.runtime.redistribute import zigzag_local
from ..core.runtime.tensor_parallel import (gather_from_tensor_model_parallel_region_group, linear_with_grad_accumulation_and_async_allreduce,
                                            scatter_to_sequence_parallel_region_group, vocab_parallel_cross_entropy)
from ..core.runtime.tensor_parallel.random import SITE_EMBEDDING, bias_dropout_add, check_probability, site
from .GPTModel_tensor_parallel import row_runs


def _size(g):
    return 1 if g is None else g.size


class GPTVocabEmbedding_(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.wte = model.wte

    def forward(self, tokens):
        return self.wte(tokens)


class GPTPositionEmbedding_(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.wpe = model.wpe

    def forward(self, position_ids):
        return self.wpe(position_ids)


class GPTEmbeddings_(nn.Module):
    def __init__(self, model):
        super().__init__()
        args = get_args()
        self.wte, self.wpe = GPTVocabEmbedding_(model.transformer), GPTPositionEmbedding_(model.transformer)
        self.sequence_parallel = args.sequence_parallel
        self.tp_group, self.sp_group, self.cp_group = self.wte.wte.tp_group, self.wte.wte.sp_group, self.wte.wte.cp_group
        # Ulysses on the embedding: each rank embeds its own sequence slice (:59-64), of the cp rank's zigzag chunks under cp
        self.seq_group = self.sp_group if args.vocab_sp else None
        self.dropout_p = check_probability(getattr(args, "hidden_dropout", 0.0), "hidden_dropout")     # :55
        self.tp_split = self.tp_group if self.sequence_parallel and _size(self.tp_group) > 1 else None
        self._runs = {}
        c, p = _size(self.cp_group), _size(self.seq_group)
        if c > 1 and args.seq_length % (2 * c * p):
            raise ValueError("GPT with context parallelism: sequence length %d must be a multiple of 2 x cp%s = %d"
                             % (args.seq_length, " x sp" if p > 1 else "", 2 * c * p))

    def forward(self, tokens, position_ids=None, attention_mask=None, labels=None):
        if position_ids is None:
            position_ids = torch.arange(0, tokens.size(-1), dtype=torch.long, device=tokens.device).unsqueeze(0)
        # this rank's tokens and their GLOBAL positions: the learned position table is looked up where the tokens sit in the sequence
        tokens = zigzag_local(tokens, self.cp_group, self.seq_group)
        position_ids = zigzag_local(position_ids, self.cp_group, self.seq_group)
        hidden_states = self.wte(tokens) + self.wpe(position_ids)
        hidden_states = hidden_states.transpose(0, 1).contiguous()           # [b, s, h] -> [s, b, h]
        if self.sequence_parallel:
            hidden_states = scatter_to_sequence_parallel_region_group(hidden_states, self.tp_group)
        if not (self.dropout_p > 0.0 and self.training):
            return hidden_states
        # embedding dropout (hidden_dropout) on the rows this rank holds after the Megatron-SP scatter, at their global token positions
        rows = hidden_states.shape[0]
        if rows not in self._runs:
            self._runs[rows] = row_runs(rows, self.cp_group, self.seq_group, self.tp_split)
        return bias_dropout_add(hidden_states, None, None, self.dropout_p, site(0, SITE_EMBEDDING), self._runs[rows])


class GPTLayers_(nn.Module):
    def __init__(self, model, layer_idx):
        super().__init__()
        self.layer = model.transformer.h[layer_idx]

    def forward(self, hidden_states, position_ids=None, attention_mask=None, labels=None):
        return self.layer(hidden_states, attention_mask=attention_mask)


class GPTPreNorm_(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.ln_f = model.transformer.ln_f

    def forward(self, hidden_states, position_ids=None, attention_mask=None, labels=None):
        return self.ln_f(hidden_states)


class GPTLoss_(nn.Module):
    def __init__(self, lm_head, sequence_parallel, tp_group):
        super().__init__()
        self.weight = lm_head.weight
        self.init_std = lm_head.init_std
        self.tp_group = tp_group
        self.sequence_parallel = bool(sequence_parallel) and _size(tp_group) > 1   # :128-131

    def reset_parameters(self):
        nn.init.normal_(self.weight, mean=0.0, std=self.init_std)
        setattr(self.weight, "tensor_model_parallel", True)

    def forward(self, hidden_states):
        # (without SP the dgrad all-reduce of copy_to_tensor_model_parallel_region :171-172 happens inside the linear)
        return linear_with_grad_accumulation_and_async_allreduce(
            input=hidden_states, weight=self.weight, bias=None, async_grad_allreduce=not self.sequence_parallel,
            sequence_parallel=self.sequence_parallel, tp_group=self.tp_group)


class GPTCls_(nn.Module):
    def __init__(self, model, parallel_loss=True, half_entropy=True):
        super().__init__()
        args = get_args()
        self.sequence_parallel = args.sequence_parallel
        head = model.lm_head
        self.tp_group, self.sp_group, self.cp_group = head.tp_group, head.sp_group, head.cp_group
        self.lm_head = GPTLoss_(head, self.sequence_parallel, self.tp_group)
        self.parallel_loss = parallel_loss
        self.half_entropy = half_entropy and not args.entropy_in_fp32
        self.vocab_sp = args.vocab_sp
        self.seq_group = self.sp_group if self.vocab_sp else None

    def forward(self, hidden_states, position_ids=None, attention_mask=None, labels=None):
        labels = zigzag_local(labels, self.cp_group, self.seq_group)
        logits_parallel = self.lm_head(hidden_states)                          # [s, b, V/t]
        labels = labels.transpose(0, 1).contiguous()                            # [b, s] -> [s, b]
        if not self.parallel_loss:
            logits = gather_from_tensor_model_parallel_region_group(logits_parallel, self.tp_group)
            logits = logits if self.half_entropy else logits.float()
            return torch.nn.functional.cross_entropy(logits.reshape(-1, logits.size(-1)), labels.reshape(-1))
        logits_in = logits_parallel if self.half_entropy else logits_parallel.float()
        loss = vocab_parallel_cross_entropy(logits_in, labels, tp_group=self.tp_group)
        if self.vocab_sp:
            loss = gather_from_tensor_model_parallel_region_group(loss, self.sp_group)
        return loss.transpose(0, 1).contiguous()                                # per-token loss [b, s]


def construct_sequential_model(model, config):
    model_ = PipeSequential()
    model_.add_module("embeddings", GPTEmbeddings_(model))
    for i in range(config.num_hidden_layers):
        model_.add_module("layer_%d" % i, GPTLayers_(model, i))
    model_.add_module("prenorm", GPTPreNorm_(model))
    model_.add_module("cls", GPTCls_(model))
    return model_


class GPTModelInfo(ModelInfo):
    def __init__(self, config, args):
        super().__init__()
        seq_len, hidden = config.max_position_embeddings, config.hidden_size
        dt = mixed_precision_dtype(args.mixed_precision)
        shape = [[seq_len, -1, hidden]] if args.shape_order == "SBH" else [[-1, seq_len, hidden]]
        self.set_layernums([config.num_hidden_layers])
        self.set_shapes([shape])
        self.set_dtypes([[dt]])
        self.set_module_types(["embed"] + ["gpt_dec"] * config.num_hidden_layers + ["norm", "cls"])

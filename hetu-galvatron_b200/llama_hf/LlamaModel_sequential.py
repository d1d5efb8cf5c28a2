"""Sequential (pipeline-able) view of the Llama model (``galvatron/models/llama_hf/LlamaModel_sequential.py``)."""
import torch
import torch.nn as nn

from ..core.runtime.arguments import get_args
from ..core.runtime.hybrid_parallel_config import ModelInfo, mixed_precision_dtype
from ..core.runtime.pipeline import PipeSequential
from ..core.runtime.redistribute import zigzag_local as _zigzag_local
from ..core.runtime.tensor_parallel import (RMSNorm, copy_to_tensor_model_parallel_region_group,
                                            gather_from_tensor_model_parallel_region_group,
                                            linear_with_grad_accumulation_and_async_allreduce,
                                            scatter_to_sequence_parallel_region_group, vocab_parallel_cross_entropy)


def _size(g):
    return 1 if g is None else g.size


class LlamaEmbeddings_(nn.Module):
    def __init__(self, model):
        super().__init__()
        args = get_args()
        self.embed_tokens = model.model.embed_tokens
        self.sequence_parallel = args.sequence_parallel
        self.tp_group, self.sp_group, self.cp_group = (self.embed_tokens.tp_group, self.embed_tokens.sp_group,
                                                       self.embed_tokens.cp_group)
        # Ulysses on the embedding: each rank embeds its own sequence slice (:45-57)
        self.seq_group = self.sp_group if args.vocab_sp else None

    def forward(self, tokens, position_ids=None, attention_mask=None, labels=None):
        tokens = _zigzag_local(tokens, self.cp_group, self.seq_group)
        hidden_states = self.embed_tokens(tokens)
        hidden_states = hidden_states.transpose(0, 1).contiguous()           # [b, s, h] -> [s, b, h]
        if self.sequence_parallel:
            hidden_states = scatter_to_sequence_parallel_region_group(hidden_states, self.tp_group)
        return hidden_states


class LlamaLayers_(nn.Module):
    def __init__(self, model, layer_idx):
        super().__init__()
        self.layer = model.model.layers[layer_idx]
        self.layer_idx = layer_idx

    def forward(self, hidden_states, position_ids=None, attention_mask=None, labels=None):
        return self.layer(hidden_states, attention_mask=attention_mask)


class LlamaPreNorm_(nn.Module):
    def __init__(self, model, config):
        super().__init__()
        args = get_args()
        self.norm = RMSNorm(config.hidden_size, eps=config.rms_norm_eps, device="meta",
                            sequence_parallel=bool(args.sequence_parallel) and args.vocab_tp > 1 and not args.vocab_sp)

    def forward(self, hidden_states, position_ids=None, attention_mask=None, labels=None):
        return self.norm(hidden_states)


class LlamaLoss_(nn.Module):
    def __init__(self, lm_head, sequence_parallel, tp_group):
        super().__init__()
        self.weight = lm_head.weight
        self.init_std = lm_head.init_std
        self.tp_group = tp_group
        self.sequence_parallel = bool(sequence_parallel) and _size(tp_group) > 1   # :103-105

    def reset_parameters(self):
        nn.init.normal_(self.weight, mean=0.0, std=self.init_std)
        setattr(self.weight, "tensor_model_parallel", True)      # a column-parallel slice (layers.py:95-105)

    def forward(self, hidden_states):
        return linear_with_grad_accumulation_and_async_allreduce(
            input=hidden_states, weight=self.weight, bias=None, async_grad_allreduce=not self.sequence_parallel,
            sequence_parallel=self.sequence_parallel, tp_group=self.tp_group)


class LlamaCls_(nn.Module):
    def __init__(self, model, parallel_loss=True, half_entropy=True):
        super().__init__()
        args = get_args()
        self.sequence_parallel = args.sequence_parallel
        head = model.lm_head
        self.tp_group, self.sp_group, self.cp_group = head.tp_group, head.sp_group, head.cp_group
        self.lm_head = LlamaLoss_(head, self.sequence_parallel, self.tp_group)
        self.parallel_loss = parallel_loss
        self.half_entropy = half_entropy and not args.entropy_in_fp32
        self.vocab_sp = args.vocab_sp
        self.seq_group = self.sp_group if self.vocab_sp else None

    def forward(self, hidden_states, position_ids=None, attention_mask=None, labels=None):
        labels = _zigzag_local(labels, self.cp_group, self.seq_group)
        # (without SP the dgrad all-reduce of copy_to_tensor_model_parallel_region :146-147 happens inside the linear)
        logits_parallel = self.lm_head(hidden_states)                          # [s, b, V/t]
        labels = labels.transpose(0, 1).contiguous()                            # [b, s] -> [s, b]
        if not self.parallel_loss:
            logits = gather_from_tensor_model_parallel_region_group(logits_parallel, self.tp_group)
            logits = logits if self.half_entropy else logits.float()
            loss = torch.nn.functional.cross_entropy(logits.reshape(-1, logits.size(-1)), labels.reshape(-1))
            return loss
        logits_in = logits_parallel if self.half_entropy else logits_parallel.float()
        loss = vocab_parallel_cross_entropy(logits_in, labels, tp_group=self.tp_group)
        if self.vocab_sp:
            loss = gather_from_tensor_model_parallel_region_group(loss, self.sp_group)   # :180-181
        return loss.transpose(0, 1).contiguous()                                # per-token loss [b, s]


def construct_sequential_model(model, config):
    model_ = PipeSequential()
    model_.add_module("embeddings", LlamaEmbeddings_(model))
    for i in range(config.num_hidden_layers):
        model_.add_module("layer_%d" % i, LlamaLayers_(model, i))
    model_.add_module("prenorm", LlamaPreNorm_(model, config))
    model_.add_module("cls", LlamaCls_(model))
    return model_


class LlamaModelInfo(ModelInfo):
    def __init__(self, config, args):
        super().__init__()
        seq_len, hidden = config.max_position_embeddings, config.hidden_size
        dt = mixed_precision_dtype(args.mixed_precision)
        shape = [[seq_len, -1, hidden]] if args.shape_order == "SBH" else [[-1, seq_len, hidden]]
        self.set_layernums([config.num_hidden_layers])
        self.set_shapes([shape])
        self.set_dtypes([[dt]])
        self.set_module_types(["embed"] + ["gpt_dec"] * config.num_hidden_layers + ["norm", "cls"])

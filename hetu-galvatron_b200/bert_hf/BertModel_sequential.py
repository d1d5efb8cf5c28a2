"""Sequential (pipeline-able) view of the BERT model (``galvatron/models/bert_hf/BertModel_sequential.py``)."""
import torch
import torch.nn as nn

from ..core.runtime.arguments import get_args
from ..core.runtime.hybrid_parallel_config import ModelInfo, mixed_precision_dtype
from ..core.runtime.pipeline import PipeSequential
from ..core.runtime.tensor_parallel import (VocabUtility, gather_from_tensor_model_parallel_region_group,
                                            linear_with_grad_accumulation_and_async_allreduce,
                                            scatter_to_sequence_parallel_region_group, vocab_parallel_cross_entropy)
from ..core.runtime.tensor_parallel.random import SITE_EMBEDDING, bias_dropout_add, check_probability, site


def _size(g):
    return 1 if g is None else g.size


def _embedding_dropout(module, hidden_states):
    """Embedding dropout (hidden_dropout) on the SBH slice this rank holds after the vocab_sp slice and the Megatron-SP scatter, at
    global token positions."""
    if not (module.dropout_p > 0.0 and module.training):
        return hidden_states
    seq_base = module.seq_start_index if module.vocab_sp else 0
    if module.sequence_parallel and _size(module.tp_group) > 1:
        seq_base += module.tp_group.rank_in_group() * hidden_states.shape[0]
    return bias_dropout_add(hidden_states, None, None, module.dropout_p, site(0, SITE_EMBEDDING), seq_base)


def _seq_slice(args, sp_group):
    """Ulysses on the vocabulary rows: each rank embeds / scores its own sequence slice (:59-64,159-165)."""
    return VocabUtility.vocab_range_from_global_vocab_size(args.seq_length, sp_group.rank_in_group() if _size(sp_group) > 1 else 0,
                                                           _size(sp_group))


class BertWordEmbedding_(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.word_embeddings = model.bert.embeddings.word_embeddings

    def forward(self, input_ids):
        return self.word_embeddings(input_ids)


class BertTokenTypeEmbedding_(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.token_type_embeddings = model.bert.embeddings.token_type_embeddings

    def forward(self, token_type_ids):
        return self.token_type_embeddings(token_type_ids)


class BertPositionEmbedding_(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.position_embeddings = model.bert.embeddings.position_embeddings

    def forward(self, position_ids):
        return self.position_embeddings(position_ids)


class BertEmbeddings_(nn.Module):
    def __init__(self, model):
        super().__init__()
        args = get_args()
        self.word_embeddings, self.token_type_embeddings = BertWordEmbedding_(model), BertTokenTypeEmbedding_(model)
        self.position_embeddings = BertPositionEmbedding_(model)
        self.LayerNorm = model.bert.embeddings.LayerNorm
        self.sequence_parallel = args.sequence_parallel
        self.tp_group = self.word_embeddings.word_embeddings.tp_group
        self.sp_group = self.word_embeddings.word_embeddings.sp_group
        self.vocab_sp = args.vocab_sp
        if self.vocab_sp:
            self.seq_start_index, self.seq_end_index = _seq_slice(args, self.sp_group)
        self.dropout_p = check_probability(getattr(args, "hidden_dropout", 0.0), "hidden_dropout")     # after the LayerNorm, :100-102

    def forward(self, input_ids, token_type_ids=None, position_ids=None, attention_mask=None, labels=None):
        if position_ids is None:
            position_ids = torch.arange(input_ids.size(1), dtype=torch.long, device=input_ids.device).unsqueeze(0).expand_as(input_ids)
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        if self.vocab_sp:
            sl = slice(self.seq_start_index, self.seq_end_index)
            input_ids, token_type_ids, position_ids = [t[:, sl].contiguous() for t in (input_ids, token_type_ids, position_ids)]
        embeddings = self.word_embeddings(input_ids) + self.position_embeddings(position_ids)
        embeddings = embeddings + self.token_type_embeddings(token_type_ids).to(embeddings.dtype)
        embeddings = self.LayerNorm(embeddings)
        embeddings = embeddings.transpose(0, 1).contiguous()                  # [b, s, h] -> [s, b, h]
        if self.sequence_parallel:
            embeddings = scatter_to_sequence_parallel_region_group(embeddings, self.tp_group)
        return _embedding_dropout(self, embeddings)


class BertLayers_(nn.Module):
    def __init__(self, model, layer_idx):
        super().__init__()
        self.layer = model.bert.encoder.layer[layer_idx]

    def forward(self, hidden_states, token_type_ids=None, position_ids=None, attention_mask=None, labels=None):
        # attention_mask [b, s] over the keys (True / 1 = a real token).  The reference expands it to the [b, 1, s, s] product mask
        # (:12-18); rows of padded QUERIES differ between the two forms, but a padded position's output never reaches a real token
        # and its own loss term is a function of its own (masked-out) row only -- the fused attention takes the key mask.
        return self.layer(hidden_states, attention_mask=attention_mask)


class BertLoss_(nn.Module):
    def __init__(self, decoder, sequence_parallel, tp_group):
        super().__init__()
        self.weight, self.bias = decoder.weight, decoder.bias
        self.init_std = decoder.init_std
        self.tp_group = tp_group
        self.sequence_parallel = bool(sequence_parallel) and _size(tp_group) > 1

    def reset_parameters(self):
        nn.init.normal_(self.weight, mean=0.0, std=self.init_std)
        nn.init.zeros_(self.bias)
        for p in (self.weight, self.bias):
            setattr(p, "tensor_model_parallel", True)

    def forward(self, hidden_states):
        # the dgrad all-reduce (no SP) happens inside the linear, so the transform in front of it sees the FULL gradient on every
        # tensor-parallel rank (the reference all-reduces before the transform, :175-181, leaving its replicas with partial sums)
        return linear_with_grad_accumulation_and_async_allreduce(
            input=hidden_states, weight=self.weight, bias=self.bias, async_grad_allreduce=not self.sequence_parallel,
            sequence_parallel=self.sequence_parallel, tp_group=self.tp_group)


class BertMLMCls_(nn.Module):
    def __init__(self, model, parallel_loss=True, half_entropy=True):
        super().__init__()
        args = get_args()
        self.sequence_parallel = args.sequence_parallel
        dec = model.cls.predictions.decoder
        self.tp_group, self.sp_group = dec.tp_group, dec.sp_group
        self.transform = model.cls.predictions.transform
        self.lm_head = BertLoss_(dec, self.sequence_parallel, self.tp_group)
        self.half_entropy = half_entropy and not args.entropy_in_fp32
        self.vocab_sp = args.vocab_sp
        if self.vocab_sp:
            self.seq_start_index, self.seq_end_index = _seq_slice(args, self.sp_group)

    def forward(self, hidden_states, token_type_ids=None, position_ids=None, attention_mask=None, labels=None):
        if self.vocab_sp:
            labels = labels[:, self.seq_start_index:self.seq_end_index].contiguous()
        logits_parallel = self.lm_head(self.transform(hidden_states))          # [s, b, V/t]
        labels = labels.transpose(0, 1).contiguous()                            # [b, s] -> [s, b]
        logits_in = logits_parallel if self.half_entropy else logits_parallel.float()
        loss = vocab_parallel_cross_entropy(logits_in, labels, tp_group=self.tp_group)
        if self.vocab_sp:
            loss = gather_from_tensor_model_parallel_region_group(loss, self.sp_group)
        return loss.transpose(0, 1).contiguous()                                # per-token loss [b, s]


def construct_sequential_model(model, config):
    model_ = PipeSequential()
    model_.add_module("embeddings", BertEmbeddings_(model))
    for i in range(config.num_hidden_layers):
        model_.add_module("layer_%d" % i, BertLayers_(model, i))
    model_.add_module("cls", BertMLMCls_(model))
    return model_


class BertModelInfo(ModelInfo):
    def __init__(self, config, args):
        super().__init__()
        seq_len, hidden = config.max_position_embeddings, config.hidden_size
        dt = mixed_precision_dtype(args.mixed_precision)
        shape = [[seq_len, -1, hidden]] if args.shape_order == "SBH" else [[-1, seq_len, hidden]]
        self.set_layernums([config.num_hidden_layers])
        self.set_shapes([shape])
        self.set_dtypes([[dt]])
        self.set_module_types(["embed"] + ["bert_enc"] * config.num_hidden_layers + ["mlm_head"])

"""Sequential (pipeline-able) view of the T5 model (``galvatron/models/T5/T5Model_sequential.py``).

Rows: embed_1, t5_enc x L_enc, pre_norm_1, embed_2, t5_dec x L_dec, pre_norm_2, cls.  The first stage takes the encoder tokens; the
decoder tokens, the labels and the reference's three masks arrive as keyword arguments of every row (the masks are not used: the
reference trains on its flash-attention path, which ignores them).  Every decoder row receives the encoder output and passes it on
unchanged with its own hidden states, so a stage boundary inside the decoder carries two tensors, [s_enc, b, h] and [s_dec, b, h];
one inside the encoder, or right after it, carries one."""
import torch.nn as nn

from ..core.runtime.arguments import get_args
from ..core.runtime.hybrid_parallel_config import ModelInfo, mixed_precision_dtype
from ..core.runtime.pipeline import PipeSequential
from ..core.runtime.tensor_parallel import scatter_to_sequence_parallel_region_group, vocab_parallel_cross_entropy
from ..gpt_hf.GPTModel_sequential import GPTLoss_


class _Embeddings(nn.Module):
    def __init__(self, embedding):
        super().__init__()
        self.embeddings = embedding
        self.sequence_parallel = get_args().sequence_parallel
        self.tp_group = embedding.tp_group

    def embed(self, tokens):
        hidden_states = self.embeddings(tokens).transpose(0, 1).contiguous()          # [b, s, h] -> [s, b, h]
        if self.sequence_parallel:
            hidden_states = scatter_to_sequence_parallel_region_group(hidden_states, self.tp_group)
        return hidden_states


class T5EncoderEmbeddings_(_Embeddings):
    def __init__(self, model):
        super().__init__(model.shared)

    def forward(self, enc_tokens, dec_tokens=None, enc_attn_mask=None, dec_attn_mask=None, enc_dec_attn_mask=None, dec_labels=None):
        return self.embed(enc_tokens)


class T5DecoderEmbeddings_(_Embeddings):
    def __init__(self, model):
        super().__init__(model.dec_shared)

    def forward(self, enc_hidden_states, dec_tokens=None, enc_attn_mask=None, dec_attn_mask=None, enc_dec_attn_mask=None,
                dec_labels=None):
        return enc_hidden_states, self.embed(dec_tokens)


class T5EncoderLayers_(nn.Module):
    def __init__(self, model, layer_idx):
        super().__init__()
        self.layer = model.encoder[layer_idx]

    def forward(self, hidden_states, dec_tokens=None, enc_attn_mask=None, dec_attn_mask=None, enc_dec_attn_mask=None, dec_labels=None):
        return self.layer(hidden_states)


class T5DecoderLayers_(nn.Module):
    def __init__(self, model, layer_idx):
        super().__init__()
        self.layer = model.decoder[layer_idx]

    def forward(self, enc_hidden_states, dec_hidden_states, dec_tokens=None, enc_attn_mask=None, dec_attn_mask=None,
                enc_dec_attn_mask=None, dec_labels=None):
        return self.layer(enc_hidden_states, dec_hidden_states)


class T5EncoderPreNorm_(nn.Module):
    def __init__(self, model):
        super().__init__()
        self.LayerNorm = model.enc_final_norm

    def forward(self, enc_hidden_states, dec_tokens=None, enc_attn_mask=None, dec_attn_mask=None, enc_dec_attn_mask=None,
                dec_labels=None):
        return self.LayerNorm(enc_hidden_states)


class T5DecoderPreNorm_(nn.Module):
    """The decoder's final norm; the encoder output ends here (the head does not read it)."""

    def __init__(self, model):
        super().__init__()
        self.LayerNorm = model.dec_final_norm

    def forward(self, enc_hidden_states, dec_hidden_states, dec_tokens=None, enc_attn_mask=None, dec_attn_mask=None,
                enc_dec_attn_mask=None, dec_labels=None):
        return self.LayerNorm(dec_hidden_states)


class T5Cls_(nn.Module):
    """Bias-free lm_head (untied) + vocab-parallel cross entropy per token -> [b, s_dec] fp32.  A label -1 (padding) is scored with
    target logit 0, as Megatron's cross entropy does; the caller's loss function masks it."""

    def __init__(self, model):
        super().__init__()
        args = get_args()
        head = model.lm_head
        self.tp_group = head.tp_group
        self.lm_head = GPTLoss_(head, args.sequence_parallel, self.tp_group)
        self.half_entropy = not args.entropy_in_fp32

    def forward(self, hidden_states, dec_tokens=None, enc_attn_mask=None, dec_attn_mask=None, enc_dec_attn_mask=None, dec_labels=None):
        logits_parallel = self.lm_head(hidden_states)                                 # [s, b, V/t]
        labels = dec_labels.transpose(0, 1).contiguous()                              # [b, s] -> [s, b]
        logits_in = logits_parallel if self.half_entropy else logits_parallel.float()
        loss = vocab_parallel_cross_entropy(logits_in, labels, tp_group=self.tp_group)
        return loss.transpose(0, 1).contiguous()


def construct_sequential_model(model, config):
    model_ = PipeSequential()
    model_.add_module("encoder_embeddings", T5EncoderEmbeddings_(model))
    for i in range(config.num_layers):
        model_.add_module("encoder_layer_%d" % i, T5EncoderLayers_(model, i))
    model_.add_module("encoder_pre_norm", T5EncoderPreNorm_(model))
    model_.add_module("decoder_embeddings", T5DecoderEmbeddings_(model))
    for i in range(config.num_decoder_layers):
        model_.add_module("decoder_layer_%d" % i, T5DecoderLayers_(model, i))
    model_.add_module("decoder_pre_norm", T5DecoderPreNorm_(model))
    model_.add_module("cls", T5Cls_(model))
    return model_


class T5ModelInfo(ModelInfo):
    def __init__(self, config, args):
        super().__init__()
        s_enc, s_dec, h = config.n_positions, config.n_decoder_positions, config.hidden_size
        dt = mixed_precision_dtype(args.mixed_precision)
        if args.shape_order == "SBH":
            shapes = [[[s_enc, -1, h]], [[s_enc, -1, h], [s_dec, -1, h]]]
        else:
            shapes = [[[-1, s_enc, h]], [[-1, s_enc, h], [-1, s_dec, h]]]
        self.set_layernums([config.num_layers, config.num_decoder_layers])
        self.set_shapes(shapes)
        self.set_dtypes([[dt], [dt, dt]])
        self.set_module_types(["embed_1"] + ["t5_enc"] * config.num_layers + ["pre_norm_1", "embed_2"]
                              + ["t5_dec"] * config.num_decoder_layers + ["pre_norm_2", "cls"])

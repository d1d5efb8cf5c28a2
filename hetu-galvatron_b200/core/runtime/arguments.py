"""Runtime arguments: the flags of ``galvatron/core/runtime/arguments.py:1-215`` that steer the hot path, plus the
process-wide ``get_args()`` singleton the reference reads inside layers and wrappers (``parallel.py:59,112``,
``redistribute.py:49-51``, ``pipeline.py:146-151``).  The reference builds this namespace through Megatron's
argparse stack (``core/arguments.py:8-30`` -> ``initialize_megatron``); that control plane is out of scope, so the
namespace is built directly (from keyword arguments or an argv list) with the same names and defaults.
"""
import argparse
import types

_ARGS = None

# name -> default, as in the reference (file:line in galvatron/core/runtime/arguments.py unless noted)
DEFAULTS = dict(
    initialize_on_meta=0,                # :23
    global_train_batch_size=32,          # :29
    dropout_prob=0.0,                    # :30 default 0.1; read by no layer here (the GPT / BERT families take hidden_dropout /
                                         # attention_dropout below); > 0 still makes the checkpoint wrapper preserve the RNG state
    # megatron's names; the GPT / BERT families set them from the HF config (resid_pdrop / attn_pdrop, hidden_dropout_prob /
    # attention_probs_dropout_prob) as the reference's overwrite_megatron_args does.  Deviation on purpose: 0 by default (the
    # reference gets 0.1 from the HF config defaults), so no run changes unless it asks for dropout.  Llama keeps 0 (as the reference).
    hidden_dropout=0.0,                  # embedding output and MLP-block output (megatron --hidden-dropout)
    attention_dropout=0.0,               # attention probabilities AND the attention-block output (megatron --attention-dropout;
                                         # the reference applies it at both, GPTModel_tensor_parallel.py:31-39)
    adam_weight_decay=0.01,              # :32
    pp_deg=2,                            # :52
    global_cp_deg=1,                     # :60
    global_tp_deg=-1,                    # :75
    chunks=-1,                           # :82
    global_tp_consec=-1,                 # :88
    sdp=0,                               # :91
    galvatron_config_path=None,          # :98
    global_checkpoint=0,                 # :103
    mixed_precision="bf16",              # :105
    pipeline_type="gpipe",               # :112
    default_dp_type="ddp",               # :119
    embed_sdp=0,                         # :126
    profile_forward=0,                   # :133
    shape_order="SBH",                   # :154
    vocab_tp=1,                          # :161
    vocab_cp=1,                          # :168
    use_ulysses=False,                   # :175
    async_grad_reduce=True,              # :180 (--no_async_grad_reduce stores False)
    reduce_in_fp32=False,                # :187
    entropy_in_fp32=False,               # :192
    distributed_checkpoint=False,        # :197
    load=None,                           # megatron --load: checkpoint directory (HF-layered, or distributed with the flag above)
    load_iteration=0,                    # :204
    save=None,                           # megatron --save: reserves the peer-visible gather buffer checkpoint export needs
    lr=1e-4,                             # :209
    local_rank=0,                        # :211
    # megatron-side flags the layer code reads
    sequence_parallel=False,             # megatron --sequence-parallel (layers.py:399-413)
    clone_scatter_output_in_embedding=True,
    seq_length=1024,
    hidden_size=768,
    ffn_hidden_size=3072,
    num_attention_heads=12,
    num_query_groups=None,
    group_query_attention=False,
    padded_vocab_size=50304,
    make_vocab_size_divisible_by=128,
    norm_epsilon=1e-5,
    init_method_std=0.02,
    rotary_base=10000.0,
    adam_beta1=0.9, adam_beta2=0.999, adam_eps=1e-8,
    seed=1234,
    vocab_sp=0,
    # this runtime's own knobs
    arena_bytes=0,                       # 0 = size the symmetric arena from the model
    fused_optimizer=False,               # AdamW inside the gradient reduce-scatter kernel (SURVEY 8f-3)
    recompute_activations=False,         # opt-in: GEMMs keep what their input was made from (SwiGLU / RMSNorm inputs) and redo the
                                         # elementwise pass in backward -- 352 MiB less per 8B layer at seq 8192
    untie_embeddings_and_output_weights=True,   # megatron's flag; False ties them (C14, grad_reduce.py:98-131; the reference's GPT default)
    zero3_pool_slots=4,                  # rotating peer-visible buffers the zero3 layers of one group gather into (0 = one per layer)
    cp_comm="allgather",                 # context parallelism's K/V exchange: "allgather" (whole-sequence K/V per layer, one gather) or
                                         # "ring" (only the local s/c rows kept; blocks travel between neighbours, c-1 hops)
)


# options that are NOT defaults of the runtime but that model families / drivers legitimately attach to the namespace
_EXTRA = {"model_size", "set_model_config_manually", "set_layernum_manually", "set_seqlen_manually", "vocab_size", "num_hidden_layers",
          "kv_channels", "train_iters", "train_samples", "lr_decay_style", "lr_decay_iters", "lr_decay_samples", "lr_warmup_iters",
          "lr_warmup_samples", "lr_warmup_fraction", "lr_warmup_init", "min_lr", "start_weight_decay", "end_weight_decay",
          "weight_decay_incr_style", "use_checkpoint_opt_param_scheduler", "override_opt_param_scheduler", "num_layers",
          "max_position_embeddings", "clip_grad", "layernorm_type", "activation", "add_bias", "position_embedding_type", "causal"}
# explicit types of the options whose default is None (argparse would otherwise hand them over as strings)
_NONE_TYPES = {"num_query_groups": int, "galvatron_config_path": str, "load": str, "save": str}


def make_args(**overrides):
    unknown = sorted(set(overrides) - set(DEFAULTS) - _EXTRA)
    if unknown:
        raise TypeError("unknown runtime argument(s) %s (a typo? known: the keys of arguments.DEFAULTS)" % ", ".join(unknown))
    ns = types.SimpleNamespace(**DEFAULTS)
    for k, v in overrides.items():
        setattr(ns, k, v)
    return ns


def parse_args(argv):
    p = argparse.ArgumentParser("hetu-galvatron_b200 runtime", allow_abbrev=False)
    for k, v in DEFAULTS.items():
        if isinstance(v, bool):
            p.add_argument("--" + k, type=lambda s: s.lower() in ("1", "true", "yes"), default=v)
        elif v is None:
            p.add_argument("--" + k, type=_NONE_TYPES.get(k, str), default=None)
        else:
            p.add_argument("--" + k, type=type(v), default=v)
    p.add_argument("--no_async_grad_reduce", action="store_false", dest="async_grad_reduce")
    p.add_argument("--use-ulysses", action="store_true", dest="use_ulysses")
    return types.SimpleNamespace(**vars(p.parse_args(argv)))


def set_args(args):
    global _ARGS
    _ARGS = args
    return args


def get_args():
    if _ARGS is None:
        raise RuntimeError("runtime arguments are not initialised: call initialize_galvatron()/set_args() first")
    return _ARGS


def initialize_galvatron(model_args=None, mode="train_dist", argv=None, **overrides):
    """``galvatron/core/arguments.py:8-30``: build the args namespace and install it as the singleton."""
    args = parse_args(argv) if argv is not None else make_args(**overrides)
    if model_args is not None:
        for k, v in (vars(model_args) if not isinstance(model_args, dict) else model_args).items():
            setattr(args, k, v)
    return set_args(args)

"""Entry points of the family (``galvatron/models/llama_hf/LlamaModel_hybrid_parallel.py``)."""
from ..core.runtime.hybrid_parallel_config import get_hybrid_parallel_configs_api
from ..core.runtime.hybrid_parallel_model import construct_hybrid_parallel_model_api
from .LlamaModel_checkpoint import load_llama_module
from .LlamaModel_sequential import LlamaCls_, LlamaEmbeddings_, LlamaModelInfo, LlamaPreNorm_, construct_sequential_model
from .LlamaModel_tensor_parallel import LlamaLayer_tp, LlamaSkeleton, construct_tensor_parallel_model
from .meta_configs import config_from_meta, set_model_config


def get_hybrid_parallel_configs(model_config, training_args):
    return get_hybrid_parallel_configs_api(model_config, training_args, LlamaModelInfo)


def construct_hybrid_parallel_model(model, model_config, training_args, hybrid_parallel_configs):
    return construct_hybrid_parallel_model_api(
        model, model_config, training_args, hybrid_parallel_configs, LlamaModelInfo, construct_sequential_model,
        construct_tensor_parallel_model, wrap_block_name=[LlamaLayer_tp], wrap_checkpoint_block_name=[LlamaLayer_tp],
        wrap_other_block_name=[LlamaEmbeddings_, LlamaPreNorm_, LlamaCls_], layernorm_name=["LayerNorm", "norm"],
        all_block_name=[LlamaEmbeddings_, LlamaLayer_tp, LlamaPreNorm_, LlamaCls_], load_module_func=load_llama_module)


def get_llama_config(args, overwrite_args=True):
    config = config_from_meta(args.model_size)
    return set_model_config(config, args, overwrite_args)


def estimate_arena_bytes(config, args, hp_configs):
    """Bytes of peer-visible memory this rank needs: bf16 gathered params + bf16 unsharded grads of its stage's layers,
    plus activation staging per communicating group and the pipeline receive slots."""
    from ..core.runtime import world as _world
    h, f, V = config.hidden_size, config.intermediate_size, args.padded_vocab_size
    hn = h // config.num_attention_heads
    layer = (config.num_attention_heads + 2 * config.num_key_value_heads) * hn * h + config.num_attention_heads * hn * h \
        + 3 * f * h + 2 * h
    pp = hp_configs["pp_deg"]
    esz = 4 if args.mixed_precision == "fp32" else 2
    gsz = 4 if getattr(args, "reduce_in_fp32", False) else esz
    world = _world.get_world_size()
    slots = int(getattr(args, "zero3_pool_slots", 0))
    chunks = args.chunks if args.chunks > 0 else 1
    pool_grads = chunks == 1 or not args.async_grad_reduce
    vocab = V * h // max(1, args.vocab_tp)
    embed_zero3 = bool(getattr(args, "embed_sdp", 0)) or args.default_dp_type == "zero3"
    worst_stage = 0
    for stage in range(pp):
        fixed_w = fixed_g = 0           # layers that keep their own buffers
        pooled = 0                      # largest pooled layer of the stage
        # Ulysses layers keep whole parameters (tp_sizes_enc is then the sequence-parallel degree) and shard them over
        # the DP x SP x CP group (comm_groups.py:475-483)
        use_sp = hp_configs.get("use_sp") or [0] * len(hp_configs["tp_sizes_enc"])
        rows = [(layer if sp else layer // tp, (dt == 1 or args.default_dp_type == "zero3"), 1 if sp else tp * max(1, cp))
                for tp, cp, dt, rank, sp in zip(hp_configs["tp_sizes_enc"], hp_configs["cp_sizes_enc"], hp_configs["dp_types_enc"],
                                                hp_configs["pp_ranks_enc"], use_sp) if rank == stage]
        if stage == 0:
            rows.append((vocab, embed_zero3, max(1, args.vocab_tp)))
        if stage == pp - 1:
            rows.append((vocab, embed_zero3, max(1, args.vocab_tp)))
            rows.append((h, embed_zero3, max(1, args.vocab_tp)))
        for n, zero3, model_par in rows:
            sharded = world // pp // model_par > 1
            if zero3 and sharded and slots > 0:
                pooled = max(pooled, n)
                fixed_g += 0 if pool_grads else n
            else:
                fixed_w += n
                fixed_g += n
        total_stage = fixed_w * esz + fixed_g * gsz + pooled * (slots * esz + (max(2, slots - 1) * gsz if pool_grads else 0))
        worst_stage = max(worst_stage, total_stage)
    total = worst_stage
    min_dp = max(1, world // pp // max(max(hp_configs["tp_sizes_enc"]), args.vocab_tp) // max(hp_configs["cp_sizes_enc"]))
    mbs = -(-args.global_train_batch_size // min_dp // max(1, args.chunks if args.chunks > 0 else 1))
    act = int(config.max_position_embeddings * mbs * h * esz * 1.5) + (1 << 20)
    n_groups = 0 if world == 1 else 8
    return int(total * 1.02) + act * n_groups + 4 * act + _cp_ring_bytes(config, args, hp_configs, mbs) + (64 << 20)


def _cp_ring_bytes(config, args, hp_configs, mbs):
    """cp_comm="ring": the receive slots hybrid_parallel_model reserves per cp group, 24 B per element of the largest local K block
    (microbatch x s/c x K/V heads at the attention call x head dim) -- for MHA (GPT) four times the activation staging of a group at
    c = 2.  Summed over the distinct (tp|sp, cp) layer strategies, each of which may have a cp group of its own."""
    from ..core.runtime.tensor_parallel.transformer import cp_comm_mode
    if cp_comm_mode() != "ring":
        return 0
    n, ng = config.num_attention_heads, config.num_key_value_heads
    hn, seq = config.hidden_size // n, config.max_position_embeddings
    use_sp = hp_configs.get("use_sp") or [0] * len(hp_configs["tp_sizes_enc"])
    total = 0
    for deg, cp, sp in set(zip(hp_configs["tp_sizes_enc"], hp_configs["cp_sizes_enc"], use_sp)):
        if cp > 1:
            # ParallelAttention.kv_heads_attn: Ulysses (degree ``deg``) leaves ng/p heads, or n/p when K/V are replicated first
            kv = ((ng if ng % deg == 0 else n) // deg) if sp else ng // deg
            total += 24 * mbs * (seq // cp) * kv * hn
    return total


def llama_model_hp(config, args):
    hybrid_parallel_configs = get_hybrid_parallel_configs(model_config=config, training_args=args)
    if not getattr(args, "arena_bytes", 0):
        args.arena_bytes = estimate_arena_bytes(config, args, hybrid_parallel_configs)
    skeleton = LlamaSkeleton(config)
    return construct_hybrid_parallel_model(model=skeleton, model_config=config, training_args=args,
                                           hybrid_parallel_configs=hybrid_parallel_configs)

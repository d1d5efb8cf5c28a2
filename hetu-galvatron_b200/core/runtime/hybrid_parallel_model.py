"""``construct_hybrid_parallel_model_api`` -- the drop-in boundary: per-layer strategy in, runnable hybrid-parallel model out.

Same signature, callback contracts and 7 construction steps as
``galvatron/core/runtime/hybrid_parallel_model.py:165-326`` and the same ``GalvatronModel.forward_backward`` (:42-70).
What is gone: the FSDP monkey-patches (:186-189) -- the per-layer ShardedUnit is an explicit state machine -- and every
``torch.distributed.new_group`` (groups are rank lists resolved by the peer-memory runtime).
"""
import inspect

import numpy as np
import torch
from torch import Tensor, nn

from . import world as _world
from .arguments import get_args
from .backend import get_backend
from .comm_groups import gen_comm_groups
from .hybrid_parallel_config import (check_hp_config, get_chunks, hp_config_whole_model, layer_shapes_dtypes_whole_model,
                                     mixed_precision_dtype)
from .parallel import finalize_pools, wrap_modules_relocation
from .sample_layout import derive_sample_layouts
from .tensor_parallel import random as dropout_random
from .tensor_parallel.transformer import ParallelAttention, cp_comm_mode


class GalvatronModel(nn.Module):
    def __init__(self, hp_model):
        super().__init__()
        self.args = get_args()
        self.model = hp_model
        self.iter = 0

    def forward_backward(self, batch, iter=None, profiler=None, loss_func=None, **kwargs):
        args, model = self.args, self.model
        self.iter = iter if iter is not None else self.iter
        if loss_func is not None:
            if len(batch) == 1 and isinstance(batch[0], Tensor):
                batch = [batch, [self.fake_tensor(batch[0])]]
            assert isinstance(batch, (tuple, list)) and isinstance(batch[0], (tuple, list)) and isinstance(batch[1], (tuple, list))
        else:
            loss_func = self.fake_loss_func
            assert isinstance(batch, (tuple, list))
            batch = [batch, [self.fake_tensor(batch[0])]]
        # dropout coordinates of this step: the iteration, the global index of this rank's first sample (the batch is split
        # contiguously over the data-parallel ranks of the vocabulary rows), and which of the samples each row holds
        dp = getattr(self, "vtp_data_group", None)
        local = next((t.shape[0] for t in batch[0] if torch.is_tensor(t)), 0)
        dropout_random.begin_iteration(getattr(args, "seed", 0), self.iter, (dp.rank_in_group() if dp is not None else 0) * local,
                                       getattr(self, "sample_layouts", None), local)
        if args.pp_deg > 1:
            if args.pipeline_type == "gpipe":
                loss = model.gpipe_forward(batch, loss_func, **kwargs)
                if profiler is not None:
                    profiler.profile_memory(self.iter, "After Forward")
                model.gpipe_backward()
            elif args.pipeline_type == "pipedream_flush":
                loss = model.pipedream_flush_forward_backward(batch, loss_func, **kwargs)
            else:
                raise ValueError("unknown pipeline_type %r" % args.pipeline_type)
        else:
            loss = model.no_pipeline_forward_backward(batch, loss_func, forward_only=bool(args.profile_forward),
                                                      profiler=profiler, iter=self.iter, **kwargs)
        self.iter += 1
        return self.loss_to_cpu(loss)

    def fake_tensor(self, x):
        return torch.zeros([x.shape[0], 1], dtype=x.dtype, device=x.device)

    def fake_loss_func(self, labels, outputs):
        """Mean over the local microbatch's tokens (hybrid_parallel_model.py:75-79)."""
        if torch.numel(outputs[0]) > 1:
            loss = outputs[0].mean()
            return loss, loss.clone().detach()
        return outputs[0], outputs[0].clone().detach()

    def loss_to_cpu(self, loss):
        if isinstance(loss, (list, tuple)):  # average loss of the microbatches
            if len(loss) == 0:
                return None
            return float(np.mean([l.item() for l in loss]))
        return loss.item()

    # the optimizer-facing parameters are the fp32 flat (sharded) masters, as with FSDP's FlatParameter
    def parameters(self, recurse=True):
        for u in self.model.units:
            yield u.flat_param

    def named_parameters(self, prefix="", recurse=True, remove_duplicate=True):
        for u in self.model.units:
            yield (prefix + ("." if prefix else "") + u.name + ".flat_param", u.flat_param)


def _call_tp_constructor(fn, model, config, tp_groups, sp_groups, cp_groups):
    """HEAD calls this with 5 positional args (hybrid_parallel_model.py:248-250) but only llama_hf accepts 5 -- accept
    both arities (SURVEY 8g)."""
    try:
        n_pos = len([p for p in inspect.signature(fn).parameters.values()
                     if p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD)])
    except (TypeError, ValueError):
        n_pos = 5
    if n_pos >= 5:
        return fn(model, config, tp_groups, sp_groups, cp_groups)
    if n_pos == 4:
        return fn(model, config, tp_groups, sp_groups)
    return fn(model, config, tp_groups)


def construct_hybrid_parallel_model_api(model, model_config, training_args, hybrid_parallel_configs, model_info,
                                        construct_sequential_model, construct_tensor_parallel_model, wrap_block_name=None,
                                        wrap_checkpoint_block_name=None, wrap_other_block_name=None, tied_wte_attr_names=None,
                                        layernorm_name=[], all_block_name=None, load_module_func=None, meta_init_buffer=True):
    if wrap_checkpoint_block_name is None:
        wrap_checkpoint_block_name = wrap_block_name
    config, args, hp_configs = model_config, training_args, hybrid_parallel_configs
    cp_comm_mode()          # an unknown cp_comm raises ValueError here, before any group or buffer exists
    be = get_backend()

    info = model_info(config, args)
    module_types, layernum_list = info.module_types(), info.layernums()
    check_hp_config(hp_configs, layernum_list)
    shapes_whole, dtypes_whole = layer_shapes_dtypes_whole_model(module_types, layernum_list, info.shapes(), info.dtypes())
    hp_whole = hp_config_whole_model(module_types, hp_configs, embed_sdp=args.embed_sdp, embed_ckpt=0, vocab_tp=args.vocab_tp,
                                     vocab_sp=args.vocab_sp, vocab_cp=getattr(args, "vocab_cp", 1))

    # Ulysses rows keep the sequence split across their group; every other row does so only under Megatron sequence
    # parallelism.  The relocation between the two layouts is keyed on --sequence-parallel (redistribute.py:60,121,282,335), so
    # without it a strategy that mixes them is silently wrong in the reference (its own hybrid tests set the flag,
    # tests/core/test_hybrid.py:45).  Refuse it.
    sp_rows = [s > 1 for s in hp_whole["sp_sizes_whole"]]
    if any(sp_rows) and not all(sp_rows) and not args.sequence_parallel:
        raise ValueError("this strategy mixes Ulysses layers (use_sp=1) with tensor-parallel / data-parallel rows: "
                         "it needs --sequence-parallel (activations must be sequence-split on both sides of a relocation)")

    cp_rows = set(hp_whole["cp_sizes_whole"])
    if len(cp_rows) > 1 and not args.sequence_parallel:
        raise ValueError("this strategy changes the context-parallel degree between rows: it needs --sequence-parallel "
                         "(the relocation re-splits the sequence only under that flag, redistribute.py:60,121)")

    # which samples each of this rank's rows holds once the relocations have split / gathered the batch (dropout draws there)
    sample_layouts = derive_sample_layouts(hp_whole, _world.get_rank(), _world.get_world_size())

    # [Step 0] communication groups (pure rank lists)
    (pp_group, tp_groups_whole, sp_groups_whole, cp_groups_whole, dp_groups_whole, seq_data_groups_whole,
     allgather_tp_sp_groups_whole, split_tp_sp_groups_whole, allgather_cp_groups_whole, split_cp_groups_whole,
     allgather_tp_sp_cp_groups_whole, split_tp_sp_cp_groups_whole, fused_allgather_groups_whole, fused_split_groups_whole,
     embedding_group, vtp_data_group) = gen_comm_groups(hp_whole["tp_sizes_whole"], hp_whole["sp_sizes_whole"],
                                                        hp_whole["cp_sizes_whole"], hp_whole["pp_deg"],
                                                        hp_whole["tp_consec_whole"],
                                                        show_rank=0 if getattr(args, "local_rank", 1) == 0 else -1)

    # [Step 1] tensor-parallel model through the family's callback
    if args.shape_order != "SBH":
        assert not args.use_ulysses, "FA model does not support ulysses!"
        model = construct_tensor_parallel_model(model, config, tp_groups_whole)
    else:
        model = _call_tp_constructor(construct_tensor_parallel_model, model, config, tp_groups_whole, sp_groups_whole,
                                     cp_groups_whole)

    # [Step 2] sequential model
    model = construct_sequential_model(model, config)

    # [Step 3] relocation wrappers where consecutive layers disagree on (tp|sp, cp)
    model = wrap_modules_relocation(model, allgather_tp_sp_groups_whole, allgather_cp_groups_whole,
                                    allgather_tp_sp_cp_groups_whole, split_tp_sp_groups_whole, split_cp_groups_whole,
                                    split_tp_sp_cp_groups_whole, fused_allgather_groups_whole, fused_split_groups_whole)

    # [Step 4] pipeline module: keeps this stage's layers
    from .pipeline import PipelineParallel
    chunks = get_chunks(args)
    hp_model = PipelineParallel(model=model, model_ranks=hp_whole["pp_ranks_whole"], layer_output_tensor_shapes=shapes_whole,
                                layer_output_tensor_dtypes=dtypes_whole, layer_dp_sizes=hp_whole["dp_sizes_whole"],
                                layer_tp_sizes=hp_whole["tp_sizes_whole"], layer_sp_sizes=hp_whole["sp_sizes_whole"],
                                layer_cp_sizes=hp_whole["cp_sizes_whole"], chunks=chunks, process_group=pp_group.ranks,
                                embedding_group=embedding_group, info=False, tied_wte_attr_names=tied_wte_attr_names)

    # [Step 5] per-layer sharded data parallelism over the SDP groups
    hp_model.wrap_pipeline_modules_data_parallel(hp_whole["dp_types_whole"], seq_data_groups_whole, module_types=module_types,
                                                 mixed_precision=mixed_precision_dtype(args.mixed_precision),
                                                 wrap_block_name=wrap_block_name, wrap_other_block_name=wrap_other_block_name,
                                                 tp_groups=tp_groups_whole, all_block_name=all_block_name,
                                                 load_module_func=load_module_func)

    # [Step 6] activation checkpointing
    hp_model.wrap_pipeline_modules_checkpoint(hp_whole["checkpoint_flags_whole"], wrap_block_name=wrap_checkpoint_block_name)

    # peer-visible activation staging for every group this rank communicates over, pipeline transport slots, then one
    # exchange of arena offsets for the whole job (replaces all NCCL communicator bootstraps)
    _reserve_activation_staging(be, args, info, hp_whole, hp_model, tp_groups_whole, sp_groups_whole, split_tp_sp_cp_groups_whole,
                                allgather_tp_sp_cp_groups_whole, fused_allgather_groups_whole, fused_split_groups_whole,
                                cp_groups_whole)
    finalize_pools(be)
    be.exchange()
    hp_model.sync_tied_embeddings()     # (a collective over the peer buffers: only now are their offsets known)

    gm = GalvatronModel(hp_model)
    gm.dp_groups_whole, gm.tp_groups_whole, gm.sp_groups_whole = dp_groups_whole, tp_groups_whole, sp_groups_whole
    gm.cp_groups_whole, gm.sdp_groups_whole = cp_groups_whole, seq_data_groups_whole
    gm.hybrid_parallel_configs, gm.vtp_data_group = hybrid_parallel_configs, vtp_data_group
    gm.pp_group, gm.embedding_group, gm.hp_configs_whole = pp_group, embedding_group, hp_whole
    gm.sample_layouts = sample_layouts
    return gm


def _reserve_activation_staging(be, args, info, hp_whole, hp_model, tp_groups, sp_groups, split_sep_groups, allgather_sep_groups,
                                fused_ag_groups, fused_sp_groups, cp_groups=None):
    """Size one staging buffer per communicating group from the boundary shapes: the largest activation message is
    seq x microbatch x hidden (bf16), the logits-side reductions are [seq x microbatch] fp32 pairs."""
    world = _world.get_world_size()
    pp = hp_whole["pp_deg"]
    seq = getattr(args, "seq_length", None) or info.shapes()[0][0][0]
    hidden = getattr(args, "hidden_size", None) or info.shapes()[0][0][-1]
    # a layer type whose boundary carries several tensors (T5's decoder: encoder output + decoder states): the relocation between two
    # such rows moves all of them, so size for their summed sequences
    multi = [shapes for shapes in info.shapes() if len(shapes) > 1]
    if multi:
        seq = max(seq, max(sum(next(d for d in s[:-1] if d != -1) for s in shapes) for shapes in multi))
    min_dp = max(1, min(hp_whole["dp_sizes_whole"]))
    max_mbs = -(-args.global_train_batch_size // min_dp // max(1, hp_model.chunks))
    esz = 2 if args.mixed_precision != "fp32" else 4
    # 1.5x: q + k + v of one Ulysses exchange, or the widest column-parallel dgrad, never exceed this for the Llama/GPT/BERT
    # shapes; the logits path adds 2 fp32 per token
    act = int(seq * max_mbs * hidden * esz * 1.5) + seq * max_mbs * 16 + (1 << 16)
    s0, s1 = hp_model.stage_start_idx, hp_model.stage_end_idx
    seen = set()

    def reserve(g):
        if g is not None and g.size > 1 and tuple(g.ranks) not in seen:
            seen.add(tuple(g.ranks))
            be.reserve_staging(g, act)

    for i in range(s0, s1):
        for lst in (tp_groups, sp_groups, split_sep_groups, allgather_sep_groups, fused_ag_groups, fused_sp_groups, cp_groups or ()):
            if lst:
                reserve(lst[i])
    # cp_comm="ring": receive slots of their own per cp group, for the largest local K block (microbatch x s/c x kv heads x head dim)
    # of this stage's context-parallel layers -- 2 x (K + V) bf16 + 2 x (dK + dV) fp32, more than the staging estimate above.  On a
    # layer that also runs Ulysses the block carries the K/V heads left after the exchange (kv_heads_attn: ng/p, or n/p replicated)
    ring_elems = {}
    for m in hp_model.modules():
        if isinstance(m, ParallelAttention) and m.use_cp and m.cp_comm == "ring" and m.cp_group is not None and m.cp_group.size > 1:
            key = tuple(m.cp_group.ranks)
            elems = max_mbs * (seq // m.cp_group.size) * m.kv_heads_attn * m.hn
            ring_elems[key] = (m.cp_group, max(elems, ring_elems.get(key, (None, 0))[1]))
    for group, elems in ring_elems.values():
        be.reserve_cp_ring(group, elems)
    # the whole job as one group (gradient-norm all-reduce of clip_grad_norm, utils.py:124-133): one NVSwitch domain
    if 1 < world <= 8:
        from .comm_groups import CommGroup
        be.world_group = CommGroup(list(range(world)))
        if tuple(be.world_group.ranks) not in seen:
            be.reserve_staging(be.world_group, 4096)
    hp_model.reserve_transport(max_mbs)

"""Pipeline engine: microbatching, the three schedules and the stage-to-stage transport.

Same observable behaviour as ``galvatron/core/runtime/pipeline/pipeline.py`` -- ``no_pipeline_forward_backward`` (:295-373),
``pipedream_flush_forward_backward`` (1F1B-flush, :375-701), ``gpipe_forward`` / ``gpipe_backward`` (:718-883),
``forward_step`` (:895-925: loss / real_chunks), ``backward_step`` (:931-969), ``update_tensor_shape`` (:264-293) and the
microbatch chunking of ``pipeline/utils.py:12-64`` -- with two differences in mechanism:

  * stage-to-stage transport (C11): the sender copies the boundary tensor straight into a receive slot in the
    neighbour's symmetric arena with ``cudaMemcpyPeerAsync``-style peer copies on a side stream and raises a device flag;
    the receiver's stream waits on the flag.  Two slots per direction, acknowledged by the receiver, no host sync
    (reference: ``batch_isend_irecv`` + ``torch.cuda.synchronize()`` per message, :1095-1127,1244; fresh
    ``torch.empty`` receive buffers per call, :1203-1216).
  * gradient reduction: each layer's reduce-scatter starts when that layer's LAST backward of the step completes
    (``DataParallelModule.sync_gradients``), overlapping the rest of the backward; the reference defers every layer's
    reduction until after the schedule (``fsdp_reduce_gradients``, :365-367,693-695).
"""
import copy

import numpy as np
import torch
import torch.nn as nn

from ..arguments import get_args
from ..backend import get_backend
from ..comm_groups import CommGroup
from ..parallel import DataParallelModule, ShardedUnit
from ..tensor_parallel import random as dropout_random
from .utils import chunk_batch, chunk_dict


class PipeSequential(nn.Sequential):
    """``nn.Sequential`` that forwards multiple inputs and kwargs (pipeline.py:1581-1593)."""

    def forward(self, *inputs, **kwargs):
        for module in self:
            if isinstance(inputs, tuple):
                inputs = module(*inputs, **kwargs)
            else:
                inputs = module(inputs, **kwargs)
        return inputs


def forward_step_function(loss_func, **kwargs):
    def forward_step(inputs, model):
        outputs = model(*inputs, **kwargs) if isinstance(inputs, (tuple, list)) else model(inputs, **kwargs)
        return outputs, loss_func

    return forward_step


def _to_list(t):
    if isinstance(t, list):
        return t
    if isinstance(t, tuple):
        return list(t)
    return [t]


class _StageLink:
    """Transport to one neighbouring pipeline stage: 2 receive slots per direction in the symmetric arena."""

    SLOTS = 2

    def __init__(self, be, my_rank, peer_rank, max_bytes, send_flag_base, recv_flag_base):
        # flag ids are per direction (forward messages 0..1, backward messages 2..3) so both ends agree; the flag arrays
        # are indexed by the OTHER rank, so the two links of a stage never collide
        self.be, self.peer, self.max_bytes = be, peer_rank, max_bytes
        self.send_flag_base, self.recv_flag_base = send_flag_base, recv_flag_base
        self.group = CommGroup([my_rank, peer_rank])
        self.slot_bytes = (max_bytes + 255) // 256 * 256
        self.buf = be.sym_alloc(self.group, self.slot_bytes * self.SLOTS)   # my receive slots; peer's are at buf.offs()
        self.me_idx = self.group.ranks.index(my_rank)
        self.peer_idx = 1 - self.me_idx
        self.n_sent = self.n_recv = 0

    def send(self, tensors):
        """Pack the tensors into the peer's next receive slot (side stream; ordered after the producer)."""
        be = self.be
        slot = self.n_sent % self.SLOTS
        self.n_sent += 1
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        peer_off = int(self.buf.offs()[self.peer_idx]) + slot * self.slot_bytes
        with torch.cuda.stream(be.p2p_stream):
            be.p2p_stream.wait_event(ev)
            if len(tensors) > 1:
                # every tensor starts on a 16-byte boundary of the slot, so a mixed-dtype boundary (bf16 activations + an int64
                # mask) unpacks with plain views on the other side
                flat = torch.zeros(self._packed_bytes(tensors), dtype=torch.uint8, device=tensors[0].device)
                off = 0
                for t in tensors:
                    nbytes = t.numel() * t.element_size()
                    flat[off:off + nbytes].copy_(t.contiguous().reshape(-1).view(torch.uint8))
                    off += (nbytes + 15) // 16 * 16
            else:
                flat = tensors[0].contiguous()
            flat.record_stream(be.p2p_stream)
            assert flat.numel() * flat.element_size() <= self.slot_bytes, "pipeline message larger than the reserved slot"
            be.comm.p2p_send(self.peer, peer_off, flat, self.send_flag_base + slot, stream=be.p2p_stream)

    @staticmethod
    def _packed_bytes(tensors):
        return sum((t.numel() * t.element_size() + 15) // 16 * 16 for t in tensors)

    def recv(self, shapes, dtypes, requires_grad):
        """Wait for the peer's next message on the current stream and unpack it into fresh tensors."""
        be = self.be
        slot = self.n_recv % self.SLOTS
        self.n_recv += 1
        be.comm.p2p_wait(self.peer, self.recv_flag_base + slot)
        raw = self.buf.u8[slot * self.slot_bytes:(slot + 1) * self.slot_bytes]
        outs, off = [], 0
        for shape, dtype in zip(shapes, dtypes):
            numel = int(np.prod(shape))
            nbytes = numel * torch.empty((), dtype=dtype).element_size()
            t = raw[off:off + nbytes].view(dtype).view(*shape).clone()
            if requires_grad and t.is_floating_point():
                t.requires_grad_(True)
            outs.append(t)
            off += nbytes if len(shapes) == 1 else (nbytes + 15) // 16 * 16
        be.comm.p2p_release(self.peer, self.recv_flag_base + slot)
        return outs


class PipelineParallel(nn.Module):
    def __init__(self, model, model_ranks, layer_output_tensor_shapes, layer_output_tensor_dtypes=None, layer_dp_sizes=None,
                 layer_tp_sizes=None, layer_sp_sizes=None, layer_cp_sizes=None, chunks=1, process_group=None,
                 embedding_group=None, nproc_per_node=None, require_loss=True, info=False, tied_wte_attr_names=None):
        super().__init__()
        from .. import world as _world
        n = len(model)
        self.total_model_len = n
        assert n == len(model_ranks) == len(layer_output_tensor_shapes)
        if layer_output_tensor_dtypes is None:
            layer_output_tensor_dtypes = [None if s is None else [torch.float] * len(s) for s in layer_output_tensor_shapes]
        ones = [1] * n
        layer_dp_sizes, layer_tp_sizes = layer_dp_sizes or ones, layer_tp_sizes or ones
        layer_sp_sizes, layer_cp_sizes = layer_sp_sizes or ones, layer_cp_sizes or ones
        self.world_size, self.global_rank = _world.get_world_size(), _world.get_rank()
        self.pp_global_ranks = list(range(self.world_size)) if process_group is None else sorted(set(process_group))
        assert self.global_rank in self.pp_global_ranks
        self.group_size = len(self.pp_global_ranks)
        self.group_rank = self.pp_global_ranks.index(self.global_rank)
        assert len(set(model_ranks)) == self.group_size and max(model_ranks) == self.group_size - 1 and min(model_ranks) == 0
        self.stage_start_idx = model_ranks.index(self.group_rank)
        self.stage_end_idx = self.stage_start_idx + model_ranks.count(self.group_rank)
        self.model_cur_stage = PipeSequential(*list(model)[self.stage_start_idx:self.stage_end_idx])
        self.chunks = int(chunks)
        assert self.chunks >= 1
        first, last = self.is_pipeline_first_stage(), self.is_pipeline_last_stage()
        s0, s1 = self.stage_start_idx, self.stage_end_idx
        self.template_stage_input_tensor_shape = [None] if first else layer_output_tensor_shapes[s0 - 1]
        self.template_stage_output_tensor_shape = [None] if last else layer_output_tensor_shapes[s1 - 1]
        self.stage_input_tensor_dtype = [None] if first else layer_output_tensor_dtypes[s0 - 1]
        self.stage_output_tensor_dtype = [None] if last else layer_output_tensor_dtypes[s1 - 1]
        pick = lambda lst, i: None if i is None else lst[i]  # noqa: E731
        pi, ci = (None if first else s0 - 1), (None if last else s1 - 1)
        self.dp_size_prev_stage, self.dp_size_cur_stage = pick(layer_dp_sizes, pi), pick(layer_dp_sizes, ci)
        self.tp_size_prev_stage, self.tp_size_cur_stage = pick(layer_tp_sizes, pi), pick(layer_tp_sizes, ci)
        self.sp_size_prev_stage, self.sp_size_cur_stage = pick(layer_sp_sizes, pi), pick(layer_sp_sizes, ci)
        self.cp_size_prev_stage, self.cp_size_cur_stage = pick(layer_cp_sizes, pi), pick(layer_cp_sizes, ci)
        self.dp_size_input = layer_dp_sizes[0]
        self.info, self.chunk_warning, self.require_loss = info, True, require_loss
        args = get_args()
        self.sequence_parallel, self.shape_order = args.sequence_parallel, args.shape_order
        self.async_grad_reduce = args.async_grad_reduce
        self.embedding_group, self.tied_wte_attr_names = embedding_group, tied_wte_attr_names
        self._tied_units = []           # filled by _setup_tied_embeddings once the stage's units exist
        self._tied_grad = None          # the tied gradient range registered over the embedding group (peer-memory backend, pp > 1)
        self.units = []
        self._links = {}
        self.real_chunks = self.chunks
        self._gpipe_state = None

    # ---- topology helpers ---------------------------------------------------------------------------------------------
    def is_pipeline_first_stage(self):
        return self.group_rank == 0

    def is_pipeline_last_stage(self):
        return self.group_rank == self.group_size - 1

    # ---- construction steps 5 / 6 ----------------------------------------------------------------------------------
    def wrap_pipeline_modules_data_parallel(self, dp_types, dp_groups, module_types, mixed_precision=torch.bfloat16,
                                            wrap_block_name=None, wrap_other_block_name=None, tp_groups=None,
                                            all_block_name=None, load_module_func=None, checkpoint_flags=None):
        """One ShardedUnit per whole-model row of this stage (pipeline.py:177-242 -> parallel.py:316-386).
        dp type: 1 -> zero3, 0 -> ``args.default_dp_type`` (parallel.py:61)."""
        args = get_args()
        assert self.total_model_len == len(dp_types) == len(dp_groups) == len(module_types)
        s0, s1 = self.stage_start_idx, self.stage_end_idx
        wrapped = []
        # zero3 gradients can share a pool only when every backward is followed by its reduction
        pool_grads = self.chunks == 1 or not args.async_grad_reduce
        for i, module in zip(range(s0, s1), self.model_cur_stage):
            dp_type = {0: args.default_dp_type, 1: "zero3"}[dp_types[i]]
            tp_group = None if tp_groups is None else tp_groups[i]
            unit = ShardedUnit(module, dp_groups[i], dp_type, name="%s_%d" % (module_types[i], i), tp_group=tp_group,
                               param_dtype=mixed_precision, reduce_in_fp32=args.reduce_in_fp32,
                               sequence_parallel=self.sequence_parallel, init_seed=args.seed + 1000 * i,
                               pool_slots=int(getattr(args, "zero3_pool_slots", 0)), pool_grads=pool_grads,
                               load_module_func=load_module_func, all_block_name=all_block_name, load=getattr(args, "load", None),
                               distributed_checkpoint=bool(getattr(args, "distributed_checkpoint", False)),
                               reserve_save_buffer=bool(getattr(args, "save", None)) or self.tied_wte_attr_names is not None)
            self.units.append(unit)
            wrapped.append(DataParallelModule(module, unit, checkpoint=False))
        for a, b in zip(wrapped[:-1], wrapped[1:]):
            a.next_unit, b.prev_unit = b.unit, a.unit
        self.model_cur_stage = PipeSequential(*wrapped)
        if self.tied_wte_attr_names is not None:
            self._setup_tied_embeddings()

    # ---- tied word embeddings (C14) ------------------------------------------------------------------------------------------------
    @staticmethod
    def _tied_param(unit, attr):
        """The word-embedding matrix inside a unit: the 2-D parameter under attribute ``attr`` of the wrapped block ("" = the block
        itself: the output head), as ``tied_wte_attr_names`` names it (hybrid_parallel_model.py:176, GPTModel_hybrid_parallel.py:42)."""
        cands = [(n, p) for n, p in unit.module.named_parameters() if p.dim() == 2 and (not attr or attr in n.split("."))]
        if not cands:
            raise ValueError("tied_wte_attr_names: no 2-D parameter under %r in unit %s" % (attr, unit.name))
        return max(cands, key=lambda np_: np_[1].numel())

    def _setup_tied_embeddings(self):
        """``sync_embedding`` (pipeline.py:228-242): the input embedding (first unit of the first stage) and the output head (last unit
        of the last stage) hold two copies of ONE matrix.  At construction both become the average of the two initialisations
        (``sync_tied_embeddings``); after every backward their unsharded gradients are summed into both (``finalize_wte_grads_func``
        :1031-1050 -- the reference's pp > 1 rule, applied here for pp = 1 too, where the reference averages sequentially and lets the
        copies drift apart), so identical optimizer steps keep them identical.  This step finds the tied units and parameters; across
        pipeline stages on a peer-memory backend it also registers the parameter's gradient range over the embedding group, which the
        in-place sum of the two copies then works on (before the backend's ``exchange()``, like every symmetric buffer)."""
        be = get_backend()
        first, last = self.is_pipeline_first_stage(), self.is_pipeline_last_stage()
        embed = self.units[0] if first else None
        head = self.units[-1] if last else None
        mine = [(u, attr) for u, attr in ((embed, self.tied_wte_attr_names[0]), (head, self.tied_wte_attr_names[-1])) if u is not None]
        if not mine:
            return
        if self.group_size > 1 and not getattr(be, "supports_tied_embedding_exchange", False):
            raise NotImplementedError("tied embeddings across pipeline stages need an all-reduce over the embedding group (first + last "
                                      "stage): not wired into this backend; run with untie_embeddings_and_output_weights=True or pp_deg=1")
        for u, attr in mine:
            if u.g_pool is not None:
                raise ValueError("tied embeddings cannot use pooled zero3 gradient buffers (set --embed_sdp 0 or --zero3_pool_slots 0)")
            name, p = self._tied_param(u, attr)
            u._tie = {"param": p, "name": name, "deferred": False}
            self._tied_units.append(u)
        register = getattr(be, "register_tied_grad", None)
        if self.group_size > 1 and register is not None:
            u = self._tied_units[0]
            self._tied_grad = register(u, u._tie["param"], self.embedding_group)

    def sync_tied_embeddings(self):
        """Construction, after the backend's ``exchange()``: both copies of the tied matrix become the fp32 average of the two
        initialisations -- what the reference's all-reduce(AVG) over the embedding group does."""
        if not self._tied_units:
            return
        be = get_backend()
        fulls = []
        for u in self._tied_units:
            full = be.gather_master(u).clone()
            fulls.append((u, full, u.named_slices(full)[u._tie["name"]]))
        if self.group_size == 1:
            (_, _, a), (_, _, b) = fulls
            if a.shape != b.shape:
                raise ValueError("tied embeddings need the same vocabulary sharding on both rows: %s vs %s" % (tuple(a.shape), tuple(b.shape)))
            avg = (a + b) / 2
            a.copy_(avg)
            b.copy_(avg)
        elif self._tied_grad is not None:
            (_, _, a), = fulls
            be.tied_average(self._tied_grad, a)
        else:
            (_, _, a), = fulls
            a.copy_(be.all_reduce(a.contiguous(), self.embedding_group) / 2)
        for u, full, _ in fulls:
            u.write_master(full)

    def _finalize_tied(self):
        """``finalize_wte_grads_func``: both copies of the tied matrix receive the SUM of their unsharded gradients; then the deferred
        reductions of the tied units are launched."""
        if not self._tied_units:
            return
        be = get_backend()
        for u in self._tied_units:
            p = u._tie["param"]
            if u._tie["deferred"] and not u.grad_started(p):
                p._bg_grad.zero_()
                u.mark_grad(p)
        live = [u for u in self._tied_units if u._tie["deferred"]]
        if live:
            if self.group_size == 1:
                a, b = (u._tie["param"]._bg_grad for u in self._tied_units)
                a.add_(b)
                b.copy_(a)
            elif self._tied_grad is not None:
                be.tied_grad_sum(self._tied_units[0], self._tied_grad)
            else:
                g = self._tied_units[0]._tie["param"]._bg_grad
                g.copy_(be.all_reduce(g.contiguous(), self.embedding_group))
        for u in live:
            u.reduce_now()
            u._tie["deferred"] = False

    def gen_sp_layernorm_info(self, *a, **k):
        """The reference attaches LayerNorm offsets to each FSDP state here (pipeline.py:244-256); the ShardedUnit finds its
        ``sequence_parallel``-tagged parameters itself."""
        return None

    def wrap_pipeline_modules_checkpoint(self, checkpoint_flags, wrap_block_name=None):
        self.checkpoint_flags_stage = checkpoint_flags[self.stage_start_idx:self.stage_end_idx]
        for m, flag in zip(self.model_cur_stage, self.checkpoint_flags_stage):
            m.checkpoint = bool(flag)

    def reserve_transport(self, max_microbatch_size):
        """Allocate the receive slots towards the neighbouring stages (must precede ``backend.exchange()``)."""
        if self.group_size == 1:
            return
        be = get_backend()

        def nbytes(shapes, dtypes, dp_size, tp, sp, cp):
            if shapes is None or shapes[0] is None:
                return 0
            total = 0
            for shape, dt in zip(shapes, dtypes):
                shape = [max_microbatch_size if d == -1 else d for d in shape]
                nb = int(np.prod(shape)) * torch.empty((), dtype=dt).element_size()
                # a message of several tensors starts each one on a 16-byte boundary (_StageLink.send)
                total += nb if len(shapes) == 1 else (nb + 15) // 16 * 16
            return total

        if not self.is_pipeline_first_stage():
            prev = self.pp_global_ranks[self.group_rank - 1]
            nb = nbytes(self.template_stage_input_tensor_shape, self.stage_input_tensor_dtype, 1, 1, 1, 1)
            self._links["prev"] = be.make_stage_link(self.global_rank, prev, nb, send_flag_base=2, recv_flag_base=0)
        if not self.is_pipeline_last_stage():
            nxt = self.pp_global_ranks[self.group_rank + 1]
            nb = nbytes(self.template_stage_output_tensor_shape, self.stage_output_tensor_dtype, 1, 1, 1, 1)
            self._links["next"] = be.make_stage_link(self.global_rank, nxt, nb, send_flag_base=0, recv_flag_base=2)

    # ---- per-step bookkeeping -----------------------------------------------------------------------------------------
    def begin_step(self):
        get_backend().begin_step()
        for u in self.units:
            u.begin_step()

    def finish_step(self):
        self._finalize_tied()
        if self.units:
            self.units[0].finish_step()

    def set_last_batch(self, state):
        """pipeline.py:258-262: marks the microbatch whose backward triggers gradient synchronisation."""
        sync = bool(state) or not self.async_grad_reduce
        for m in self.model_cur_stage:
            if isinstance(m, DataParallelModule):
                m.sync_gradients = sync

    def _flush_backward(self):
        for m in self.model_cur_stage:
            if isinstance(m, DataParallelModule):
                m.flush_backward()

    def _chunk(self, batch, kwargs):
        micro_kwargs = chunk_dict(kwargs, self.chunks)
        microbatches = [chunk_batch(batch[0], self.chunks), chunk_batch(batch[1], self.chunks)]
        self.real_chunks = len(microbatches[0])
        if self.chunks != self.real_chunks and self.chunk_warning and self.global_rank == 0:
            print("\nWarning from PipelineParallel Module: Real chunks is %d !" % self.real_chunks,
                  "Microbatch sizes is", [m[0].shape[0] for m in microbatches[0]])
            self.chunk_warning = False
        while len(micro_kwargs) < self.real_chunks:
            micro_kwargs.append(micro_kwargs[-1] if micro_kwargs else {})
        # (first sample, size) of every microbatch inside the local batch: the dropout context of its forward
        sizes = [next((t.shape[0] for t in mb if torch.is_tensor(t)), 0) for mb in microbatches[0]]
        self._mb_span = [(sum(sizes[:i]), sizes[i]) for i in range(len(sizes))]
        return microbatches, micro_kwargs

    def _begin_microbatch(self, i):
        dropout_random.set_microbatch(*self._mb_span[i])

    def update_tensor_shape(self, microbatches, dp_size_input, dp_size, tp_size, sp_size, template_tensor_shape, cp_size=None):
        """Concrete boundary shapes for the regular and the last microbatch (pipeline.py:264-293)."""
        cp_size = cp_size or 1
        out = []
        for mb in (microbatches[0][0], microbatches[0][-1]):
            shape = copy.deepcopy(template_tensor_shape)
            mbs = mb[0].shape[0] * dp_size_input // dp_size
            # context parallelism always splits the sequence; tp|sp only under --sequence-parallel (the reference divides by
            # neither without the flag, :277-281, which leaves cp x pp without sequence parallelism broken there)
            size = (sp_size if tp_size == 1 else tp_size) * cp_size if self.sequence_parallel else cp_size
            for i in range(len(shape)):
                shape[i] = [mbs if d == -1 else d for d in shape[i]]
                if size > 1:
                    if self.shape_order == "SBH":
                        shape[i][0] = shape[i][0] // size
                    else:
                        shape[i] = [shape[i][0] * shape[i][1] // size, shape[i][2]]
            out.append(shape)
        return out[0], out[1]

    # ---- forward / backward of one microbatch (pipeline.py:895-969) -------------------------------------------------------
    def forward_step(self, forward_step_func, batch, model, input_tensor, losses_reduced):
        input_tensor = _to_list(input_tensor)
        for x in input_tensor:
            if x is not None and x.is_floating_point():
                x.requires_grad = True
        if input_tensor[0] is None:
            output_tensor, loss_func = forward_step_func(batch[0], model)
        else:
            output_tensor, loss_func = forward_step_func(input_tensor, model)
        output_tensor = _to_list(output_tensor)
        if self.is_pipeline_last_stage():
            if self.require_loss:
                loss, loss_reduced = loss_func(batch[1], output_tensor)
                losses_reduced.append(loss_reduced)
                return loss / self.real_chunks
            return output_tensor
        return output_tensor

    def backward_step(self, input_tensor, output_tensor, output_tensor_grad):
        unwrap = not isinstance(input_tensor, list)
        inputs = [input_tensor] if unwrap else input_tensor
        inputs = [None if t is None or not t.requires_grad else t for t in inputs]
        for x in inputs:
            if x is not None:
                x.retain_grad()
        outs = output_tensor if isinstance(output_tensor, list) else [output_tensor]
        grads = output_tensor_grad if isinstance(output_tensor_grad, list) else [output_tensor_grad]
        if len(grads) < len(outs):
            grads = grads + [None] * (len(outs) - len(grads))
        pairs = [(t, g) for t, g in zip(outs, grads) if t is not None and t.requires_grad]
        for m in self.model_cur_stage:
            if isinstance(m, DataParallelModule):
                m.arm_backward()
        torch.autograd.backward([t for t, _ in pairs], grad_tensors=[g for _, g in pairs])
        self._flush_backward()
        in_grads = [None if x is None else x.grad for x in inputs]
        return in_grads[0] if unwrap else in_grads

    # ---- schedule: no pipeline (pp_deg == 1), gradient accumulation over microbatches ---------------------------------------
    def no_pipeline_forward_backward(self, batch, loss_func, forward_only=False, profiler=None, iter=0, **kwargs):
        model = self.model_cur_stage
        microbatches, micro_kwargs = self._chunk(batch, kwargs)
        n_mb = self.real_chunks
        losses_reduced = []
        self.begin_step()
        self.set_last_batch(False)
        for i in range(n_mb):
            if i == n_mb - 1:
                self.set_last_batch(True)
            cur = [microbatches[0][i], microbatches[1][i]]
            self._begin_microbatch(i)
            out = self.forward_step(forward_step_function(loss_func, **micro_kwargs[i]), cur, model, None, losses_reduced)
            if profiler is not None and i == n_mb - 1:
                profiler.profile_memory(iter, "After Forward")
            if forward_only:
                continue
            self.backward_step(None, out, None)
        if not forward_only:
            self.finish_step()
        return losses_reduced

    # ---- transport wrappers ------------------------------------------------------------------------------------------------------
    def _send(self, where, tensors):
        tensors = [t for t in _to_list(tensors) if t is not None]
        if tensors:
            self._links[where].send([t.detach() for t in tensors])

    def _recv(self, where, shapes, dtypes, requires_grad):
        if shapes is None or shapes[0] is None:
            return [None]
        return self._links[where].recv(shapes, dtypes, requires_grad)

    # ---- schedule: 1F1B with flush (pipedream_flush) -----------------------------------------------------------------------------
    def pipedream_flush_forward_backward(self, batch, loss_func, forward_only=False, **kwargs):
        assert self.group_size > 1
        model = self.model_cur_stage
        microbatches, micro_kwargs = self._chunk(batch, kwargs)
        n_mb = self.real_chunks
        n_warm = min(self.group_size - self.group_rank - 1, n_mb)     # pipeline.py:408-410
        n_rest = n_mb - n_warm
        first, last = self.is_pipeline_first_stage(), self.is_pipeline_last_stage()
        in_shape = in_shape_last = out_shape = out_shape_last = [None]
        if not first:
            in_shape, in_shape_last = self.update_tensor_shape(microbatches, self.dp_size_input, self.dp_size_prev_stage,
                                                               self.tp_size_prev_stage, self.sp_size_prev_stage,
                                                               self.template_stage_input_tensor_shape, self.cp_size_prev_stage)
        if not last:
            out_shape, out_shape_last = self.update_tensor_shape(microbatches, self.dp_size_input, self.dp_size_cur_stage,
                                                                 self.tp_size_cur_stage, self.sp_size_cur_stage,
                                                                 self.template_stage_output_tensor_shape, self.cp_size_cur_stage)
        in_dt, out_dt = self.stage_input_tensor_dtype, self.stage_output_tensor_dtype
        shp = lambda k, regular, final: final if k == n_mb - 1 else regular  # noqa: E731
        input_tensors, output_tensors, losses_reduced = [], [], []
        fwd_num = bwd_num = 0
        self.begin_step()
        self.set_last_batch(False)

        def run_forward(i):
            nonlocal fwd_num
            inp = [None] if first else self._recv("prev", shp(fwd_num, in_shape, in_shape_last), in_dt, True)
            cur = [microbatches[0][i], microbatches[1][i]]
            self._begin_microbatch(i)
            out = self.forward_step(forward_step_function(loss_func, **micro_kwargs[i]), cur, model, inp, losses_reduced)
            fwd_num += 1
            if not last:
                self._send("next", out)
            return inp, out

        def run_backward(inp, out):
            nonlocal bwd_num
            if bwd_num == n_mb - 1:
                self.set_last_batch(True)
            grad = [None] if last else self._recv("next", shp(bwd_num, out_shape, out_shape_last), out_dt, False)
            in_grad = self.backward_step(inp, out, grad)
            bwd_num += 1
            if not first:
                self._send("prev", in_grad)

        for i in range(n_warm):                       # warm-up forwards
            inp, out = run_forward(i)
            if not forward_only:
                input_tensors.append(inp)
                output_tensors.append(out)
        for i in range(n_rest):                       # steady state: one forward, one backward
            inp, out = run_forward(i + n_warm)
            if forward_only:
                continue
            input_tensors.append(inp)
            output_tensors.append(out)
            run_backward(input_tensors.pop(0), output_tensors.pop(0))
        if not forward_only:
            for _ in range(n_warm):                   # cool-down backwards
                run_backward(input_tensors.pop(0), output_tensors.pop(0))
            self.finish_step()
        return losses_reduced

    # ---- schedule: GPipe (all forwards, then all backwards) ------------------------------------------------------------------------
    def gpipe_forward(self, batch, loss_func, forward_only=False, **kwargs):
        model = self.model_cur_stage
        microbatches, micro_kwargs = self._chunk(batch, kwargs)
        n_mb = self.real_chunks
        first, last = self.is_pipeline_first_stage(), self.is_pipeline_last_stage()
        in_shape = in_shape_last = out_shape = out_shape_last = [None]
        if not first:
            in_shape, in_shape_last = self.update_tensor_shape(microbatches, self.dp_size_input, self.dp_size_prev_stage,
                                                               self.tp_size_prev_stage, self.sp_size_prev_stage,
                                                               self.template_stage_input_tensor_shape, self.cp_size_prev_stage)
        if not last:
            out_shape, out_shape_last = self.update_tensor_shape(microbatches, self.dp_size_input, self.dp_size_cur_stage,
                                                                 self.tp_size_cur_stage, self.sp_size_cur_stage,
                                                                 self.template_stage_output_tensor_shape, self.cp_size_cur_stage)
        losses_reduced, inputs, outputs = [], [], []
        self.begin_step()
        self.set_last_batch(False)
        for i in range(n_mb):
            shape = in_shape_last if i == n_mb - 1 else in_shape
            inp = [None] if first else self._recv("prev", shape, self.stage_input_tensor_dtype, True)
            cur = [microbatches[0][i], microbatches[1][i]]
            self._begin_microbatch(i)
            out = self.forward_step(forward_step_function(loss_func, **micro_kwargs[i]), cur, model, inp, losses_reduced)
            if not last:
                self._send("next", out)
            inputs.append(inp)
            outputs.append(out)
        self._gpipe_state = (inputs, outputs, out_shape, out_shape_last, n_mb)
        return losses_reduced

    def gpipe_backward(self):
        inputs, outputs, out_shape, out_shape_last, n_mb = self._gpipe_state
        first, last = self.is_pipeline_first_stage(), self.is_pipeline_last_stage()
        for i in range(n_mb):                         # the reference also walks microbatches front to back (:825-883)
            if i == n_mb - 1:
                self.set_last_batch(True)
            shape = out_shape_last if i == n_mb - 1 else out_shape
            grad = [None] if last else self._recv("next", shape, self.stage_output_tensor_dtype, False)
            in_grad = self.backward_step(inputs[i], outputs[i], grad)
            if not first:
                self._send("prev", in_grad)
        self._gpipe_state = None
        self.finish_step()

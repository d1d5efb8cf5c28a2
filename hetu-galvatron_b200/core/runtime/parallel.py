"""Per-layer data-parallel wrapping: the sharded unit that owns a layer's flat parameter / gradient buffers and issues
the SDP collectives, activation checkpointing, and the relocation wrapper.

Replaces ``galvatron/core/runtime/parallel.py`` (``wrap_module_fsdp_manually`` :92-199, ``wrap_modules_data_parallel``
:316-386, ``wrap_modules_checkpoint`` :229-240, ``Module_with_relocation`` :279-313) and the FSDP1 machinery it drives
(``torch/distributed/fsdp/_flat_param.py`` FlatParamHandle, ``_runtime_utils.py`` _unshard / _reduce_grad, plus the three
monkey-patches in ``pipeline/grad_reduce.py`` and ``pipeline/sp_grad_reduce.py``) with one explicit state machine per
layer whose observable semantics are the reference's:

  dp type     master (fp32)        forward params (bf16)            gradient reduction
  ddp         full                 local cast                       all-reduce          (NO_SHARD)
  zero2       1/d shard            all-gather+cast once per step    reduce-scatter      (SHARD_GRAD_OP)
  zero3       1/d shard            all-gather+cast fwd and bwd*     reduce-scatter      (FULL_SHARD)
  (* zero3 layers gather into a small rotating pool of peer-visible buffers (``SlotPool``), released after every forward
     and backward exactly where FSDP reshards; a released copy stays valid until its slot is reclaimed, so the second gather
     is skipped when the pool is large enough -- comm volume <= the reference's, memory = pool size, not model size.)

  * gradients accumulate UNSHARDED in bf16 across microbatches and are reduced once per step, on the last microbatch
    (default ``async_grad_reduce``; grad_reduce.py:47-64,177-198) -- but each layer's reduce-scatter is launched as soon
    as that layer's last backward finishes, on a side stream, instead of after the whole backward;
  * with ``--no_async_grad_reduce`` every microbatch is reduced and summed into the fp32 shard (_runtime_utils.py:917-926);
  * pre-divide / post-divide factors and padding follow FSDP (default_hooks.py:38-42, _runtime_utils.py:852,879,896-901),
    fused into the reduce-scatter kernel together with the bf16->fp32 cast and the ``+=``;
  * under Megatron-SP, gradients of ``sequence_parallel``-tagged params (norm weights, row-parallel bias) are summed over
    the TP group on the last microbatch (sp_grad_reduce.py:104-123).
"""
import torch
import torch.nn as nn

from .backend import get_backend
from .redistribute import fused_split_allgather
from .tensor_parallel import random as dropout_random

_DP_TYPES = ("ddp", "zero2", "zero3")


def fsdp_divide_factors(world_size):
    """(predivide, postdivide) of FSDP's DefaultState (default_hooks.py:38-42): d=2->(2,1), 4->(2,2), 8->(4,2)."""
    factor = 1
    while world_size % factor == 0 and world_size / factor > factor:
        factor *= 2
    return float(factor), world_size / float(factor)


class _Slot:
    __slots__ = ("buf", "owner", "version", "free_event", "index")

    def __init__(self, buf, index):
        self.buf, self.index, self.owner, self.version, self.free_event = buf, index, None, None, None


class SlotPool:
    """Rotating peer-visible buffers shared by the zero3 units of one (group, dtype, role): what FSDP's alloc/free of the
    padded unsharded flat parameter (``_flat_param.py`` _alloc_padded_unsharded_flat_param / _free_unsharded_flat_param)
    becomes when the memory must stay peer-mapped.  Every member of the group walks the same program, so the same slot
    index is chosen everywhere and the peers' pushes land in the matching slot.  Ordering between successive occupants is
    by CUDA events on the owner's streams plus the collective's own entry barrier across ranks."""

    def __init__(self, be, group, dtype, n_slots, role):
        self.be, self.group, self.dtype, self.n_slots, self.role = be, group, dtype, int(n_slots), role
        self.max_elems = 0
        self.slots = None
        self.free = []          # release order: oldest first
        self.held = {}          # id(unit) -> slot
        self.n_gather_skipped = 0

    def register(self, unit):
        assert self.slots is None, "zero3 pool already allocated"
        self.max_elems = max(self.max_elems, unit.padded)

    def finalize(self):
        if self.slots is None:
            esz = torch.empty((), dtype=self.dtype).element_size()
            self.slots = [_Slot(self.be.sym_alloc(self.group, self.max_elems * esz), i) for i in range(self.n_slots)]
            self.free = list(self.slots)

    def nbytes(self):
        return self.n_slots * self.max_elems * torch.empty((), dtype=self.dtype).element_size()

    def acquire(self, unit, version=None, demand=True):
        """-> (slot, cached).  ``cached``: the slot still holds this unit's data of this ``version`` (no gather needed).
        Without a free slot a demand acquire evicts a prefetched, not-yet-used occupant; a prefetch just gives up (None)."""
        self.finalize()
        if version is not None:
            for i, s in enumerate(self.free):
                if s.owner is unit and s.version == version:
                    del self.free[i]
                    self.held[id(unit)] = s
                    self.n_gather_skipped += 1
                    return s, True
        if not self.free:
            if not demand:
                return None, False
            victim = next((s.owner for s in self.held.values() if s.owner._in_use == 0 and s.owner is not unit), None)
            if victim is None:
                raise RuntimeError("zero3 %s pool of %d slots exhausted by layers in use: raise --zero3_pool_slots" % (self.role, self.n_slots))
            victim.evict(self.role)
        s = self.free.pop(0)
        s.owner, s.version = unit, version
        self.held[id(unit)] = s
        return s, False

    def release(self, unit, event):
        s = self.held.pop(id(unit))
        s.free_event = event
        self.free.append(s)


def get_pool(be, group, dtype, n_slots, role):
    pools = be.__dict__.setdefault("_zero3_pools", {})
    key = (tuple(group.ranks), dtype, role)
    if key not in pools:
        pools[key] = SlotPool(be, group, dtype, n_slots, role)
    return pools[key]


def finalize_pools(be):
    """Allocate every registered pool (before ``backend.exchange()``)."""
    for pool in be.__dict__.get("_zero3_pools", {}).values():
        pool.finalize()


class ShardedUnit:
    """One layer's flat parameter, sharded over ``group`` (what an FSDP unit is in the reference)."""

    def __init__(self, module, group, dp_type, name="", tp_group=None, param_dtype=torch.bfloat16, reduce_in_fp32=False,
                 sequence_parallel=False, init_seed=None, pool_slots=0, pool_grads=False, load_module_func=None,
                 all_block_name=None, load=None, distributed_checkpoint=False, reserve_save_buffer=False):
        assert dp_type in _DP_TYPES, dp_type
        be = get_backend()
        self.be, self.module, self.group, self.dp_type, self.name = be, module, group, dp_type, name
        self.tp_group, self.sequence_parallel = tp_group, sequence_parallel
        self.param_dtype = param_dtype
        self.reduce_dtype = torch.float32 if reduce_in_fp32 else param_dtype
        self.rank_in_group = group.rank_in_group(be.rank) if group.size > 1 else 0
        d = group.size
        device = be.device

        # ---- materialise (meta -> device) and collect parameters ---------------------------------------------
        self._materialize(module, device, init_seed)
        if load is not None and load_module_func is not None:
            self._load(module, load_module_func, all_block_name, load, distributed_checkpoint)
        seen, params = set(), []
        for p in module.parameters():
            if id(p) not in seen:
                seen.add(id(p))
                params.append(p)
        self.params = params
        self.numels = [p.numel() for p in params]
        self.offsets = [0]
        for n in self.numels:
            # keep every parameter 16-byte aligned inside the flat buffers (vector loads, TMA bases)
            self.offsets.append(self.offsets[-1] + (n + 7) // 8 * 8)
        total = self.offsets[-1]
        self.total = total
        self.padded = (total + 8 * d - 1) // (8 * d) * (8 * d)
        self.shard_elems = self.padded // d

        # ---- fp32 master (what the optimizer sees) ---------------------------------------------------------------
        full = torch.zeros(self.padded, dtype=torch.float32, device=device)
        for p, off, n in zip(params, self.offsets, self.numels):
            full[off:off + n].copy_(p.detach().reshape(-1).float())
        if dp_type == "ddp":
            master = full
        else:
            master = full[self.rank_in_group * self.shard_elems:(self.rank_in_group + 1) * self.shard_elems].clone()
        self.flat_param = nn.Parameter(master, requires_grad=True)
        self.flat_param._bg_unit = self
        # fp32 gradient shard: allocated on first use (never with the fused optimizer, except for pooled zero3 units under clipping)
        self._master_grad = None
        self.fused_opt = None          # set by FusedShardedAdamW: the reduction's epilogue applies the update

        # ---- peer-visible flat buffers: W (gathered params) and G (unsharded grads) --------------------------------
        # zero3 layers take theirs from a rotating pool (``pool_slots`` > 0): memory is the pool's, not the model's.
        esz = torch.empty((), dtype=param_dtype).element_size()
        gsz = torch.empty((), dtype=self.reduce_dtype).element_size()
        self.shapes = [p.shape for p in params]
        pooled = dp_type == "zero3" and d > 1 and pool_slots > 0
        self.w_pool = get_pool(be, group, param_dtype, pool_slots, "param") if pooled else None
        self.g_pool = get_pool(be, group, self.reduce_dtype, max(2, pool_slots - 1), "grad") if pooled and pool_grads else None
        self.W = self.G = self.w_flat = self.g_flat = None
        self._w_version, self._in_use, self._w_wait_event = 0, 0, None
        for p in params:
            p._bg_unit = self
        if self.w_pool is None:
            self._bind_w(be.sym_alloc(group, self.padded * esz))
            self.w_flat.copy_(full.to(param_dtype))  # valid until the first optimizer step
        else:
            self.w_pool.register(self)
            placeholder = torch.empty(0, dtype=param_dtype, device=device)
            for p in params:
                p.data = placeholder       # FSDP's freed unsharded flat parameter
        if self.g_pool is None:
            self._bind_g(be.sym_alloc(group, self.padded * gsz))
            self.g_flat.zero_()
        else:
            self.g_pool.register(self)
        del full
        self._ln_params = [p for p in params if getattr(p, "sequence_parallel", False)] if (
            sequence_parallel and tp_group is not None and tp_group.size > 1) else []

        if reserve_save_buffer:
            be.reserve_checkpoint_gather(group, self.padded * 4)
        self.prediv, self.postdiv = fsdp_divide_factors(d)
        self._started = set()          # params whose G slice holds this step's gradient
        self._w_valid = self.w_pool is None
        self._unshard_event = None
        self._reduce_event = None      # the last reduction of this unit (reduce stream) has read G
        self._reduced_this_step = False
        self._pending = False          # backward ran since the last reduction
        self.n_unshard = self.n_reduce = 0
        # tied word embeddings (C14, pipeline/grad_reduce.py:98-131): {"param": the tied weight, "deferred": bool}.  Such a unit does not
        # reduce at its own post-backward: PipelineParallel.finish_step first exchanges the unsharded gradient with the partner unit
        # (the other copy of the matrix), then launches the reduction.
        self._tie = None

    @property
    def master_grad(self):
        if self._master_grad is None:
            self._master_grad = torch.zeros_like(self.flat_param.data)
        return self._master_grad

    def uses_fused_optimizer(self):
        # the fused epilogue covers the sharded (and single-rank) reduction paths; replicated DDP layers keep the plain path
        return self.fused_opt is not None and (self.dp_type != "ddp" or self.group.size == 1)

    # ---- construction helpers -------------------------------------------------------------------------------------
    @staticmethod
    def _materialize(module, device, seed):
        """meta-device init as the reference's ``param_init_fn`` (parallel.py:79-89): to_empty + reset_parameters."""
        has_meta = any(p.device.type == "meta" for p in module.parameters())
        if has_meta:
            module.to_empty(device=device)
            gen_state = None
            if seed is not None:
                gen_state = torch.get_rng_state() if device.type == "cpu" else torch.cuda.get_rng_state(device)
                torch.manual_seed(seed)
            for sub in module.modules():
                if callable(getattr(sub, "reset_parameters", None)) and any(True for _ in sub.parameters(recurse=False)):
                    sub.reset_parameters()
            if gen_state is not None:
                torch.set_rng_state(gen_state) if device.type == "cpu" else torch.cuda.set_rng_state(gen_state, device)
        else:
            module.to(device)

    def _bind_w(self, buf):
        self.W = buf
        self.w_flat = buf.view(self.param_dtype, self.padded)
        for p, off, n, shape in zip(self.params, self.offsets, self.numels, self.shapes):
            p.data = self.w_flat[off:off + n].view(shape)

    def _bind_g(self, buf):
        self.G = buf
        self.g_flat = buf.view(self.reduce_dtype, self.padded)
        for p, off, n, shape in zip(self.params, self.offsets, self.numels, self.shapes):
            p._bg_grad = self.g_flat[off:off + n].view(shape)

    def _load(self, module, load_module_func, all_block_name, load, distributed_checkpoint):
        """The reference's ``param_init_fn`` with ``--load`` (parallel.py:79-89): every parameter-owning submodule of the
        wrapped block is filled by the family's ``load_module_func(load, tp_group, name, submodule, block, distributed)``,
        names relative to the block (``attention.attention.query_key_value`` ...)."""
        kinds = tuple(all_block_name or ())
        blocks = [m for m in module.modules() if kinds and isinstance(m, kinds)] or [module]
        with torch.no_grad():
            for block in blocks:
                for name, sub in block.named_modules():
                    if callable(getattr(sub, "reset_parameters", None)) and any(True for _ in sub.parameters(recurse=False)):
                        load_module_func(load, self.tp_group, name, sub, block, distributed_checkpoint)

    # ---- step protocol ------------------------------------------------------------------------------------------------
    def begin_step(self, params_changed=True):
        """Called once per training iteration before the first forward (the optimizer has updated the master)."""
        if params_changed:
            self._w_version += 1
            if self.w_pool is not None and self._w_valid:
                self.reshard()
            self._w_valid = False
        self._reduced_this_step = False
        self._started.clear()
        self._pending = False

    def unshard(self, prefetch=False):
        """Launch (once) the all-gather + fp32->bf16 cast of this layer's parameters on the unshard stream (C1)."""
        if self._w_valid:
            return
        if self.w_pool is not None:
            slot, cached = self.w_pool.acquire(self, self._w_version, demand=not prefetch)
            if slot is None:
                return                  # no free slot for a prefetch: gather on demand later
            self._bind_w(slot.buf)
            self._w_wait_event = slot.free_event   # the previous occupant's last use (its owner's compute stream)
            if cached:
                self._w_valid = True
                return
        self.be.unit_unshard(self)
        self._w_wait_event = None
        self._w_valid = True
        self.n_unshard += 1

    def wait_unshard(self):
        self.be.unit_wait_unshard(self)

    def reshard(self):
        """FULL_SHARD's free of the unsharded parameters after forward / backward (_runtime_utils.py _reshard): hand the slot
        back; the copy stays usable until another layer reclaims it."""
        if self.w_pool is None or not self._w_valid or self._in_use:
            return
        self.be.unit_wait_unshard(self)     # the releasing stream has then seen the gather it is about to order after
        self.w_pool.release(self, self.be.record_event())
        self._w_valid = False

    def evict(self, role):
        """Give a prefetched-but-unused slot back to the pool (called by the pool on a demand acquire)."""
        assert role == "param" and self._in_use == 0
        self.reshard()

    def acquire_grads(self):
        """zero3 with pooled gradients: take a G slot before this layer's backward writes its first wgrad."""
        if self.g_pool is None or self.G is not None:
            return
        slot, _ = self.g_pool.acquire(self)
        self.be.wait_event(slot.free_event)   # its previous occupant's reduce-scatter has read it (here and on the peers)
        self._bind_g(slot.buf)

    def release_grads(self):
        if self.g_pool is None or self.G is None:
            return
        self.g_pool.release(self, self.be.reduce_done_event())
        self.G = self.g_flat = None
        for p in self.params:
            p._bg_grad = None

    def read_full_params(self):
        """Clone of the gathered low-precision flat parameter (tests, checkpoint export)."""
        self.unshard()
        self.wait_unshard()
        out = self.w_flat.clone()
        self.reshard()
        return out

    def grad_started(self, p):
        return id(p) in self._started

    def mark_grad(self, p):
        self._started.add(id(p))
        self._pending = True

    def _collect_autograd_grads(self):
        """Parameters whose gradient was produced by plain autograd (norm weights, ...) -> into the flat G buffer."""
        for p in self.params:
            if p.grad is not None:
                g = p.grad
                if self.grad_started(p):
                    p._bg_grad.add_(g.to(p._bg_grad.dtype))
                else:
                    p._bg_grad.copy_(g)
                self.mark_grad(p)
                p.grad = None

    def _sum_sequence_parallel_grads(self):
        """C4: all-reduce the norm / SP-tagged grads over the TP group (sp_grad_reduce.py:104-123), packed in one message."""
        if not self._ln_params:
            return
        flat = torch.cat([p._bg_grad.reshape(-1) for p in self._ln_params])
        pad = (-flat.numel()) % 8
        if pad:
            flat = torch.cat([flat, flat.new_zeros(pad)])
        red = self.be.all_reduce(flat, self.tp_group)
        off = 0
        for p in self._ln_params:
            p._bg_grad.copy_(red[off:off + p.numel()].view_as(p._bg_grad))
            off += p.numel()

    def post_backward(self, sync_gradients):
        """After this layer's backward for one microbatch.  With ``sync_gradients`` launch the gradient reduction (C2/C3)."""
        self._collect_autograd_grads()
        if not sync_gradients:
            if self.g_pool is not None:
                raise RuntimeError("pooled zero3 gradients need a reduction after every backward (chunks == 1 or --no_async_grad_reduce)")
            return
        if self._tie is not None:           # reduced once per step, by finish_step, after the exchange with the other copy
            self._tie["deferred"] = True
            return
        self.reduce_now()

    def reduce_now(self):
        """Launch this unit's gradient reduction over its sharded-data-parallel group (C2/C3) on what G holds now."""
        if not self._pending:
            self.release_grads()
            return
        be = self.be
        for p in self.params:               # a parameter that received no gradient this step must contribute zeros
            if not self.grad_started(p):
                p._bg_grad.zero_()
        self._sum_sequence_parallel_grads()
        if self.uses_fused_optimizer():
            if self._reduced_this_step:
                raise RuntimeError("the fused optimizer needs one gradient reduction per step (async_grad_reduce)")
            if self.fused_opt.deferred:     # clipping: only the norm pass now, the update at optimizer.step()
                self.fused_opt.norm_pass(self)
            else:
                self.be.unit_reduce_adamw(self, self.fused_opt)
        else:
            self.be.unit_reduce(self, accumulate=self._reduced_this_step)
            self.flat_param.grad = self.master_grad
        self._reduced_this_step = True
        self._started.clear()
        self._pending = False
        self.n_reduce += 1
        # the reduction reads G on the reduce stream: the NEXT backward of this layer (another microbatch under
        # --no_async_grad_reduce) must not overwrite G before it has been read -- _pre_backward waits for this event
        self._reduce_event = be.reduce_done_event()
        self.release_grads()

    def write_master(self, full):
        """Replace the fp32 master by (this rank's part of) ``full`` -- a flat fp32 tensor of ``padded`` elements, identical on every
        member of the group -- and refresh the gathered low-precision copy."""
        with torch.no_grad():
            if self.dp_type == "ddp" or self.group.size == 1:
                self.flat_param.data.copy_(full)
            else:
                self.flat_param.data.copy_(full[self.rank_in_group * self.shard_elems:(self.rank_in_group + 1) * self.shard_elems])
            self._w_version += 1
            if self.w_pool is None:
                self.w_flat.copy_(full.to(self.param_dtype))
            else:
                if self._w_valid:
                    self.reshard()
                self._w_valid = False

    def finish_step(self):
        """Make the optimizer (current stream) wait for this step's reductions."""
        self.be.finish_reductions()

    # ---- introspection (tests, checkpointing) ---------------------------------------------------------------------------
    def named_slices(self, flat):
        """name -> view of ``flat`` (a full-length flat tensor: ``w_flat``, ``g_flat`` or a gathered master)."""
        names = {id(p): n for n, p in self.module.named_parameters()}
        return {names[id(p)]: flat[off:off + n].view(p.shape) for p, off, n in zip(self.params, self.offsets, self.numels)}

    def local_master_slices(self, tensor=None):
        """For an un-sharded unit (group of 1, or ddp): name -> fp32 master (or ``tensor``, e.g. ``master_grad``) views."""
        assert self.dp_type == "ddp" or self.group.size == 1, "sharded master: gather it first"
        return self.named_slices(self.flat_param.data if tensor is None else tensor)


# ---------------------------------------------------------------------------------------------------------------------
# module wrappers
# ---------------------------------------------------------------------------------------------------------------------
class _PostBackwardHook(torch.autograd.Function):
    """Identity on the layer INPUTS; its backward runs after every gradient of the layer has been produced."""

    @staticmethod
    def forward(ctx, wrapper, *tensors):
        ctx.wrapper = wrapper
        return tensors if len(tensors) > 1 else tensors[0]

    @staticmethod
    def backward(ctx, *grads):
        ctx.wrapper._post_backward()
        return (None,) + grads


class _PreBackwardHook(torch.autograd.Function):
    """Identity on the layer OUTPUTS; its backward runs before the layer's backward (zero3 re-gather point)."""

    @staticmethod
    def forward(ctx, wrapper, *tensors):
        ctx.wrapper = wrapper
        return tensors if len(tensors) > 1 else tensors[0]

    @staticmethod
    def backward(ctx, *grads):
        ctx.wrapper._pre_backward()
        return (None,) + grads


class _CheckpointFn(torch.autograd.Function):
    """Activation checkpointing of one wrapped layer (parallel.py:229-240 checkpoint_wrapper): keep only the inputs,
    recompute inside backward -- under the backward unshard, so no third all-gather (SURVEY 8h)."""

    @staticmethod
    def forward(ctx, wrapper, kwargs, anchor, *inputs):
        # ``anchor``: an empty tensor that requires grad, so that this node is part of the graph (and its backward runs, producing
        # the layer's PARAMETER gradients) even when no activation input requires grad (a checkpointed first layer).
        ctx.wrapper, ctx.kwargs = wrapper, kwargs
        ctx.save_for_backward(*[t for t in inputs if torch.is_tensor(t)])
        ctx.is_tensor = [torch.is_tensor(t) for t in inputs]
        ctx.others = [t for t in inputs if not torch.is_tensor(t)]
        # dropout inside the layer must draw the same masks when it is recomputed (checkpoint_wrapper preserves the RNG state,
        # torch/utils/checkpoint.py); only captured when dropout is on.  The hidden-state masks need the microbatch's dropout
        # context (the backward may run under another microbatch's), attention-probability dropout the default generator AND the
        # model-parallel tracker's streams.
        ctx.rng = None
        if wrapper.preserve_rng:
            dev = next((t.device for t in inputs if torch.is_tensor(t) and t.is_cuda), None)
            ctx.rng = (torch.get_rng_state(), dev, torch.cuda.get_rng_state(dev) if dev is not None else None,
                       dropout_random.get_context(), dropout_random.get_rng_tracker().get_states())
        with torch.no_grad():
            out = wrapper.module(*inputs, **kwargs)
        return out

    @staticmethod
    def backward(ctx, *grads):
        wrapper = ctx.wrapper
        wrapper._pre_backward()
        saved, others = list(ctx.saved_tensors), list(ctx.others)
        inputs = []
        for is_t in ctx.is_tensor:
            if is_t:
                t = saved.pop(0).detach()
                t.requires_grad_(t.is_floating_point())
                inputs.append(t)
            else:
                inputs.append(others.pop(0))
        if ctx.rng is not None:
            cpu_state, dev, cuda_state, drop_ctx, tracker_states = ctx.rng
            tracker = dropout_random.get_rng_tracker()
            now = (torch.get_rng_state(), torch.cuda.get_rng_state(dev) if dev is not None else None, dropout_random.get_context(),
                   tracker.get_states())
            torch.set_rng_state(cpu_state)
            if dev is not None:
                torch.cuda.set_rng_state(cuda_state, dev)
            dropout_random.set_context(drop_ctx)
            tracker.set_states(tracker_states)
        with torch.enable_grad():
            out = wrapper.module(*inputs, **ctx.kwargs)
        if ctx.rng is not None:
            torch.set_rng_state(now[0])
            if dev is not None:
                torch.cuda.set_rng_state(now[1], dev)
            dropout_random.set_context(now[2])
            tracker.set_states(now[3])
        outs = out if isinstance(out, (tuple, list)) else (out,)
        pairs = [(o, g) for o, g in zip(outs, grads) if torch.is_tensor(o) and o.requires_grad and g is not None]
        torch.autograd.backward([o for o, _ in pairs], [g for _, g in pairs])
        wrapper._post_backward()
        return (None, None, None) + tuple(t.grad if torch.is_tensor(t) and t.requires_grad else None for t in inputs)


class DataParallelModule(nn.Module):
    """A pipeline-stage layer wrapped in its ShardedUnit (+ optional checkpointing).  Plays the role of the per-layer
    FSDP wrapper (parallel.py:163-213) and of ``checkpoint_wrapper`` (parallel.py:229-240)."""

    def __init__(self, module, unit, checkpoint=False):
        super().__init__()
        self.module, self.unit, self.checkpoint = module, unit, checkpoint
        self.next_unit = None           # forward prefetch target (the next layer of the stage)
        self.prev_unit = None           # backward prefetch target
        self.sync_gradients = True      # set per microbatch by the schedule (PipelineParallel.set_last_batch)
        self._fired = True              # did _post_backward run during the current backward_step?
        self._anchor = None
        try:
            from .arguments import get_args
            args = get_args()
            self.preserve_rng = any(float(getattr(args, k, 0.0)) > 0.0 for k in ("dropout_prob", "hidden_dropout", "attention_dropout"))
        except RuntimeError:
            self.preserve_rng = False

    def _pre_backward(self):
        unit = self.unit
        if unit._reduce_event is not None:      # G is about to be rewritten: its previous reduction must have read it
            unit.be.wait_event(unit._reduce_event)
            unit._reduce_event = None
        unit.unshard()
        if self.prev_unit is not None:
            self.prev_unit.unshard(prefetch=True)   # backward prefetch: the previous layer's re-gather overlaps this backward
        unit.wait_unshard()
        unit._in_use += 1
        unit.acquire_grads()

    def _post_backward(self):
        self._fired = True
        unit = self.unit
        unit.post_backward(self.sync_gradients)
        unit._in_use = max(0, unit._in_use - 1)
        unit.reshard()

    def arm_backward(self):
        """Called by the schedule right before ``autograd.backward`` of one microbatch."""
        self._fired = False

    def flush_backward(self):
        """Called by the schedule right after ``autograd.backward``: layers whose inputs carry no gradient (embedding)
        never see their input-side hook fire."""
        if not self._fired:
            self._post_backward()

    def forward(self, *inputs, **kwargs):
        unit = self.unit
        unit.unshard()
        if self.next_unit is not None:
            self.next_unit.unshard(prefetch=True)   # the next layer's all-gather overlaps this layer's compute
        unit.wait_unshard()
        unit._in_use += 1
        try:
            return self._forward(inputs, kwargs)
        finally:
            unit._in_use -= 1
            unit.reshard()              # zero3: free the gathered copy (FULL_SHARD reshards after forward)

    def _forward(self, inputs, kwargs):
        grad_mode = torch.is_grad_enabled()
        if self.checkpoint and grad_mode:
            if self._anchor is None or self._anchor.device != self.unit.flat_param.device:
                self._anchor = torch.empty(0, device=self.unit.flat_param.device, requires_grad=True)
            return _CheckpointFn.apply(self, kwargs, self._anchor, *inputs)
        if grad_mode:
            float_in = [i for i, t in enumerate(inputs) if torch.is_tensor(t) and t.is_floating_point() and t.requires_grad]
            if float_in:
                hooked = _PostBackwardHook.apply(self, *[inputs[i] for i in float_in])
                hooked = hooked if isinstance(hooked, tuple) else (hooked,)
                inputs = list(inputs)
                for i, h in zip(float_in, hooked):
                    inputs[i] = h
        out = self.module(*inputs, **kwargs)
        if grad_mode:
            if isinstance(out, tuple):
                out = _PreBackwardHook.apply(self, *out)
            else:
                out = _PreBackwardHook.apply(self, out)
        return out


class Module_with_relocation(nn.Module):
    """Redistribute the activations entering a layer whose (tp|sp, cp) differs from its predecessor's
    (parallel.py:279-313).  Float tensors take the sequence-parallel aware path, integer tensors (tokens, labels, masks)
    the plain batch split / gather."""

    def __init__(self, module, allgather_tp_sp_group, allgather_cp_group, allgather_tp_sp_cp_group, split_tp_sp_group,
                 split_cp_group, split_tp_sp_cp_group, fused_allgather_group, fused_split_group):
        super().__init__()
        self.module = module
        self.groups = (allgather_tp_sp_group, allgather_cp_group, allgather_tp_sp_cp_group, split_tp_sp_group, split_cp_group,
                       split_tp_sp_cp_group, fused_allgather_group, fused_split_group)
        if hasattr(module, "get_extended_attention_mask"):
            self.get_extended_attention_mask = module.get_extended_attention_mask

    def forward(self, *inputs, **kwargs):
        moved = tuple(fused_split_allgather(x, x.is_floating_point(), *self.groups) if torch.is_tensor(x) else x for x in inputs)
        return self.module(*moved, **kwargs)


def wrap_modules_relocation(module_list, allgather_tp_sp_groups, allgather_cp_groups, allgather_tp_sp_cp_groups,
                            split_tp_sp_groups, split_cp_groups, split_tp_sp_cp_groups, fused_allgather_groups,
                            fused_split_groups):
    """parallel.py:435-451: wrap layer i when any of its relocation groups is set."""
    assert len(module_list) == len(allgather_tp_sp_groups) == len(fused_split_groups)
    for i in range(len(module_list)):
        groups = (allgather_tp_sp_groups[i], allgather_cp_groups[i], allgather_tp_sp_cp_groups[i], split_tp_sp_groups[i],
                  split_cp_groups[i], split_tp_sp_cp_groups[i], fused_allgather_groups[i], fused_split_groups[i])
        if any(g is not None for g in groups):
            module_list[i] = Module_with_relocation(module_list[i], *groups)
    return module_list

"""The execution backend the layer/runtime code talks to.

Product = ``CudaBackend``: every method lands in a hand-written sm_90a kernel through the C ABI (``_bg``), or --
for attention only -- in the flash-attn library the reference itself calls (transformer.py:495, SURVEY K3).
There is no CPU implementation in this package: ``get_backend()`` raises when the extension or a GPU is missing.

Host-logic tests run the same layer/schedule code on CPU by *injecting* a backend with ``set_backend()``; that
backend (``oracle/gloo_backend.py``) lives with the oracle, is never imported from here, and is only ever installed
by tests/ and bench.py's reference arm.
"""
import contextlib
import os

import torch

from . import world as _world

_BACKEND = None


def set_backend(backend):
    global _BACKEND
    _BACKEND = backend
    return backend


def get_backend():
    global _BACKEND
    if _BACKEND is None:
        _BACKEND = CudaBackend()
    return _BACKEND


def reset_backend():
    global _BACKEND
    if _BACKEND is not None and hasattr(_BACKEND, "close"):
        _BACKEND.close()
    _BACKEND = None


class StagingLayout:
    """Byte layout of a group's activation staging buffer reserved for ``n`` data bytes (a multiple of 256):

      [0, n)                   region 0: general staging, the all-gather landing, the unfused GEMM output and the stage of
                               ``all_gather_gemm``.  The unfused dgrad GEMM + collective writes here over the re-gathered input of
                               the same layer, so that layer's wgrad GEMM must have read the input before.
      [n, 2n)                  partial tiles of the fused GEMM + reduce-scatter / all-reduce
      [2n, 3n)                 the fused all-reduce result, which every member's tile reducer broadcasts into
      [3n, 3n + F/2)           per-tile arrival counters of the scattering GEMMs
      [3n + F/2, 3n + F)       per-block arrival counters of the gathering GEMM

    F = FLAG_BYTES; the buffer is 3n + F bytes.  The counters are zero at rest."""

    FLAG_BYTES = 1 << 16
    COUNTER_BYTES = FLAG_BYTES // 2        # each of the two counter blocks

    def __init__(self, n):
        self.n = n
        self.partials = n
        self.result = 2 * n
        self.scatter_counters = 3 * n
        self.gather_counters = 3 * n + self.COUNTER_BYTES
        self.total = 3 * n + self.FLAG_BYTES


# fusion pays when the GEMM lasts at least as long as the transfer of its output; below that the GEMM outruns NVLink and the fused
# kernel only adds its reducer tail (thresholds from measurements on an earlier GPU; not re-measured on H100)
FUSE_MIN_K = 3072          # GEMM + reduce-scatter
FUSE_AR_MIN_K = 2048       # GEMM + all-reduce
FUSE_ENV = {"gemm_rs": "HGB_FUSE_GEMM_RS", "gemm_ar": "HGB_FUSE_GEMM_AR", "ag_gemm": "HGB_FUSE_AG_GEMM"}


def fusion_allowed(kind, m, n, k, p, data_bytes, on, force=False):
    """Does the fused GEMM + collective ``kind`` ("gemm_rs", "gemm_ar" or "ag_gemm") run for the [m, n] = [m, k] x [k, n] GEMM
    (m: the full, gathered / unscattered rows) on a group of ``p`` ranks whose staging buffer holds ``data_bytes`` (None: none
    reserved)?  ``on``: the kind's switch is not "0"; ``force``: it is "force", which lifts the K threshold (k None: no threshold).
    The fused kernels need M in whole 128-row tiles per rank and their arrival counters inside the staging buffer's counter block."""
    if not on or p < 2 or m % (p * 128) or data_bytes is None:
        return False
    if kind == "ag_gemm":
        return k % 8 == 0 and data_bytes >= 2 * m * k and 4 * (m // 128) <= StagingLayout.COUNTER_BYTES
    tiles = (m // p // 128) * ((n + 127) // 128)
    if kind == "gemm_rs":
        min_k, counter_bytes = FUSE_MIN_K, StagingLayout.COUNTER_BYTES
    else:
        # half the block (the C side's limit is the whole block); raising it would move shapes onto the fused path
        min_k, counter_bytes = FUSE_AR_MIN_K, StagingLayout.COUNTER_BYTES // 2
    return (n % 8 == 0 and (k is None or k >= min_k or force) and data_bytes >= 2 * m * n
            and 4 * tiles <= counter_bytes)


class _SymBuffers:
    """The backend's own symmetric (peer-visible) buffers, one per (purpose, group).  Every member reserves them identically before
    ``exchange()``.  A larger request before then allocates a new buffer and leaves the smaller one in the arena (every member does
    the same, so the arena layouts stay identical); after ``exchange()`` it raises."""

    def __init__(self, comm):
        self.comm = comm
        self._bufs = {}            # (purpose, group ranks) -> (SymBuffer, size)

    def reserve(self, purpose, group, size, nbytes):
        """The ``purpose`` buffer of ``group`` for ``size`` (in the purpose's own unit); when the current one is smaller, allocates
        ``nbytes``.  -> (buffer, allocated by this call)"""
        key = (purpose, tuple(group.ranks))
        cur = self._bufs.get(key)
        if cur is not None and cur[1] >= size:
            return cur[0], False
        if cur is not None and cur[0].offsets is not None:
            from ... import _bg
            raise _bg.BgError("%s buffer of group %s holds %d, need %d (reserve before exchange())" % (purpose, key[1], cur[1], size))
        buf = self.comm.sym_alloc(group, nbytes)
        self._bufs[key] = (buf, size)
        return buf, True

    def get(self, purpose, group):
        """-> (buffer, size) as reserved, or (None, 0)"""
        return self._bufs.get((purpose, tuple(group.ranks)), (None, 0))


class CudaBackend:
    """H100 backend: symmetric-memory communicator + fused kernels."""

    name = "cuda-sm90a"
    is_cuda = True

    def __init__(self, comm=None, arena_bytes=None, device=None):
        from ... import _bg
        if not torch.cuda.is_available():
            raise _bg.BgError("hetu-galvatron_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.bg = _bg
        _bg.lib()
        self.rank, self.world = _world.get_rank(), _world.get_world_size()
        self.device_index = _world.get_local_rank() % torch.cuda.device_count() if device is None else device
        torch.cuda.set_device(self.device_index)
        self.device = torch.device("cuda", self.device_index)
        self.nvls = False
        self.nvls_regions = {}     # group ranks -> multicast-bound arena range, set by exchange()
        if comm is None:
            if arena_bytes is None:
                arena_bytes = int(os.environ.get("HGB_ARENA_BYTES", 0))
                if not arena_bytes:
                    try:
                        from .arguments import get_args
                        arena_bytes = int(getattr(get_args(), "arena_bytes", 0))
                    except RuntimeError:
                        arena_bytes = 0
                arena_bytes = arena_bytes or (1 << 30)
            # NVLS (default on a multi-GPU job; HGB_NVLS=0 switches it off): the arena comes from the virtual-memory API so that
            # NVSwitch multicast objects can bind it; collectives on multicast-bound buffers then reduce / replicate inside
            # the switch above 1 MiB.  A driver or fabric without multicast keeps the cudaMalloc + cudaIpc arena.
            self.nvls = os.environ.get("HGB_NVLS", "1") == "1" and self.world > 1
            comm = None
            if self.nvls:
                try:
                    comm = _bg.BgComm(self.rank, self.world, self.device_index, arena_bytes, vmm=True)
                    if not comm.arena_mode()[1]:
                        comm.close()
                        comm = None
                except _bg.BgError:
                    comm = None
                if self.world > 1:      # every rank must take the same decision (one box, one driver: it does; checked anyway)
                    import torch.distributed as dist
                    flags = [None] * self.world
                    dist.all_gather_object(flags, comm is not None)
                    if not all(flags):
                        if comm is not None:
                            comm.close()
                        comm = None
                self.nvls = comm is not None
            if comm is None:
                comm = _bg.BgComm(self.rank, self.world, self.device_index, arena_bytes, vmm=False)
            if self.world > 1:
                comm.connect_vmm() if self.nvls else comm.connect_ipc()
        self.comm = comm
        if os.environ.get("HGB_TIMEOUT_MS"):      # device-side barrier timeout (default 60 s): shorter for debugging runs
            _bg.set_tunable("timeout_ms", int(os.environ["HGB_TIMEOUT_MS"]))
        # communication streams are HIGH priority: the CTA distributor then places a slim collective CTA (which fits beside the
        # persistent GEMM CTAs) ahead of any compute grid that is still waiting for SMs, instead of queueing it behind that grid
        self.unshard_stream = torch.cuda.Stream(device=self.device, priority=-1)
        self.reduce_stream = torch.cuda.Stream(device=self.device, priority=-1)
        self.p2p_stream = torch.cuda.Stream(device=self.device, priority=-1)
        self.comm_stream = torch.cuda.Stream(device=self.device, priority=-1)  # push kernels of the fused all-gather + GEMM; overlapped gathers
        self.fuse = {kind: os.environ.get(env, "1") != "0" for kind, env in FUSE_ENV.items()}
        self.n_fused = {"gemm_rs": 0, "gemm_ar": 0, "ag_gemm": 0}
        self.comm_profile = None   # bench.py: {kind: [(start_event, end_event, algorithmic_bus_bytes)]} while timing the collectives
        self.attn_impl = os.environ.get("HGB_ATTN", "cudnn")
        self._bufs = _SymBuffers(comm)
        self._cp_rings = {}        # group ranks -> _CpRing
        self.world_group = None    # the whole job as one group, once its staging is reserved (clip_grad_norm's all-reduce)
        self._scratch = {}
        self.gemm_profile = None   # bench.py: list of (start_event, end_event, flops) while timing the dominant kernel
        # RMSNorm / LayerNorm backward: one fp32 weight-gradient partial row per CTA, 3 CTAs of 256 threads x <= 76 registers per SM
        self.norm_partials = 3 * torch.cuda.get_device_properties(self.device).multi_processor_count

    def close(self):
        if self.comm is not None:
            torch.cuda.synchronize()
            self.comm.close()
            self.comm = None

    # ---- in-step timing of the collectives (bench.py path legs) ----------------------------------------------------
    def _timed(self, kind, bus_bytes, stream=None, flops=0.0):
        """Context manager: when ``comm_profile`` is a dict, bracket the launch with CUDA events on its stream and record the
        algorithmic bus bytes (nccl-tests convention: AG/RS/A2A (p-1)/p*N, AR 2(p-1)/p*N, p2p N) of the call -- and, for a fused
        GEMM + collective, the GEMM's FLOPs (its roofline is the slower of FLOPs / GEMM peak and bytes / NVLink)."""
        return _Timed(self, kind, bus_bytes, stream, flops)

    # ---- memory -------------------------------------------------------------------------------------------
    def sym_alloc(self, group, nbytes):
        return self.comm.sym_alloc(group, nbytes)

    def exchange(self):
        self.comm.exchange()
        if self.nvls:
            self.nvls_regions = self.comm.setup_nvls()

    def reserve_staging(self, group, nbytes):
        """Per-group activation staging buffer (peer-visible, laid out as ``StagingLayout`` for ``nbytes`` rounded up to 256).  Must
        be called (identically on all members) before ``exchange()``; later requests larger than the reservation raise."""
        if group is None or group.size == 1:
            return None
        layout = StagingLayout((int(nbytes) + 255) // 256 * 256)
        buf, new = self._bufs.reserve("staging", group, layout.n, layout.total)
        if new:
            buf.layout = layout
            buf.u8[layout.scatter_counters:].zero_()
        return buf

    def reserve_cp_ring(self, group, elems):
        """Receive slots of the context-parallel ring for ``group`` (``cp_comm="ring"``): a region of their own, sized for a local
        K block of ``elems`` elements -- per step parity one [K | V] bf16 slot and one [dK | dV] fp32 slot, 24 B per element.  Before
        ``exchange()``, identically on every member."""
        if group is None or group.size == 1:
            return
        elems = (int(elems) + 7) // 8 * 8
        self._bufs.reserve("cp_ring", group, elems, _CpRing.slot_bytes(elems))

    def cp_ring(self, group):
        """The ring transport of ``group`` (one per group: its flags' first-use state is shared by every layer on the group)."""
        key = tuple(group.ranks)
        if key not in self._cp_rings:
            buf, elems = self._bufs.get("cp_ring", group)
            if buf is None:
                raise self.bg.BgError("no cp ring slots reserved for group %s (models built with cp_comm='ring' reserve them)" % (key,))
            self._cp_rings[key] = _CpRing(self.comm, group, buf, elems, comm_stream=self.comm_stream, counts=self.n_fused)
        return self._cp_rings[key]

    def lse_merge(self, blk_out, blk_lse, acc_out, acc_lse, final_out=None, row_off=0, init=False):
        self.bg.lse_merge(blk_out.contiguous(), blk_lse.contiguous(), acc_out, acc_lse, final_out, row_off, init)

    def staging(self, group, nbytes, byte_offset=0):
        buf, n = self._bufs.get("staging", group)
        if buf is None or n < nbytes + byte_offset:
            raise self.bg.BgError("no staging buffer of %d B reserved for group %s" % (nbytes + byte_offset, group.ranks))
        return buf

    def staging_tensor(self, group, shape, dtype, byte_offset=0):
        numel = 1
        for s in shape:
            numel *= int(s)
        nbytes = numel * torch.empty((), dtype=dtype).element_size()
        buf = self.staging(group, nbytes, byte_offset)
        return buf.u8[byte_offset: byte_offset + nbytes].view(dtype).view(*shape), buf

    def _is_staging(self, t, buf):
        base = buf.u8.data_ptr()
        return base <= t.data_ptr() < base + buf.layout.n

    def _stage(self, x, group, byte_offset=0):
        """Make ``x`` peer-visible: no-op when it already lives in the group's staging buffer."""
        buf = self.staging(group, x.numel() * x.element_size(), byte_offset)
        if self._is_staging(x, buf):
            return buf, x.data_ptr() - buf.u8.data_ptr()
        dst = buf.u8[byte_offset: byte_offset + x.numel() * x.element_size()].view(x.dtype)
        dst.copy_(x.reshape(-1))
        return buf, byte_offset

    # ---- sharded-unit collectives (side streams) ------------------------------------------------------------------
    def unit_unshard(self, unit):
        """C1 on the unshard stream: all-gather + fp32->bf16 cast of the unit's flat parameter."""
        with torch.cuda.stream(self.unshard_stream):
            if getattr(unit, "_w_wait_event", None) is not None:    # pooled slot: its previous occupant's last use
                self.unshard_stream.wait_event(unit._w_wait_event)
            if unit.dp_type == "ddp":
                self.cast(unit.flat_param.data, unit.w_flat)
            else:
                d = unit.group.size
                with self._timed("sdp_all_gather", (d - 1) / d * unit.padded * 2, self.unshard_stream):
                    self.comm.all_gather_cast(unit.group, unit.flat_param.data, unit.W, shard_elems=unit.shard_elems,
                                              lane=self.bg.LANE_UNSHARD, dst_dtype=unit.param_dtype)
            unit._unshard_event = torch.cuda.Event()
            unit._unshard_event.record(self.unshard_stream)

    def unit_wait_unshard(self, unit):
        if unit._unshard_event is not None:
            torch.cuda.current_stream().wait_event(unit._unshard_event)
            unit._unshard_event = None

    def begin_step(self):
        """The optimizer (current stream) has rewritten the masters: the unshard stream must see that."""
        self.unshard_stream.wait_stream(torch.cuda.current_stream())

    @contextlib.contextmanager
    def _on_reduce_stream(self, unit, kind=None):
        """Run the body on the reduce stream, ordered after the work already queued on the current stream (the unit's backward);
        with ``kind``, time it as that reduce-scatter of the unit's gradient."""
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        with torch.cuda.stream(self.reduce_stream):
            self.reduce_stream.wait_event(ev)
            if kind is None:
                yield
            else:
                d, gsz = unit.group.size, (4 if unit.reduce_dtype == torch.float32 else 2)
                with self._timed(kind, (d - 1) / d * unit.padded * gsz, self.reduce_stream):
                    yield

    def unit_reduce(self, unit, accumulate):
        """C2/C3 on the reduce stream, ordered after the unit's backward on the current stream."""
        if unit.dp_type != "ddp":
            with self._on_reduce_stream(unit, "sdp_reduce_scatter"):
                self.comm.reduce_scatter_acc(unit.group, unit.G, unit.reduce_dtype, unit.master_grad,
                                             shard_elems=unit.shard_elems, prescale=1.0 / unit.prediv,
                                             postscale=1.0 / unit.postdiv, accumulate=accumulate, lane=self.bg.LANE_REDUCE)
            return
        with self._on_reduce_stream(unit):
            if unit.group.size == 1:
                self.cast(unit.g_flat, unit.master_grad, accumulate=accumulate)
            else:  # DDP layers: all-reduce of the full flat gradient (_runtime_utils.py:932-950), then cast/accumulate
                key = (unit.reduce_dtype, unit.padded)
                tmp = self._scratch.get(key)
                if tmp is None:
                    tmp = self._scratch[key] = torch.empty(unit.padded, dtype=unit.reduce_dtype, device=self.device)
                self.comm.all_reduce(unit.group, unit.G, tmp, elems=unit.padded, scale=1.0 / (unit.prediv * unit.postdiv),
                                     lane=self.bg.LANE_REDUCE)
                self.cast(tmp, unit.master_grad, accumulate=accumulate)

    def unit_reduce_adamw(self, unit, opt, clip_coef=None):
        """C2 with the AdamW epilogue (reduce stream): gradients are consumed in registers, no fp32 gradient shard.  ``clip_coef``
        (fp32 device scalar): the step pass of deferred clipping, the reduced gradient multiplied by it."""
        lr, b1, b2, eps, wd, step = opt.hyper()
        with self._on_reduce_stream(unit, "sdp_reduce_scatter_adamw"):
            if clip_coef is None:
                self.comm.reduce_scatter_adamw(unit.group, unit.G, unit.reduce_dtype, unit.flat_param.data, unit.exp_avg,
                                               unit.exp_avg_sq, unit.shard_elems, 1.0 / unit.prediv, 1.0 / unit.postdiv, lr, b1, b2,
                                               eps, wd, step, lane=self.bg.LANE_REDUCE)
            else:
                self.comm.reduce_scatter_adamw_clipped(unit.group, unit.G, unit.reduce_dtype, unit.flat_param.data, unit.exp_avg,
                                                       unit.exp_avg_sq, unit.shard_elems, 1.0 / unit.prediv, 1.0 / unit.postdiv, lr,
                                                       b1, b2, eps, wd, step, clip_coef, lane=self.bg.LANE_REDUCE)
                self._count("rs_adamw_clipped")

    def clip_partials(self, n_units):
        """Zeroed fp32 [n_units, k]: one row per unit for the norm pass's per-warp sums of squares (4 warps x the largest grid)."""
        k = 4 * max(self.bg.get_tunable("comm_ctas"), self.bg.get_tunable("local_ctas"))
        return torch.zeros(n_units, k, dtype=torch.float32, device=self.device)

    def unit_reduce_sumsq(self, unit, partials, skip, into_master=False):
        """Norm pass of deferred clipping (reduce stream): the unit's reduce-scatter, whose epilogue only writes the per-warp sums of
        squares of the reduced gradient into ``partials`` (leaving out the shard-relative ranges ``skip``); ``into_master``: also
        the fp32 gradient shard (units whose G cannot be read again at the step)."""
        with self._on_reduce_stream(unit, "sdp_reduce_scatter_sumsq"):
            self.comm.reduce_scatter_sumsq(unit.group, unit.G, unit.reduce_dtype, unit.shard_elems, 1.0 / unit.prediv,
                                           1.0 / unit.postdiv, partials, skip, dst=unit.master_grad if into_master else None,
                                           lane=self.bg.LANE_REDUCE)
        self._count("rs_sumsq")

    def unit_adamw_clipped(self, unit, opt, clip_coef):
        """The clipped AdamW step on the unit's fp32 gradient shard (current stream, after ``finish_reductions``)."""
        lr, b1, b2, eps, wd, step = opt.hyper()
        self.bg.adamw_clipped(unit.flat_param.data, unit.exp_avg, unit.exp_avg_sq, unit.master_grad, lr, b1, b2, eps, wd, step, clip_coef)
        self._count("adamw_clipped")

    def _count(self, kind):
        self.n_fused[kind] = self.n_fused.get(kind, 0) + 1

    def finish_reductions(self):
        torch.cuda.current_stream().wait_stream(self.reduce_stream)

    # ---- checkpoint export: gather the fp32 master shards of one unit (C1 with an fp32 destination) -----------------------
    def reserve_checkpoint_gather(self, group, nbytes):
        """Peer-visible landing buffer for ``gather_master`` (one per group, sized for its largest unit); before ``exchange()``."""
        if group is None or group.size == 1:
            return
        # its size is what sym_alloc allocates for the request (a whole number of 256-byte blocks)
        self._bufs.reserve("checkpoint_gather", group, (int(nbytes) + 255) // 256 * 256, int(nbytes))

    def gather_master(self, unit):
        """Full fp32 flat parameter of ``unit`` on every member of its group (collective)."""
        if unit.dp_type == "ddp" or unit.group.size == 1:
            return unit.flat_param.data
        buf, nbytes = self._bufs.get("checkpoint_gather", unit.group)
        if buf is None or nbytes < unit.padded * 4:
            raise self.bg.BgError("no checkpoint gather buffer reserved for group %s: construct the model with args.save set" % (unit.group.ranks,))
        self.comm.all_gather_cast(unit.group, unit.flat_param.data, buf, shard_elems=unit.shard_elems, lane=self.bg.LANE_MISC,
                                  dst_dtype=torch.float32)
        return buf.view(torch.float32, unit.padded).clone()

    # ---- tied word embeddings across pipeline stages (C14): the two copies' gradient ranges, summed in place over peer memory ---------
    supports_tied_embedding_exchange = True

    def register_tied_grad(self, unit, param, group):
        """``param``'s range of the unit's gradient buffer G as a symmetric buffer over ``group`` (the embedding group: the first and
        the last stage, which hold the two copies of the tied matrix).  No memory of its own.  Before ``exchange()``, in the same
        order on both members; ``exchange()`` refuses the pair when the two ranges differ in size."""
        i = next(k for k, p in enumerate(unit.params) if p is param)
        esz = unit.g_flat.element_size()
        n = (unit.numels[i] + 7) // 8 * 8        # (the flat layout starts every parameter on a whole 8-element block)
        return self.comm.sym_register(group, unit.G.offset + unit.offsets[i] * esz, n * esz)

    def tied_grad_sum(self, unit, buf):
        """Both copies' gradients (``buf`` from ``register_tied_grad``) <- their sum, in place, on the reduce stream after the
        backward already queued; the unit's reduction, launched next on the same stream, reads the sum."""
        with self._on_reduce_stream(unit):
            self.comm.pair_sum_inplace(buf.group, buf, unit.reduce_dtype, lane=self.bg.LANE_REDUCE)
        self._count("tied_pair_sum")

    def tied_average(self, buf, x):
        """fp32 ``x`` <- (x + the other member's x) / 2 in place (construction).  The matrix passes through the registered gradient
        range -- unused before the first backward -- in as many pieces as it needs (two when G is bf16); the range is left zeroed."""
        flat = x.view(-1)
        stage = buf.u8.view(torch.float32)
        cap = stage.numel() // 4 * 4
        for lo in range(0, flat.numel(), cap):
            k = min(cap, flat.numel() - lo)
            kp = (k + 3) // 4 * 4
            stage[:k].copy_(flat[lo:lo + k])
            stage[k:kp].zero_()
            self.comm.pair_sum_inplace(buf.group, buf, torch.float32, elems=kp, scale=0.5, lane=self.bg.LANE_REDUCE)
            self._count("tied_pair_sum")
            flat[lo:lo + k].copy_(stage[:k])
        buf.u8.zero_()

    def barrier_all(self):
        torch.cuda.synchronize()
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            dist.barrier()

    # ---- events (ordering between successive occupants of a pooled zero3 buffer) ------------------------------------------
    def record_event(self):
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        return ev

    def reduce_done_event(self):
        ev = torch.cuda.Event()
        ev.record(self.reduce_stream)
        return ev

    def wait_event(self, ev):
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)

    def make_stage_link(self, my_rank, peer_rank, max_bytes, send_flag_base, recv_flag_base):
        from .pipeline.pipeline import _StageLink
        return _StageLink(self, my_rank, peer_rank, max_bytes, send_flag_base, recv_flag_base)

    # ---- activation collectives (compute stream, LANE_ACT) ---------------------------------------------------
    def all_reduce(self, x, group, op="sum"):
        if group is None or group.size == 1:
            return x
        x = x.contiguous()
        if x.numel() % _vec(x):
            out = torch.empty_like(x)
            self._all_reduce_padded(x, group, op, out)
            return out
        buf, off = self._stage(x, group)
        out = torch.empty_like(x)
        # (above 1 MiB on a multicast-bound staging buffer the C side reduces and replicates inside the NVSwitch)
        with self._timed("all_reduce", 2.0 * (group.size - 1) / group.size * x.numel() * x.element_size()):
            self.comm.all_reduce(group, buf, out, elems=x.numel(), op=self.bg.MAX if op == "max" else self.bg.SUM,
                                 src_byte_offset=off)
        return out

    def _all_reduce_padded(self, x, group, op, out):
        n = x.numel()
        padded = (n + 7) // 8 * 8
        buf = self.staging(group, padded * x.element_size())
        tmp_in = buf.u8[: padded * x.element_size()].view(x.dtype)
        tmp_in[:n].copy_(x.reshape(-1))
        tmp_in[n:].zero_()
        tmp_out = torch.empty(padded, dtype=x.dtype, device=x.device)
        self.comm.all_reduce(group, buf, tmp_out, elems=padded, op=self.bg.MAX if op == "max" else self.bg.SUM)
        out.copy_(tmp_out[:n].view_as(out))

    def all_gather_first_dim(self, x, group):
        """[s, ...] -> [n*s, ...] in rank order (mappings_group.py:84-102 _gather_along_first_dim)."""
        if group is None or group.size == 1:
            return x
        x = x.contiguous()
        buf, off = self._stage(x, group)
        n = group.size
        out = torch.empty((n * x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        chunk = x.numel()
        self._check_vec(x, chunk)
        with self._timed("all_gather", (n - 1) / n * out.numel() * out.element_size()):
            self.comm.all_to_all_rows(group, [dict(src=buf, src_byte_offset=off, dst=out, batch=1, rows=1, row_elems=chunk,
                                                   src_bs=0, src_rs=0, src_me_off=0, dst_bs=0, dst_rs=0, dst_peer_off=chunk)], x.dtype)
        return out

    def all_gather_into_staging(self, x, group, overlap=False):
        """Push all-gather whose result stays in the group's staging buffer (operand of the next GEMM only):
        the Megatron-SP gather of layers.py:399-413.  ``overlap``: launch it on the communication stream, ordered after the
        work already in the current stream, and return (tensor, event) -- the caller runs independent work (the dgrad GEMM,
        as layers.py:449-462 overlaps them) and waits for the event before touching the gathered tensor."""
        x = x.contiguous()
        n = group.size
        out, buf = self.staging_tensor(group, (n * x.shape[0],) + tuple(x.shape[1:]), x.dtype)
        self._check_vec(x, x.numel())
        bus = (n - 1) / n * out.numel() * out.element_size()
        if not overlap:
            with self._timed("all_gather", bus):
                self.comm.all_gather_cast(group, x, buf, shard_elems=x.numel(), lane=self.bg.LANE_ACT, dst_dtype=x.dtype)
            return out
        cur = torch.cuda.current_stream()
        self.comm_stream.wait_stream(cur)
        with torch.cuda.stream(self.comm_stream):
            with self._timed("all_gather", bus, self.comm_stream):
                self.comm.all_gather_cast(group, x, buf, shard_elems=x.numel(), lane=self.bg.LANE_PUSH, dst_dtype=x.dtype)
            ev = torch.cuda.Event()
            ev.record(self.comm_stream)
        x.record_stream(self.comm_stream)
        return out, ev

    def reduce_scatter_first_dim(self, x, group):
        """[n*s, ...] -> [s, ...] sum (mappings_group.py:105-122 _reduce_scatter_along_first_dim)."""
        if group is None or group.size == 1:
            return x
        x = x.contiguous()
        n = group.size
        assert x.shape[0] % n == 0, "First dimension of the tensor should be divisible by tensor parallel size"
        buf, off = self._stage(x, group)
        out = torch.empty((x.shape[0] // n,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        self._check_vec(x, out.numel())
        with self._timed("reduce_scatter", (n - 1) / n * x.numel() * x.element_size()):
            self.comm.reduce_scatter_acc(group, buf, x.dtype, out, shard_elems=out.numel(), lane=self.bg.LANE_ACT, src_byte_offset=off)
        return out

    def all_gather_last_dim(self, x, group):
        """mappings_group.py:63-81 _gather_along_last_dim: gather then concatenate along the last dimension."""
        if group is None or group.size == 1:
            return x
        n = group.size
        g = self.all_gather_first_dim(x.contiguous().unsqueeze(0), group)  # [n, ...]
        return torch.cat([g[i] for i in range(n)], dim=-1).contiguous()

    def _check_vec(self, x, numel):
        if numel % _vec(x):
            raise self.bg.BgError("collective chunk of %d %s elements is not a multiple of 16 bytes" % (numel, x.dtype))

    def ulysses_all_to_all(self, tensors, group, to_heads):
        """Ulysses exchange of [b, s, n, d] tensors, all in ONE launch (transformer.py:1928-1987 + :2132-2145).
        to_heads=True : [b, s/p, n, d] -> [b, s, n/p, d]  (scatter heads, gather sequence; q/k/v before attention)
        to_heads=False: [b, s, n/p, d] -> [b, s/p, n, d]  (inverse; context after attention)"""
        p = group.size
        if p == 1:
            return list(tensors)
        descs, outs, off = [], [], 0
        for t in tensors:
            t = t.contiguous()
            b, s_in, n_in, d = t.shape
            buf, boff = self._stage(t, group, byte_offset=off)
            off = max(off, (boff + t.numel() * t.element_size() + 255) // 256 * 256)
            if to_heads:
                assert n_in % p == 0, "Number of heads (%d) must be divisible by the sequence parallel size (%d)!" % (n_in, p)
                hp = n_in // p
                out = torch.empty(b, s_in * p, hp, d, dtype=t.dtype, device=t.device)
                descs.append(dict(src=buf, src_byte_offset=boff, dst=out, batch=b, rows=s_in, row_elems=hp * d,
                                  src_bs=s_in * n_in * d, src_rs=n_in * d, src_me_off=hp * d,
                                  dst_bs=s_in * p * hp * d, dst_rs=hp * d, dst_peer_off=s_in * hp * d))
            else:
                assert s_in % p == 0
                sl = s_in // p
                out = torch.empty(b, sl, n_in * p, d, dtype=t.dtype, device=t.device)
                descs.append(dict(src=buf, src_byte_offset=boff, dst=out, batch=b, rows=sl, row_elems=n_in * d,
                                  src_bs=s_in * n_in * d, src_rs=n_in * d, src_me_off=sl * n_in * d,
                                  dst_bs=sl * n_in * p * d, dst_rs=n_in * p * d, dst_peer_off=n_in * d))
            outs.append(out)
        with self._timed("all_to_all", (p - 1) / p * sum(t.numel() * t.element_size() for t in tensors)):
            self.comm.all_to_all_rows(group, descs, tensors[0].dtype)
        return outs

    # ---- math ops --------------------------------------------------------------------------------------------
    @staticmethod
    def _mnk(a, b, layout):
        """-> (layout code, M, N, K) of A op B.  layout 'tn': a[M,K] b[N,K]; 'nn': a[M,K] b[K,N]; 'nt': a[K,M] b[K,N]."""
        code = {"tn": 0, "nn": 1, "nt": 2}[layout]
        if code == 2:
            k_, m_ = a.shape
        else:
            m_, k_ = a.shape
        return code, m_, (b.shape[0] if code == 0 else b.shape[1]), k_

    def gemm(self, a, b, layout, out=None, accumulate=False, addend=None):
        """bf16 GEMM on wgmma (layouts: ``_mnk``).
        ``addend`` [M,N]: out = A op B + addend in the epilogue (the residual add behind a projection, one rounding)."""
        code, m_, n_, k_ = self._mnk(a, b, layout)
        if out is None:
            out = torch.empty(m_, n_, dtype=torch.bfloat16, device=a.device)
        if a.dtype != torch.bfloat16 or b.dtype != torch.bfloat16 or out.dtype != torch.bfloat16:
            raise self.bg.BgError("the GEMM path is bf16-only (mixed_precision must be bf16)")
        assert a.is_contiguous() and b.is_contiguous() and out.is_contiguous()
        if m_ % 8 or n_ % 8 or k_ % 8:
            raise self.bg.BgError("GEMM dims (%d,%d,%d) must be multiples of 8" % (m_, n_, k_))
        if addend is not None:
            assert not accumulate and addend.dtype == torch.bfloat16 and addend.is_contiguous() and addend.numel() == m_ * n_
            launch = lambda: self.bg.gemm_bf16_add(a, b, out, addend, m_, n_, k_, code)  # noqa: E731
        else:
            launch = lambda: self.bg.gemm_bf16(a, b, out, m_, n_, k_, code, accumulate=accumulate)  # noqa: E731
        if self.gemm_profile is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            launch()
            e1.record()
            extra = 2 if (accumulate or addend is not None) else 1
            self.gemm_profile.append((e0, e1, 2.0 * m_ * n_ * k_, 2.0 * (m_ * k_ + k_ * n_ + m_ * n_ * extra)))
        else:
            launch()
        return out

    # ---- GEMM + collective: one fused operation where ``fusion_allowed`` says so, else the GEMM into the group's staging buffer
    # followed by the stand-alone collective ------------------------------------------------------------------------------------------
    def fuses(self, kind, m, n, k, group):
        """Would the fused ``kind`` ("gemm_rs", "gemm_ar", "ag_gemm") run for the [m, n] = [m, k] x [k, n] GEMM over ``group``?
        The on/off switches are read when the backend is built, "force" at every call."""
        p = 1 if group is None else group.size
        buf, data_bytes = self._bufs.get("staging", group) if p > 1 else (None, 0)
        return fusion_allowed(kind, m, n, k, p, None if buf is None else data_bytes, self.fuse[kind],
                              os.environ.get(FUSE_ENV[kind]) == "force")

    def gemm_reduce_scatter(self, a, b, layout, group):
        """[M, N] = A op B, reduce-scattered along M over ``group`` -> [M/p, N].  Fused: the wgmma GEMM's epilogue stores each
        partial tile into the owning rank's HBM and a tile reducer sums them as they land (GEMM + C8 in one operation)."""
        code, m_, n_, k_ = self._mnk(a, b, layout)
        if not self.fuses("gemm_rs", m_, n_, k_, group):
            staged, _ = self.staging_tensor(group, (m_, n_), a.dtype)
            self.gemm(a, b, layout, out=staged)
            return self.reduce_scatter_first_dim(staged, group)
        buf = self.staging(group, m_ * n_ * 2)
        out = torch.empty(m_ // group.size, n_, dtype=torch.bfloat16, device=a.device)
        with self._timed("gemm_reduce_scatter", (group.size - 1) / group.size * m_ * n_ * 2, flops=2.0 * m_ * n_ * k_):
            self.comm.gemm_reduce_scatter(group, a, b, m_, n_, k_, code, buf, buf.layout.partials, buf.layout.scatter_counters, out)
        self._count("gemm_rs")
        return out

    def gemm_all_reduce(self, a, b, layout, group):
        """[M, N] = sum over ``group`` of A op B, on every member.  Fused (GEMM + C5/C6 in one operation): partial tiles go to
        their owner's HBM, the owner's tile reducer sums them as they land and broadcasts the rows into every member's result."""
        code, m_, n_, k_ = self._mnk(a, b, layout)
        if not self.fuses("gemm_ar", m_, n_, k_, group):
            staged, _ = self.staging_tensor(group, (m_, n_), a.dtype)
            self.gemm(a, b, layout, out=staged)
            return self.all_reduce(staged, group)
        buf = self.staging(group, m_ * n_ * 2)
        lay = buf.layout
        with self._timed("gemm_all_reduce", 2.0 * (group.size - 1) / group.size * m_ * n_ * 2, flops=2.0 * m_ * n_ * k_):
            self.comm.gemm_all_reduce(group, a, b, m_, n_, k_, code, buf, lay.partials, lay.scatter_counters, lay.result)
        self._count("gemm_ar")
        # the symmetric result buffer is rewritten by the next fused all-reduce of this group: hand out a private copy
        return buf.u8[lay.result: lay.result + m_ * n_ * 2].view(torch.bfloat16).view(m_, n_).clone()

    def all_gather_gemm(self, a_local, b, layout, group):
        """out[M, N] = gather_rows(a_local[M/p, K]) op B, layout 'tn' or 'nn'.  Returns (out, gathered A): on both paths the
        gathered operand sits complete in region 0 of the group's staging buffer afterwards (the wgrad GEMM of the same layer reads
        it there).  Fused (C7 + GEMM in one operation): the GEMM consumes the gathered blocks as they land."""
        assert layout != "nt", "all_gather_gemm gathers the rows of A[M, K]"
        p = group.size
        code, ml, n_, k_ = self._mnk(a_local, b, layout)
        m_ = ml * p
        if not self.fuses("ag_gemm", m_, n_, k_, group):
            gathered = self.all_gather_into_staging(a_local, group)
            return self.gemm(gathered, b, layout), gathered
        buf = self.staging(group, m_ * k_ * 2)
        out = torch.empty(m_, n_, dtype=torch.bfloat16, device=a_local.device)
        with self._timed("all_gather_gemm", (p - 1) / p * m_ * k_ * 2, flops=2.0 * m_ * n_ * k_):
            self.comm.all_gather_gemm(group, a_local, b, out, m_, n_, k_, code, buf, 0, buf.layout.gather_counters, self.comm_stream)
        a_local.record_stream(self.comm_stream)
        self._count("ag_gemm")
        return out, buf.u8[: m_ * k_ * 2].view(torch.bfloat16).view(m_, k_)

    def rmsnorm_fwd(self, x, weight, eps):
        x2 = x.reshape(-1, x.shape[-1])
        y = torch.empty_like(x2)
        rstd = torch.empty(x2.shape[0], dtype=torch.float32, device=x.device)
        L = self.bg.lib()
        self.bg.check(L.bg_rmsnorm_fwd(_p(x2), _p(weight), _p(y), _p(rstd), x2.shape[0], x2.shape[1], float(eps), _s()))
        return y.view_as(x), rstd

    def rmsnorm_bwd(self, dy, x, weight, rstd):
        x2, dy2 = x.reshape(-1, x.shape[-1]), dy.reshape(-1, x.shape[-1])
        dx = torch.empty_like(x2)
        npart = min(self.norm_partials, max(1, x2.shape[0]))
        dwp = torch.empty(npart, x2.shape[1], dtype=torch.float32, device=x.device)
        L = self.bg.lib()
        self.bg.check(L.bg_rmsnorm_bwd(_p(dy2), _p(x2), _p(weight), _p(rstd), _p(dx), _p(dwp), x2.shape[0], x2.shape[1], npart, _s()))
        return dx.view_as(x), dwp.sum(0).to(weight.dtype)

    def layernorm_fwd(self, x, weight, bias, eps):
        """LayerNorm with bias (GPT / BERT families): -> (y, mean[rows], rstd[rows]) fp32 statistics."""
        x2 = x.reshape(-1, x.shape[-1])
        y = torch.empty_like(x2)
        mean = torch.empty(x2.shape[0], dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        self.bg.check(self.bg.lib().bg_layernorm_fwd(_p(x2), _p(weight), _p(bias), _p(y), _p(mean), _p(rstd), x2.shape[0], x2.shape[1],
                                                     float(eps), _s()))
        return y.view_as(x), mean, rstd

    def layernorm_bwd(self, dy, x, weight, mean, rstd):
        x2, dy2 = x.reshape(-1, x.shape[-1]), dy.reshape(-1, x.shape[-1])
        dx = torch.empty_like(x2)
        npart = min(self.norm_partials, max(1, x2.shape[0]))       # partial-sum rows (one per CTA; summed below)
        dwp = torch.empty(npart, x2.shape[1], dtype=torch.float32, device=x.device)
        dbp = torch.empty_like(dwp)
        self.bg.check(self.bg.lib().bg_layernorm_bwd(_p(dy2), _p(x2), _p(weight), _p(mean), _p(rstd), _p(dx), _p(dwp), _p(dbp),
                                                     x2.shape[0], x2.shape[1], npart, _s()))
        return dx.view_as(x), dwp.sum(0).to(weight.dtype), dbp.sum(0).to(weight.dtype)

    def bias_gelu_fwd(self, x, bias, tanh_form=True):
        x2 = x.reshape(-1, x.shape[-1])
        y = torch.empty_like(x2)
        self.bg.check(self.bg.lib().bg_bias_gelu(_p(x2), _p(bias) if bias is not None else None, None, _p(y), x2.shape[0], x2.shape[1],
                                                 1 if tanh_form else 0, _s()))
        return y.view_as(x)

    def bias_gelu_bwd(self, dy, x, bias, tanh_form=True):
        x2, dy2 = x.reshape(-1, x.shape[-1]), dy.reshape(-1, x.shape[-1])
        dx = torch.empty_like(x2)
        self.bg.check(self.bg.lib().bg_bias_gelu(_p(x2), _p(bias) if bias is not None else None, _p(dy2), _p(dx), x2.shape[0], x2.shape[1],
                                                 1 if tanh_form else 0, _s()))
        return dx.view_as(x)

    def bias_tanh_fwd(self, x, bias):
        x2 = x.reshape(-1, x.shape[-1])
        y = torch.empty_like(x2)
        self.bg.check(self.bg.lib().bg_bias_tanh(_p(x2), _p(bias) if bias is not None else None, None, _p(y), x2.shape[0], x2.shape[1], _s()))
        return y.view_as(x)

    def bias_tanh_bwd(self, dy, x, bias):
        x2, dy2 = x.reshape(-1, x.shape[-1]), dy.reshape(-1, x.shape[-1])
        dx = torch.empty_like(x2)
        self.bg.check(self.bg.lib().bg_bias_tanh(_p(x2), _p(bias) if bias is not None else None, _p(dy2), _p(dx), x2.shape[0], x2.shape[1],
                                                 _s()))
        return dx.view_as(x)

    def vit_patchify(self, pixels, patch, rows_pad):
        """pixels [B, C, H, W] (fp32 / bf16) -> bf16 patch rows [rows_pad, p*p*C] in (p1 p2 c) order, rows past B*P zero."""
        b, c, hgt, wid = pixels.shape
        pixels = pixels.contiguous()
        out = torch.empty(rows_pad, patch * patch * c, dtype=torch.bfloat16, device=pixels.device)
        self.bg.check(self.bg.lib().bg_vit_patchify(_p(pixels), self.bg.dtype_code(pixels.dtype), _p(out), b, c, hgt, wid, patch, rows_pad,
                                                    _s()))
        return out

    def vit_embed_fwd(self, patch_out, bias, cls, pos, batch, s_run, p, seed, iteration, site, sample_base):
        """-> y [s_run, batch, h]: cls + pos[0], then patch_out rows + bias + pos[1..P], then zero rows (dropout fused when p > 0)."""
        n_patches, h = pos.shape[0] - 1, pos.shape[1]
        y = torch.empty(s_run, batch, h, dtype=torch.bfloat16, device=patch_out.device)
        self.bg.check(self.bg.lib().bg_vit_embed_fwd(_p(patch_out), _p(bias), _p(cls), _p(pos), _p(y), batch, n_patches, s_run, h,
                                                     int(sample_base), float(p), int(seed), int(iteration), int(site), _s()))
        return y

    def vit_embed_bwd(self, dy, n_patches, rows_pad, p, seed, iteration, site, sample_base):
        """-> (dpatch [rows_pad, h] bf16, dcls [h] fp32, dpos [P + 1, h] fp32, dbias [h] fp32) from dy [s_run, batch, h]."""
        s_run, batch, h = dy.shape
        dy = dy.contiguous()
        dpatch = torch.empty(rows_pad, h, dtype=torch.bfloat16, device=dy.device)
        dpos = torch.empty(n_patches + 1, h, dtype=torch.float32, device=dy.device)
        npart = min(self.norm_partials, n_patches)
        dbp = torch.empty(npart, h, dtype=torch.float32, device=dy.device)
        self.bg.check(self.bg.lib().bg_vit_embed_bwd(_p(dy), _p(dpatch), _p(dpos), _p(dbp), npart, batch, n_patches, s_run, rows_pad, h,
                                                     int(sample_base), float(p), int(seed), int(iteration), int(site), _s()))
        return dpatch, dpos[0], dpos, dbp.sum(0)

    # ---- Swin: window relayouts through a token map (map[w * L + i] = token at position i of window w, inv its inverse; int32 on
    # the device), patch merging + LayerNorm, mean-pool and per-sample drop path (include/bg_galvatron.h)
    def swin_window_qkv_fwd(self, mixed, bias, tmap, inv, n_windows, mb, heads, hn):
        """mixed [T_run * mb, heads * 3 * hn] SBH rows + bias -> q, k, v [mb * n_windows, L, heads, hn]."""
        L = tmap.numel() // n_windows
        q, k, v = [torch.empty(mb * n_windows, L, heads, hn, dtype=mixed.dtype, device=mixed.device) for _ in range(3)]
        self.bg.check(self.bg.lib().bg_swin_window_qkv_fwd(_p(mixed), _p(bias), _p(tmap), _p(q), _p(k), _p(v), mb, tmap.numel(),
                                                           mixed.numel() // (mb * heads * 3 * hn), n_windows, L, heads, hn, _s()))
        return q, k, v

    def swin_window_qkv_bwd(self, dq, dk, dv, tmap, inv, n_windows, mb, t_run):
        """-> (dmixed [t_run * mb, heads * 3 * hn] with zero padding-token rows, dbias [heads * 3 * hn] fp32)."""
        heads, hn = dq.shape[2], dq.shape[3]
        dmixed = torch.empty(t_run * mb, heads * 3 * hn, dtype=dq.dtype, device=dq.device)
        npart = min(self.norm_partials, t_run * mb)
        dbp = torch.empty(npart, heads * 3 * hn, dtype=torch.float32, device=dq.device)
        self.bg.check(self.bg.lib().bg_swin_window_qkv_bwd(_p(dq.contiguous()), _p(dk.contiguous()), _p(dv.contiguous()), _p(dmixed), _p(dbp),
                                                           npart, _p(inv), mb, tmap.numel(), t_run, n_windows, tmap.numel() // n_windows,
                                                           heads, hn, _s()))
        return dmixed, dbp.sum(0)

    def swin_rel_bias_fwd(self, table, index, shift_mask, mb, n_windows, window):
        """table [(2w-1)^2, heads] (bf16 / fp32), index int32 [L * L], shift_mask uint8 [n_windows, L, L] or None -> the additive bf16
        mask [mb * n_windows, heads, L, L]: a view of rows padded to a multiple of 8 columns, the stride the memory-efficient
        attention kernel takes without a copy."""
        L, heads = window * window, table.shape[1]
        ld = (L + 7) // 8 * 8
        out = torch.empty(mb * n_windows, heads, L, ld, dtype=torch.bfloat16, device=table.device)
        self.bg.check(self.bg.lib().bg_swin_rel_bias_fwd(_p(table), self.bg.dtype_code(table.dtype), _p(index),
                                                         _p(shift_mask) if shift_mask is not None else None, _p(out), mb, n_windows,
                                                         heads, window, L, ld, _s()))
        return out[..., :L]

    def swin_rel_bias_bwd(self, dbias, cells, offsets, n_windows, window):
        """dbias [mb * n_windows, heads, L, L] bf16 (rows may be padded) -> the table's gradient [(2w-1)^2, heads] fp32; cells / offsets
        list the cells of every table entry (WindowLayout.rel_maps)."""
        n, heads, L = dbias.shape[0], dbias.shape[1], dbias.shape[2]
        ld = dbias.stride(2)
        if dbias.stride(3) != 1 or ld % 8 or ld < L or dbias.stride(1) != L * ld or dbias.stride(0) != heads * L * ld:
            ld = (L + 7) // 8 * 8
            dbias = torch.nn.functional.pad(dbias, (0, ld - L))
        n_table = (2 * window - 1) ** 2
        npart = max(1, min(n, -(-self.norm_partials // heads)))
        part = torch.empty(npart, n_table, heads, dtype=torch.float32, device=dbias.device)
        self.bg.check(self.bg.lib().bg_swin_rel_bias_bwd(_p(dbias), _p(cells), _p(offsets), _p(part), npart, n // n_windows, n_windows,
                                                         heads, window, L, ld, _s()))
        return part.sum(0)

    # ---- T5 cross-attention: the query / key_value projections' outputs <-> the attention layout (include/bg_galvatron.h)
    def cross_attn_qkv_fwd(self, q_mixed, q_bias, kv_mixed, kv_bias, heads, hn):
        """q_mixed [s_q, b, heads * hn] + q_bias, kv_mixed [s_k, b, heads * 2 * hn] (per head k | v) + kv_bias -> q [b, s_q, heads, hn],
        k, v [b, s_k, heads, hn]."""
        s_q, b, s_k = q_mixed.shape[0], q_mixed.shape[1], kv_mixed.shape[0]
        q = torch.empty(b, s_q, heads, hn, dtype=q_mixed.dtype, device=q_mixed.device)
        k, v = [torch.empty(b, s_k, heads, hn, dtype=q_mixed.dtype, device=q_mixed.device) for _ in range(2)]
        self.bg.check(self.bg.lib().bg_cross_attn_qkv_fwd(_p(q_mixed.contiguous()), _p(q_bias) if q_bias is not None else None,
                                                          _p(kv_mixed.contiguous()), _p(kv_bias) if kv_bias is not None else None, _p(q),
                                                          _p(k), _p(v), s_q, s_k, b, heads, hn, _s()))
        return q, k, v

    def cross_attn_qkv_bwd(self, dq, dk, dv):
        """-> (dq_mixed [s_q, b, heads * hn], dkv_mixed [s_k, b, heads * 2 * hn], dq_bias, dkv_bias fp32)."""
        b, s_q, heads, hn = dq.shape
        s_k = dk.shape[1]
        dqm = torch.empty(s_q, b, heads * hn, dtype=dq.dtype, device=dq.device)
        dkvm = torch.empty(s_k, b, heads * 2 * hn, dtype=dq.dtype, device=dq.device)
        npart = min(self.norm_partials, max(s_q, s_k) * b)
        dbp = torch.empty(npart, heads * 3 * hn, dtype=torch.float32, device=dq.device)
        self.bg.check(self.bg.lib().bg_cross_attn_qkv_bwd(_p(dq.contiguous()), _p(dk.contiguous()), _p(dv.contiguous()), _p(dqm), _p(dkvm),
                                                          _p(dbp), npart, s_q, s_k, b, heads, hn, _s()))
        db = dbp.sum(0)
        return dqm, dkvm, db[:heads * hn], db[heads * hn:]

    def swin_window_merge_fwd(self, windows, tmap, inv, n_windows, mb, t_run):
        """attention output [mb * n_windows, L, heads, hn] -> SBH rows [t_run, mb, heads * hn], padding-token rows zero."""
        windows = windows.contiguous()
        cols = windows.shape[2] * windows.shape[3]
        rows = torch.empty(t_run, mb, cols, dtype=windows.dtype, device=windows.device)
        self.bg.check(self.bg.lib().bg_swin_window_merge_fwd(_p(windows), _p(rows), _p(tmap), _p(inv), mb, tmap.numel(), t_run, n_windows,
                                                             tmap.numel() // n_windows, cols, _s()))
        return rows

    def swin_window_merge_bwd(self, drows, tmap, inv, n_windows, mb, heads, hn):
        drows = drows.contiguous()
        L = tmap.numel() // n_windows
        dwin = torch.empty(mb * n_windows, L, heads, hn, dtype=drows.dtype, device=drows.device)
        self.bg.check(self.bg.lib().bg_swin_window_merge_bwd(_p(drows), _p(dwin), _p(tmap), _p(inv), mb, tmap.numel(),
                                                             drows.numel() // (mb * heads * hn), n_windows, L, heads * hn, _s()))
        return dwin

    def swin_merge_ln_fwd(self, x, add_bias, weight, bias, eps, mb, height, width, r, in_bsh, t_out_run):
        """x: the height x width grid of mb samples (SBH rows, or with ``in_bsh`` the patch GEMM's (sample, patch) rows), C columns ->
        (y [t_out_run, mb, r * r * C] with zero padding-token rows, mean, rstd)."""
        x = x.contiguous()
        c = x.shape[-1]
        y = torch.empty(t_out_run, mb, r * r * c, dtype=x.dtype, device=x.device)
        mean = torch.empty(t_out_run * mb, dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        self.bg.check(self.bg.lib().bg_swin_merge_ln_fwd(_p(x), _p(add_bias) if add_bias is not None else None, _p(weight), _p(bias), _p(y),
                                                         _p(mean), _p(rstd), mb, height, width, r, 1 if in_bsh else 0, x.numel() // c, c,
                                                         t_out_run, float(eps), _s()))
        return y, mean, rstd

    def swin_merge_ln_bwd(self, dy, x, add_bias, weight, mean, rstd, mb, height, width, r, in_bsh):
        """-> (dx in x's layout, zero past the real rows; dweight, dbias of the norm; d(add_bias) fp32 or None)."""
        x, dy = x.contiguous(), dy.contiguous()
        c = x.shape[-1]
        dx = torch.empty_like(x)
        npart = min(self.norm_partials, max(1, mb * (height // r) * (width // r)))
        dwp = torch.empty(npart, r * r * c, dtype=torch.float32, device=x.device)
        dbp = torch.empty_like(dwp)
        dap = torch.empty_like(dwp) if add_bias is not None else None
        self.bg.check(self.bg.lib().bg_swin_merge_ln_bwd(_p(dy), _p(x), _p(add_bias) if add_bias is not None else None, _p(weight), _p(mean),
                                                         _p(rstd), _p(dx), _p(dwp), _p(dbp), _p(dap) if dap is not None else None, npart, mb,
                                                         height, width, r, 1 if in_bsh else 0, x.numel() // c, c, _s()))
        return dx, dwp.sum(0).to(weight.dtype), dbp.sum(0).to(weight.dtype), (dap.sum(0) if dap is not None else None)

    def swin_mean_pool_fwd(self, x, tokens, rows_out):
        """x [t_run, mb, C] -> [rows_out, C]: the mean of the first ``tokens`` tokens of each sample, zero rows past mb."""
        x = x.contiguous()
        t_run, mb, c = x.shape
        y = torch.empty(rows_out, c, dtype=x.dtype, device=x.device)
        self.bg.check(self.bg.lib().bg_swin_mean_pool_fwd(_p(x), _p(y), tokens, t_run, mb, rows_out, c, _s()))
        return y

    def swin_mean_pool_bwd(self, dy, tokens, t_run, mb):
        dy = dy.contiguous()
        dx = torch.empty(t_run, mb, dy.shape[-1], dtype=dy.dtype, device=dy.device)
        self.bg.check(self.bg.lib().bg_swin_mean_pool_bwd(_p(dy), _p(dx), tokens, t_run, mb, dy.shape[-1], _s()))
        return dx

    def drop_path_add_fwd(self, x, bias, residual, p, seed, iteration, site, sample_base):
        """y = residual + keep_b * scale * (x + bias) on an SBH tensor x [s, b, h] of samples sample_base..; bias [h] bf16 / fp32."""
        s, b, h = x.shape
        x, residual = x.contiguous(), residual.contiguous()
        y = torch.empty_like(x)
        bcode = self.bg.dtype_code(bias.dtype) if bias is not None else 0
        self.bg.check(self.bg.lib().bg_drop_path_add_fwd(_p(x), _p(bias) if bias is not None else None, bcode, _p(residual), _p(y), s * b, h,
                                                         b, int(sample_base), float(p), int(seed), int(iteration), int(site), _s()))
        return y

    def drop_path_add_bwd(self, dy, p, seed, iteration, site, sample_base, with_bias):
        """-> (dx = keep_b * scale * dy, its fp32 column sums or None)."""
        s, b, h = dy.shape
        dy = dy.contiguous()
        dx = torch.empty_like(dy)
        npart = min(self.norm_partials, max(1, s * b))
        dbp = torch.empty(npart, h, dtype=torch.float32, device=dy.device) if with_bias else None
        self.bg.check(self.bg.lib().bg_drop_path_add_bwd(_p(dy), _p(dx), _p(dbp) if dbp is not None else None, npart, s * b, h, b,
                                                         int(sample_base), float(p), int(seed), int(iteration), int(site), _s()))
        return dx, (dbp.sum(0) if dbp is not None else None)

    def dropout_add_fwd(self, x, bias, residual, p, seed, iteration, site, seq_base, sample_base):
        """y = residual + keep * scale * (x + bias) on an SBH tensor x [s_loc, b_loc, h] whose rows are tokens seq_base.. of samples
        sample_base.. (mask: include/bg_galvatron.h).  bias [h] (bf16 / fp32) and residual (x's shape) may be None."""
        s, b, h = x.shape
        x = x.contiguous()
        y = torch.empty_like(x)
        if residual is not None:
            residual = residual.contiguous()
            assert residual.shape == x.shape and residual.dtype == x.dtype
        bcode = self.bg.dtype_code(bias.dtype) if bias is not None else 0
        self.bg.check(self.bg.lib().bg_dropout_add_fwd(_p(x), _p(bias) if bias is not None else None, bcode,
                                                       _p(residual) if residual is not None else None, _p(y), s * b, h, b,
                                                       int(seq_base), int(sample_base), float(p), int(seed), int(iteration),
                                                       int(site), _s()))
        return y

    def dropout_bwd(self, dy, p, seed, iteration, site, seq_base, sample_base, with_bias):
        """-> (dx = keep * scale * dy, dbias = its fp32 column sums or None), the mask regenerated from the same coordinates."""
        s, b, h = dy.shape
        dy = dy.contiguous()
        dx = torch.empty_like(dy)
        npart = min(self.norm_partials, max(1, s * b))
        dbp = torch.empty(npart, h, dtype=torch.float32, device=dy.device) if with_bias else None
        self.bg.check(self.bg.lib().bg_dropout_bwd(_p(dy), _p(dx), _p(dbp) if dbp is not None else None, npart, s * b, h, b,
                                                   int(seq_base), int(sample_base), float(p), int(seed), int(iteration), int(site),
                                                   _s()))
        return dx, (dbp.sum(0) if dbp is not None else None)

    @staticmethod
    def _check_sample_ids(ids, b, x):
        assert ids.dtype == torch.int32 and ids.shape == (b,) and ids.is_contiguous() and ids.device == x.device, \
            "sample_ids must be a contiguous int32 [%d] tensor on %s" % (b, x.device)

    def dropout_add_fwd_ids(self, x, bias, residual, p, seed, iteration, site, seq_base, sample_ids):
        """``dropout_add_fwd`` with row r of x [s_loc, b_loc, h] at sample ``sample_ids[r % b_loc]`` (int32 [b_loc] on x's device, read
        as uint32): the samples a relocation gathered from several data-parallel ranks."""
        s, b, h = x.shape
        self._check_sample_ids(sample_ids, b, x)
        x = x.contiguous()
        y = torch.empty_like(x)
        if residual is not None:
            residual = residual.contiguous()
            assert residual.shape == x.shape and residual.dtype == x.dtype
        bcode = self.bg.dtype_code(bias.dtype) if bias is not None else 0
        self.bg.check(self.bg.lib().bg_dropout_add_fwd_ids(_p(x), _p(bias) if bias is not None else None, bcode,
                                                           _p(residual) if residual is not None else None, _p(y), s * b, h, b,
                                                           int(seq_base), _p(sample_ids), float(p), int(seed), int(iteration),
                                                           int(site), _s()))
        return y

    def dropout_bwd_ids(self, dy, p, seed, iteration, site, seq_base, sample_ids, with_bias):
        """``dropout_bwd`` at the sample map of ``dropout_add_fwd_ids``."""
        s, b, h = dy.shape
        self._check_sample_ids(sample_ids, b, dy)
        dy = dy.contiguous()
        dx = torch.empty_like(dy)
        npart = min(self.norm_partials, max(1, s * b))
        dbp = torch.empty(npart, h, dtype=torch.float32, device=dy.device) if with_bias else None
        self.bg.check(self.bg.lib().bg_dropout_bwd_ids(_p(dy), _p(dx), _p(dbp) if dbp is not None else None, npart, s * b, h, b,
                                                       int(seq_base), _p(sample_ids), float(p), int(seed), int(iteration), int(site),
                                                       _s()))
        return dx, (dbp.sum(0) if dbp is not None else None)

    def swiglu_fwd(self, gate_up):
        rows, two_f = gate_up.reshape(-1, gate_up.shape[-1]).shape
        y = torch.empty(gate_up.shape[:-1] + (two_f // 2,), dtype=gate_up.dtype, device=gate_up.device)
        self.bg.check(self.bg.lib().bg_swiglu_fwd(_p(gate_up), _p(y), rows, two_f // 2, _s()))
        return y

    def swiglu_bwd(self, dy, gate_up):
        rows, two_f = gate_up.reshape(-1, gate_up.shape[-1]).shape
        dgu = torch.empty_like(gate_up)
        self.bg.check(self.bg.lib().bg_swiglu_bwd(_p(dy), _p(gate_up), _p(dgu), rows, two_f // 2, _s()))
        return dgu

    def qkv_rope_fwd(self, mixed, cos, sin, ng, r, hn, stage_group=None):
        """mixed [s,b,ng*(r+2)*hn] -> q [b,s,ng*r,hn], k,v [b,s,ng,hn] (rotated).  With ``stage_group`` the
        outputs are written straight into that group's staging buffer (Ulysses source, no extra copy)."""
        s, b = mixed.shape[0], mixed.shape[1]
        shapes = [(b, s, ng * r, hn), (b, s, ng, hn), (b, s, ng, hn)]
        if stage_group is not None and stage_group.size > 1:
            outs, off = [], 0
            for sh in shapes:
                t, _ = self.staging_tensor(stage_group, sh, mixed.dtype, byte_offset=off)
                outs.append(t)
                off = (off + t.numel() * t.element_size() + 255) // 256 * 256
            q, k, v = outs
        else:
            q, k, v = [torch.empty(sh, dtype=mixed.dtype, device=mixed.device) for sh in shapes]
        self.bg.check(self.bg.lib().bg_qkv_rope(_p(mixed), _p(q), _p(k), _p(v), _p(cos), _p(sin), s, b, ng, r, hn, 0, _s()))
        return q, k, v

    def qkv_rope_bwd(self, dq, dk, dv, cos, sin, ng, r, hn):
        b, s = dq.shape[0], dq.shape[1]
        dmixed = torch.empty(s, b, ng * (r + 2) * hn, dtype=dq.dtype, device=dq.device)
        self.bg.check(self.bg.lib().bg_qkv_rope(_p(dmixed), _p(dq.contiguous()), _p(dk.contiguous()), _p(dv.contiguous()),
                                                _p(cos), _p(sin), s, b, ng, r, hn, 1, _s()))
        return dmixed

    def rope_tables(self, seq_len, head_dim, base, offset, dtype, device):
        inv_freq = 1.0 / (base ** (torch.arange(0, head_dim, 2, dtype=torch.float32, device=device) / head_dim))
        pos = torch.arange(seq_len, dtype=torch.float32, device=device) + offset
        freqs = torch.outer(pos, inv_freq)
        # the reference casts cos/sin to the activation dtype before applying them (apply_rotary_pos_emb)
        return torch.cos(freqs).to(dtype).float().contiguous(), torch.sin(freqs).to(dtype).float().contiguous()

    def attention(self, q, k, v, causal, softmax_scale, key_mask=None, dropout_p=0.0, window_mask=None, window_bias=None):
        """Attention is a LIBRARY call, as in the reference (transformer.py:495 calls flash-attn; K3 is not a collective and
        is outside the hot-path scope).  The default is cuDNN's fused SDPA, reached
        through torch SDPA; HGB_ATTN=flash selects flash-attn 2.  q [b,s,n,d], k/v [b,s,ng,d] (GQA un-expanded).  Differentiable.
        ``dropout_p`` > 0: dropout on the attention probabilities (transformer.py:443-503), drawn from torch's CUDA generator (the
        caller runs this under the model-parallel RNG tracker); SDPA may then pick the flash or memory-efficient kernel instead of
        cuDNN's.  ``window_mask`` / ``window_bias``: Swin's additive shift mask, or its learned relative-position bias (differentiable).
        """
        import torch.nn.functional as F
        from torch.nn.attention import SDPBackend, sdpa_kernel
        if window_mask is not None or window_bias is not None:
            # Swin's shifted windows: an additive [windows, 1, L, L] mask (0 / -inf, q's dtype), one row of windows per sample; or
            # the relative-position bias [windows, heads, L, L] (shift mask included), which needs its gradient: cuDNN's backward
            # returns only dq, dk and dv, the memory-efficient kernel's also the bias gradient, so the bias pins that kernel (also
            # where no gradient is taken, so that a checkpointed block's recompute runs the forward's kernel)
            assert not causal and key_mask is None and dropout_p == 0.0
            backends = [SDPBackend.EFFICIENT_ATTENTION] if window_bias is not None else \
                [SDPBackend.CUDNN_ATTENTION, SDPBackend.EFFICIENT_ATTENTION, SDPBackend.MATH]
            with sdpa_kernel(backends):
                o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
                                                   attn_mask=window_bias if window_bias is not None else window_mask, scale=softmax_scale)
            return o.transpose(1, 2)
        if key_mask is not None:
            # BERT's padding mask (bert_hf/BertModel_sequential.py: get_extended_attention_mask): key j of sample b is visible iff
            # key_mask[b, j]; fused SDPA with an additive mask (cuDNN where it accepts the mask, the memory-efficient kernel else)
            assert not causal
            bias = torch.zeros(key_mask.shape[0], 1, 1, key_mask.shape[1], dtype=q.dtype, device=q.device)
            bias.masked_fill_(~key_mask.bool()[:, None, None, :], float("-inf"))
            with sdpa_kernel([SDPBackend.CUDNN_ATTENTION, SDPBackend.EFFICIENT_ATTENTION, SDPBackend.MATH]):
                o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), attn_mask=bias,
                                                   dropout_p=dropout_p, scale=softmax_scale, enable_gqa=k.shape[2] != q.shape[2])
            return o.transpose(1, 2)
        if self.attn_impl != "cudnn":
            return None
        backends = [SDPBackend.CUDNN_ATTENTION]
        if dropout_p > 0.0:
            backends += [SDPBackend.FLASH_ATTENTION, SDPBackend.EFFICIENT_ATTENTION]
        with sdpa_kernel(backends):
            o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=causal,
                                               dropout_p=dropout_p, scale=softmax_scale, enable_gqa=k.shape[2] != q.shape[2])
        return o.transpose(1, 2)

    def attention_prefix(self, q, k, v, softmax_scale):
        """Causal attention of a query block against a LONGER key/value prefix, diagonal aligned to the bottom-right corner
        (query i sees keys j <= i + sk - sq): one zigzag chunk of a context-parallel rank against everything before it.
        Library call, as all attention here: flash-attn 2 (its causal mask has exactly this alignment for sq != sk; torch's
        SDPA aligns top-left).  q [b,sq,n,d], k/v [b,sk,ng,d].  Differentiable."""
        from flash_attn import flash_attn_func
        return flash_attn_func(q, k, v, dropout_p=0.0, softmax_scale=softmax_scale, causal=True)

    def attention_fwd(self, q, k, v, causal, softmax_scale, key_mask=None, dropout_p=0.0):
        """flash-attn 2 library call (the reference's choice); used when HGB_ATTN=flash.  Its backward replays ``rng``."""
        from flash_attn.flash_attn_interface import _flash_attn_forward
        assert key_mask is None, "the flash-attn path takes no padding mask"
        out, lse, _, rng = _flash_attn_forward(q, k, v, dropout_p, softmax_scale, causal=causal, window_size_left=-1,
                                               window_size_right=-1, softcap=0.0, alibi_slopes=None, return_softmax=False)
        return out, lse, rng

    def attention_bwd(self, dout, q, k, v, out, lse, causal, softmax_scale, rng, dropout_p=0.0):
        from flash_attn.flash_attn_interface import _flash_attn_backward
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        _flash_attn_backward(dout.contiguous(), q, k, v, out, lse, dq, dk, dv, dropout_p, softmax_scale, causal, -1, -1, 0.0, None,
                             False, rng_state=rng)
        return dq, dk, dv

    def ce_fwd(self, logits2d, target, vocab_start, tp_group):
        """vocab-parallel CE forward on [rows, V/t]: returns (loss[rows] fp32, rowmax, sum2) -- cross_entropy.py:14-100."""
        L, rows, vl = self.bg.lib(), logits2d.shape[0], logits2d.shape[1]
        code = self.bg.dtype_code(logits2d.dtype)
        rowmax = torch.empty(rows, dtype=torch.float32, device=logits2d.device)
        self.bg.check(L.bg_ce_rowmax(_p(logits2d), code, _p(rowmax), rows, vl, _s()))
        rowmax = self.all_reduce(rowmax, tp_group, op="max")
        out2 = torch.empty(rows, 2, dtype=torch.float32, device=logits2d.device)
        self.bg.check(L.bg_ce_sumexp(_p(logits2d), code, _p(target), _p(rowmax), _p(out2), rows, vl, int(vocab_start), _s()))
        out2 = self.all_reduce(out2, tp_group)
        loss = torch.log(out2[:, 0]) - out2[:, 1]
        return loss, rowmax, out2

    def ce_bwd(self, logits2d, target, rowmax, sum2, grad_loss, vocab_start):
        """in place: logits <- dlogits (cross_entropy.py:103-152)."""
        L, rows, vl = self.bg.lib(), logits2d.shape[0], logits2d.shape[1]
        self.bg.check(L.bg_ce_bwd(_p(logits2d), self.bg.dtype_code(logits2d.dtype), _p(target), _p(rowmax), _p(sum2),
                                  _p(grad_loss.contiguous()), rows, vl, int(vocab_start), _s()))
        return logits2d

    def cast(self, src, dst, scale=1.0, accumulate=False):
        self.bg.cast(src, dst, scale=scale, accumulate=accumulate)

    def launch_count(self):
        return self.bg.launch_count()


class _CpRing:
    """Peer-HBM transport of the context-parallel ring (include/bg_galvatron.h, C15): step i of a schedule holds the K/V block that
    arrived in slot parity i % 2 and pushes it on into the next member's slot (i + 1) % 2.  The K/V push runs on ``comm_stream``
    (when given), ordered after the work already queued, so it overlaps the step's attention; the accumulate-and-forward push
    depends on the step's gradients and runs in stream order.  A push into a parity waits for the receiver's release of it, except
    on the slot's very first use."""

    @staticmethod
    def slot_bytes(elems):
        return 2 * (2 * elems * 2 + 2 * elems * 4)

    def __init__(self, comm, group, buf, capacity, comm_stream=None, counts=None):
        from ... import _bg
        self.bg, self.comm, self.group, self.buf, self.capacity = _bg, comm, group, buf, int(capacity)
        self.size, self.rank = group.size, group.rank_in_group(comm.rank)
        self.comm_stream, self.counts = comm_stream, counts
        self._used = set()             # (kind, parity) pushed into at least once
        self._pushed = {}              # parity of the slot a K/V push read -> its completion event (comm_stream)
        self.shape = None

    def _kv_off(self, parity):
        return parity * 4 * self.capacity

    def _acc_off(self, parity):
        return 8 * self.capacity + parity * 8 * self.capacity

    def _first(self, kind, parity):
        first = (kind, parity) not in self._used
        self._used.add((kind, parity))
        return first

    def _count(self):
        if self.counts is not None:
            self.counts["cp_ring"] = self.counts.get("cp_ring", 0) + 1

    def _check(self, t):
        if t.numel() > self.capacity:
            raise self.bg.BgError("cp ring block of %d elements > the %d reserved" % (t.numel(), self.capacity))

    def send_kv(self, step, k, v):
        """push this step's K/V block to the next member, for its step + 1"""
        self._check(k)
        self.shape = tuple(k.shape)
        parity = (step + 1) % 2
        wait_free = not self._first(0, parity)
        slot = self.buf.sub(self._kv_off(parity))
        if self.comm_stream is None:
            self.comm.cp_ring_push(self.group, slot, parity, wait_free, k, v)
        else:
            cur = torch.cuda.current_stream()
            self.comm_stream.wait_stream(cur)
            self.comm.cp_ring_push(self.group, slot, parity, wait_free, k, v, stream=self.comm_stream)
            if step > 0:               # (step 0 pushes the rank's own block, not a slot)
                ev = torch.cuda.Event()
                ev.record(self.comm_stream)
                self._pushed[step % 2] = ev
            k.record_stream(self.comm_stream)
            v.record_stream(self.comm_stream)
        self._count()

    def recv_kv(self, step):
        """(k, v) of this step: views of the receive slot, valid until ``release_kv(step)``"""
        n = 1
        for d in self.shape:
            n *= d
        self.comm.cp_ring_wait(self.group, self.bg.RING_KV, step % 2, n)
        kv = self.buf.u8[self._kv_off(step % 2): self._kv_off(step % 2) + 4 * n].view(torch.bfloat16)
        return kv[:n].view(self.shape), kv[n:].view(self.shape)

    def release_kv(self, step):
        ev = self._pushed.pop(step % 2, None)
        if ev is not None:             # the push that forwarded this slot has read it
            torch.cuda.current_stream().wait_event(ev)
        n = 1
        for d in self.shape:
            n *= d
        self.comm.cp_ring_release(self.group, self.bg.RING_KV, step % 2, n)

    def send_acc(self, step, acc_in, dk, dv, c_row0, c_rows):
        """next member's [dK | dV] = acc_in (None at step 0) + this step's dk, dv (rows c_row0 .. of the block)"""
        b, s, ng, d = self.shape
        parity = (step + 1) % 2
        self.comm.cp_ring_acc_push(self.group, self.buf.sub(self._acc_off(parity)), parity, not self._first(1, parity), acc_in,
                                   dk.contiguous(), dv.contiguous(), b, s, ng * d, c_row0, c_rows)
        self._count()

    def recv_acc(self, step):
        """the fp32 [dK | dV] accumulators that arrived for this step (step = size: the finished sums, back at their owner)"""
        n = 1
        for d in self.shape:
            n *= d
        self.comm.cp_ring_wait(self.group, self.bg.RING_ACC, step % 2, n)
        return self.buf.u8[self._acc_off(step % 2): self._acc_off(step % 2) + 8 * n].view(torch.float32)

    def release_acc(self, step):
        n = 1
        for d in self.shape:
            n *= d
        self.comm.cp_ring_release(self.group, self.bg.RING_ACC, step % 2, n)


class _Timed:
    def __init__(self, be, kind, bus_bytes, stream, flops=0.0):
        self.be, self.kind, self.bus_bytes, self.stream, self.flops = be, kind, bus_bytes, stream, flops

    def __enter__(self):
        prof = self.be.comm_profile
        if prof is not None:
            self.e0, self.e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            self.e0.record(self.stream or torch.cuda.current_stream())
        return self

    def __exit__(self, *exc):
        prof = self.be.comm_profile
        if prof is not None and exc[0] is None:
            self.e1.record(self.stream or torch.cuda.current_stream())
            prof.setdefault(self.kind, []).append((self.e0, self.e1, float(self.bus_bytes), float(self.flops)))
        return False


def _vec(x):
    return 16 // x.element_size()


def _p(t):
    import ctypes
    return ctypes.c_void_p(t.data_ptr())


def _s():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

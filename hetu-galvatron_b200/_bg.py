"""ctypes binding of the C-ABI library (include/bg_galvatron.h) + the per-rank communicator object.

There is no CPU path: if ``libbg_galvatron.so`` is missing or fails to load, every use raises.  PyTorch is
plumbing here (device memory, streams, the bootstrap exchange of IPC handles); the collectives themselves
are the hand-written sm_90a kernels in ``csrc/``.
"""
import contextlib
import ctypes
import os
import threading

# the runtime keeps 4 streams busy at once (compute, unshard, grad-reduce, pipeline p2p) and some of their kernels wait
# on peers: give every stream its own hardware queue so none is falsely ordered behind a waiting kernel.  Only takes
# effect when set before the CUDA context exists.
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libbg_galvatron.so")

BF16, F32 = 0, 1
SUM, MAX = 0, 1
MAX_PEERS = 8
# LANE_RING: the context-parallel ring's hop flags (bg_cp_ring_*), nothing else
LANE_UNSHARD, LANE_REDUCE, LANE_ACT, LANE_MISC, LANE_PUSH, LANE_RING = 0, 1, 2, 3, 4, 5
RING_KV, RING_ACC = 0, 1

_c = ctypes
_vp, _sz, _i, _ll, _f = _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_longlong, _c.c_float


class bg_a2a_desc(_c.Structure):
    _fields_ = [("src_offs", _c.POINTER(_sz)), ("dst", _vp), ("batch", _ll), ("rows", _ll), ("row_elems", _ll),
                ("src_bs", _ll), ("src_rs", _ll), ("src_me_off", _ll), ("dst_bs", _ll), ("dst_rs", _ll),
                ("dst_peer_off", _ll)]


# name -> (restype, argtypes); every symbol declared in include/bg_galvatron.h
SIGNATURES = {
    "bg_abi_version": (_i, []),
    "bg_last_error": (_c.c_char_p, []),
    "bg_set_tunable": (_i, [_c.c_char_p, _ll]),
    "bg_get_tunable": (_ll, [_c.c_char_p]),
    "bg_launch_count": (_c.c_ulonglong, []),
    "bg_ctx_create": (_i, [_i, _i, _i, _sz, _c.POINTER(_vp)]),
    "bg_ctx_destroy": (_i, [_vp]),
    "bg_arena_info": (_i, [_vp, _c.POINTER(_vp), _c.POINTER(_sz), _c.POINTER(_sz)]),
    "bg_arena_alloc": (_i, [_vp, _sz, _c.POINTER(_sz)]),
    "bg_arena_export": (_i, [_vp, _vp]),
    "bg_arena_import": (_i, [_vp, _i, _vp]),
    "bg_arena_attach_local": (_i, [_vp, _i, _vp]),
    "bg_ctx_error_flag": (_i, [_vp, _c.POINTER(_i)]),
    "bg_ctx_error_info": (_i, [_vp, _c.POINTER(_i)]),
    "bg_ctx_create_ex": (_i, [_i, _i, _i, _sz, _c.c_uint, _c.POINTER(_vp)]),
    "bg_arena_alloc_aligned": (_i, [_vp, _sz, _sz, _c.POINTER(_sz)]),
    "bg_arena_mode": (_i, [_vp, _c.POINTER(_i), _c.POINTER(_i), _c.POINTER(_sz)]),
    "bg_arena_export_fd": (_i, [_vp, _c.POINTER(_i)]),
    "bg_arena_import_fd": (_i, [_vp, _i, _i]),
    "bg_group_mc_create": (_i, [_vp, _i, _sz, _c.POINTER(_i)]),
    "bg_group_mc_join": (_i, [_vp, _i, _i, _sz]),
    "bg_group_mc_bind": (_i, [_vp, _i, _sz]),
    "bg_group_mc_disable": (_i, [_vp, _i]),
    "bg_group_create": (_i, [_vp, _c.POINTER(_i), _i, _c.POINTER(_i)]),
    "bg_group_info": (_i, [_vp, _i, _c.POINTER(_i), _c.POINTER(_i), _c.POINTER(_i)]),
    "bg_build_groups": (_i, [_i, _i, _i, _i, _c.POINTER(_i), _c.POINTER(_i), _c.POINTER(_i), _c.POINTER(_i),
                             _c.POINTER(_i), _c.POINTER(_i), _c.POINTER(_i)]),
    "bg_barrier": (_i, [_vp, _i, _i, _vp]),
    "bg_all_gather_cast": (_i, [_vp, _i, _i, _vp, _i, _c.POINTER(_sz), _i, _sz, _vp]),
    "bg_reduce_scatter_acc": (_i, [_vp, _i, _i, _c.POINTER(_sz), _i, _vp, _i, _sz, _f, _f, _i, _vp]),
    "bg_all_reduce": (_i, [_vp, _i, _i, _c.POINTER(_sz), _vp, _sz, _i, _i, _f, _vp]),
    "bg_pair_sum_inplace": (_i, [_vp, _i, _i, _c.POINTER(_sz), _sz, _i, _f, _vp]),
    "bg_reduce_scatter_adamw": (_i, [_vp, _i, _i, _c.POINTER(_sz), _i, _vp, _vp, _vp, _sz, _f, _f, _f, _f, _f, _f, _f, _ll, _vp]),
    "bg_reduce_scatter_sumsq": (_i, [_vp, _i, _i, _c.POINTER(_sz), _i, _vp, _sz, _f, _f, _vp, _i, _c.POINTER(_sz), _i, _vp]),
    "bg_reduce_scatter_adamw_clipped": (_i, [_vp, _i, _i, _c.POINTER(_sz), _i, _vp, _vp, _vp, _sz, _f, _f, _f, _f, _f, _f, _f, _ll, _vp,
                                             _vp]),
    "bg_adamw_clipped": (_i, [_vp, _vp, _vp, _vp, _sz, _f, _f, _f, _f, _f, _ll, _vp, _vp]),
    "bg_all_to_all_rows": (_i, [_vp, _i, _i, _c.POINTER(bg_a2a_desc), _i, _i, _vp]),
    "bg_p2p_send": (_i, [_vp, _i, _sz, _vp, _sz, _i, _vp]),
    "bg_p2p_wait": (_i, [_vp, _i, _i, _vp]),
    "bg_p2p_release": (_i, [_vp, _i, _i, _vp]),
    "bg_cp_ring_push": (_i, [_vp, _i, _i, _i, _vp, _vp, _sz, _c.POINTER(_sz), _vp]),
    "bg_cp_ring_acc_push": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _ll, _ll, _ll, _ll, _ll, _c.POINTER(_sz), _vp]),
    "bg_cp_ring_wait": (_i, [_vp, _i, _i, _i, _sz, _vp]),
    "bg_cp_ring_release": (_i, [_vp, _i, _i, _i, _sz, _vp]),
    "bg_lse_merge": (_i, [_vp, _vp, _vp, _vp, _vp, _ll, _ll, _ll, _ll, _ll, _ll, _i, _vp]),
    "bg_cast": (_i, [_vp, _i, _vp, _i, _sz, _f, _i, _vp]),
    "bg_rmsnorm_fwd": (_i, [_vp, _vp, _vp, _vp, _ll, _ll, _f, _vp]),
    "bg_rmsnorm_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _ll, _ll, _i, _vp]),
    "bg_layernorm_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _ll, _ll, _f, _vp]),
    "bg_layernorm_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _ll, _i, _vp]),
    "bg_bias_gelu": (_i, [_vp, _vp, _vp, _vp, _ll, _ll, _i, _vp]),
    "bg_dropout_add_fwd": (_i, [_vp, _vp, _i, _vp, _vp, _ll, _ll, _ll, _ll, _ll, _c.c_double, _c.c_uint, _c.c_uint, _c.c_uint, _vp]),
    "bg_dropout_bwd": (_i, [_vp, _vp, _vp, _i, _ll, _ll, _ll, _ll, _ll, _c.c_double, _c.c_uint, _c.c_uint, _c.c_uint, _vp]),
    "bg_dropout_add_fwd_ids": (_i, [_vp, _vp, _i, _vp, _vp, _ll, _ll, _ll, _ll, _vp, _c.c_double, _c.c_uint, _c.c_uint, _c.c_uint, _vp]),
    "bg_dropout_bwd_ids": (_i, [_vp, _vp, _vp, _i, _ll, _ll, _ll, _ll, _vp, _c.c_double, _c.c_uint, _c.c_uint, _c.c_uint, _vp]),
    "bg_vit_patchify": (_i, [_vp, _i, _vp, _ll, _ll, _ll, _ll, _ll, _ll, _vp]),
    "bg_vit_embed_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _ll, _ll, _ll, _ll, _ll, _c.c_double, _c.c_uint, _c.c_uint, _c.c_uint, _vp]),
    "bg_vit_embed_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _ll, _ll, _ll, _ll, _ll, _ll, _c.c_double, _c.c_uint, _c.c_uint, _c.c_uint, _vp]),
    "bg_bias_tanh": (_i, [_vp, _vp, _vp, _vp, _ll, _ll, _vp]),
    "bg_swin_window_qkv_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _ll, _ll, _ll, _ll, _ll, _ll, _ll, _vp]),
    "bg_swin_window_qkv_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp, _ll, _ll, _ll, _ll, _ll, _ll, _ll, _vp]),
    "bg_swin_rel_bias_fwd": (_i, [_vp, _i, _vp, _vp, _vp, _ll, _ll, _ll, _ll, _ll, _ll, _vp]),
    "bg_swin_rel_bias_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _ll, _ll, _ll, _ll, _ll, _ll, _vp]),
    "bg_cross_attn_qkv_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _ll, _ll, _ll, _ll, _vp]),
    "bg_cross_attn_qkv_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _ll, _ll, _ll, _ll, _ll, _vp]),
    "bg_swin_window_merge_fwd": (_i, [_vp, _vp, _vp, _vp, _ll, _ll, _ll, _ll, _ll, _ll, _vp]),
    "bg_swin_window_merge_bwd": (_i, [_vp, _vp, _vp, _vp, _ll, _ll, _ll, _ll, _ll, _ll, _vp]),
    "bg_swin_merge_ln_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _ll, _ll, _ll, _i, _ll, _ll, _ll, _f, _vp]),
    "bg_swin_merge_ln_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _ll, _ll, _ll, _ll, _i, _ll, _ll, _vp]),
    "bg_swin_mean_pool_fwd": (_i, [_vp, _vp, _ll, _ll, _ll, _ll, _ll, _vp]),
    "bg_swin_mean_pool_bwd": (_i, [_vp, _vp, _ll, _ll, _ll, _ll, _vp]),
    "bg_drop_path_add_fwd": (_i, [_vp, _vp, _i, _vp, _vp, _ll, _ll, _ll, _ll, _c.c_double, _c.c_uint, _c.c_uint, _c.c_uint, _vp]),
    "bg_drop_path_add_bwd": (_i, [_vp, _vp, _vp, _i, _ll, _ll, _ll, _ll, _c.c_double, _c.c_uint, _c.c_uint, _c.c_uint, _vp]),
    "bg_philox4x32_10": (None, [_c.POINTER(_c.c_uint32), _c.POINTER(_c.c_uint32), _c.POINTER(_c.c_uint32)]),
    "bg_swiglu_fwd": (_i, [_vp, _vp, _ll, _ll, _vp]),
    "bg_swiglu_bwd": (_i, [_vp, _vp, _vp, _ll, _ll, _vp]),
    "bg_qkv_rope": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _ll, _ll, _ll, _ll, _ll, _i, _vp]),
    "bg_ce_rowmax": (_i, [_vp, _i, _vp, _ll, _ll, _vp]),
    "bg_ce_sumexp": (_i, [_vp, _i, _vp, _vp, _vp, _ll, _ll, _ll, _vp]),
    "bg_ce_bwd": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _ll, _ll, _ll, _vp]),
    "bg_gemm_bf16": (_i, [_vp, _vp, _vp, _ll, _ll, _ll, _i, _i, _vp]),
    "bg_gemm_bf16_add": (_i, [_vp, _vp, _vp, _vp, _ll, _ll, _ll, _i, _vp]),
    "bg_gemm_reduce_scatter": (_i, [_vp, _i, _i, _vp, _vp, _ll, _ll, _ll, _i, _c.POINTER(_sz), _c.POINTER(_sz), _vp, _vp]),
    "bg_gemm_all_reduce": (_i, [_vp, _i, _i, _vp, _vp, _ll, _ll, _ll, _i, _c.POINTER(_sz), _c.POINTER(_sz), _c.POINTER(_sz), _vp]),
    "bg_all_gather_gemm": (_i, [_vp, _i, _i, _vp, _c.POINTER(_sz), _c.POINTER(_sz), _vp, _vp, _ll, _ll, _ll, _i, _vp, _vp]),
}

_lib = None
_lib_lock = threading.Lock()
_SERIAL = os.environ.get("HGB_SERIAL_COLLECTIVES", "0") == "1"


class BgError(RuntimeError):
    pass


def lib():
    """The loaded C-ABI library; raises (never falls back) when it is not built."""
    global _lib
    if _lib is None:
        with _lib_lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise BgError("CUDA extension not built: %s is missing (run `python -c 'import __graft_entry__ as g; "
                                  "g.build()'`). There is no CPU fallback." % LIB_PATH)
                handle = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
                for name, (res, args) in SIGNATURES.items():
                    fn = getattr(handle, name)  # AttributeError = ABI mismatch: fail loudly
                    fn.restype, fn.argtypes = res, args
                if handle.bg_abi_version() != 1:
                    raise BgError("bg_galvatron ABI version mismatch")
                _lib = handle
    return _lib


def check(rc):
    if rc != 0:
        raise BgError("bg_galvatron error %d: %s" % (rc, lib().bg_last_error().decode()))


def set_tunable(name, value):
    check(lib().bg_set_tunable(name.encode(), int(value)))


def get_tunable(name):
    return int(lib().bg_get_tunable(name.encode()))


def launch_count():
    return int(lib().bg_launch_count())


def dtype_code(dt):
    import torch
    if dt == torch.bfloat16:
        return BF16
    if dt == torch.float32:
        return F32
    raise BgError("unsupported dtype %s (bf16/fp32 only)" % dt)


def _stream_ptr(stream=None):
    import torch
    s = torch.cuda.current_stream() if stream is None else stream
    return _vp(s.cuda_stream)


def _ptr(t):
    return _vp(t.data_ptr())


class _ArenaExport:
    """``__cuda_array_interface__`` carrier so torch can alias arena memory without copying."""

    def __init__(self, ptr, nbytes, owner):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3,
                                         "strides": None}
        self._owner = owner


class SymBuffer:
    """A symmetric buffer: one allocation per member of ``group`` (arena offsets differ per rank).  ``registered``: a view of an
    existing arena range (``BgComm.sym_register``) rather than an allocation of its own."""

    def __init__(self, comm, group, nbytes, offset, tensor_u8, key, registered=False):
        self.comm, self.group, self.nbytes, self.offset, self.u8, self.key = comm, group, nbytes, offset, tensor_u8, key
        self.registered = registered
        self.offsets = None  # ctypes size_t[group.size] once exchanged

    def view(self, dtype, numel=None):
        t = self.u8.view(dtype)
        return t if numel is None else t[:numel]

    def offs(self):
        if self.offsets is None:
            if self.group.size == 1:
                self.offsets = (_sz * 1)(self.offset)
            else:
                raise BgError("symmetric buffer %r used before BgComm.exchange()" % (self.key,))
        return self.offsets

    def sub(self, byte_offset):
        """ctypes offsets array for a sub-range starting ``byte_offset`` bytes into every member's buffer."""
        base = self.offs()
        return (_sz * len(base))(*[int(o) + int(byte_offset) for o in base])


class _FdChannel:
    """POSIX file descriptors between the processes of one node: a listening unix socket per rank, SCM_RIGHTS messages
    tagged (source rank, tag).  Used for the VMM arena handles and the multicast objects (a cudaIpc handle cannot carry
    either).  The socket paths travel over the bootstrap process group."""

    def __init__(self, rank, world, pg=None):
        import socket
        import tempfile
        import torch.distributed as dist
        self.rank, self.world = rank, world
        self.path = os.path.join(tempfile.gettempdir(), "hgb_fd_%d_%d_%d.sock" % (os.getuid(), os.getpid(), rank))
        if os.path.exists(self.path):
            os.unlink(self.path)
        self.srv = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        self.srv.bind(self.path)
        self.srv.listen(max(8, world))
        paths = [None] * world
        dist.all_gather_object(paths, self.path, group=pg)
        self.paths = paths

    def exchange(self, outgoing, n_expected):
        """outgoing: [(dest_rank, tag, fd)]; returns {(src_rank, tag): fd} for ``n_expected`` incoming descriptors."""
        import pickle
        import socket
        import threading

        def send_all():
            for dest, tag, fd in outgoing:
                with socket.socket(socket.AF_UNIX, socket.SOCK_STREAM) as s:
                    s.connect(self.paths[dest])
                    socket.send_fds(s, [pickle.dumps((self.rank, tag))], [fd])
        sender = threading.Thread(target=send_all)
        sender.start()
        got = {}
        while len(got) < n_expected:
            conn, _ = self.srv.accept()
            with conn:
                msg, fds, _, _ = socket.recv_fds(conn, 4096, 1)
                got[pickle.loads(msg)] = fds[0]
        sender.join()
        return got

    def close(self):
        self.srv.close()
        if os.path.exists(self.path):
            os.unlink(self.path)


class BgComm:
    """One rank's handle on the peer-memory runtime: arena, groups, collectives.

    ``BgComm(rank, world, device, arena_bytes)`` then either ``connect_ipc()`` (one process per GPU; handles
    exchanged once over the bootstrap torch.distributed group) or ``BgComm.local_world(n, ...)`` (n virtual
    ranks inside this process -- what the single-GPU parity tests use).
    """

    def __init__(self, rank, world, device, arena_bytes, vmm=False):
        import torch
        self.rank, self.world, self.device = int(rank), int(world), int(device)
        self._last_coll, self._coll_events, self._coll_i = None, None, 0
        self._ctx = _vp()
        self.vmm, self._fd_channel, self._nvls = bool(vmm), None, {}
        torch.cuda.set_device(self.device)
        torch.cuda.init()
        if vmm:   # arena from the virtual-memory API: what NVSwitch multicast objects can bind (opt-in, HGB_NVLS=1)
            check(lib().bg_ctx_create_ex(self.rank, self.world, self.device, int(arena_bytes), 1, ctypes.byref(self._ctx)))
        else:
            check(lib().bg_ctx_create(self.rank, self.world, self.device, int(arena_bytes), ctypes.byref(self._ctx)))
        base, nbytes, used = _vp(), _sz(), _sz()
        check(lib().bg_arena_info(self._ctx, ctypes.byref(base), ctypes.byref(nbytes), ctypes.byref(used)))
        self.arena_ptr, self.arena_bytes = base.value, nbytes.value
        self._arena_u8 = torch.as_tensor(_ArenaExport(self.arena_ptr, self.arena_bytes, self), device="cuda:%d" % self.device)
        self._first_aligned = 0
        if vmm:   # multicast ranges start on a multicast-granularity boundary behind the signal pad
            gran = self.arena_mode()[2]
            if gran:
                o = _sz()
                check(lib().bg_arena_alloc_aligned(self._ctx, 0, int(gran), ctypes.byref(o)))
                self._first_aligned = o.value
        self._sym = {}       # key -> SymBuffer
        self._sym_seq = {}   # group ranks -> next sequence number
        self._pending = []   # SymBuffers whose peer offsets are not known yet
        self._local_peers = None
        self._gids = {}

    # ---- bootstrap ------------------------------------------------------------------------------------
    @classmethod
    def local_world(cls, n, device=0, arena_bytes=64 << 20):
        comms = [cls(r, n, device, arena_bytes) for r in range(n)]
        for a in comms:
            for b in comms:
                if a is not b:
                    check(lib().bg_arena_attach_local(a._ctx, b.rank, b._ctx))
            a._local_peers = comms
        return comms

    def connect_ipc(self, pg=None):
        """Exchange cudaIpc handles over the bootstrap process group and map every peer's arena."""
        import torch.distributed as dist
        if self.world == 1:
            return
        handle = (ctypes.c_ubyte * 64)()
        check(lib().bg_arena_export(self._ctx, handle))
        gathered = [None] * self.world
        dist.all_gather_object(gathered, bytes(handle), group=pg)
        for peer, h in enumerate(gathered):
            if peer != self.rank:
                buf = (ctypes.c_ubyte * 64).from_buffer_copy(h)
                check(lib().bg_arena_import(self._ctx, peer, buf))

    def arena_mode(self):
        """(vmm arena?, multicast supported?, multicast granularity in bytes)"""
        v, m, g = _i(), _i(), _sz()
        check(lib().bg_arena_mode(self._ctx, ctypes.byref(v), ctypes.byref(m), ctypes.byref(g)))
        return bool(v.value), bool(m.value), int(g.value)

    def connect_vmm(self, pg=None):
        """``connect_ipc`` for a VMM arena: every rank exports its arena as a file descriptor, sends it to every peer over the
        unix-socket channel and maps the peers' arenas."""
        if self.world == 1:
            return
        self._fd_channel = _FdChannel(self.rank, self.world, pg)
        fd = _i()
        check(lib().bg_arena_export_fd(self._ctx, ctypes.byref(fd)))
        got = self._fd_channel.exchange([(peer, "arena", fd.value) for peer in range(self.world) if peer != self.rank], self.world - 1)
        for (src, _tag), pfd in got.items():
            check(lib().bg_arena_import_fd(self._ctx, src, pfd))
            os.close(pfd)
        os.close(fd.value)

    def setup_nvls(self, pg=None):
        """Collective over the whole job, after ``exchange()``: for every group of >= 2 ranks, ONE multicast object over the arena
        range that holds the group's symmetric buffers (those that sit at the same offset on every member -- SPMD allocation
        makes that the rule).  The group's first rank creates the object and hands its descriptor to the members; everybody
        adds its device; barrier; everybody binds its own arena range; the outcome is agreed on by all ranks, and a group whose
        setup failed anywhere simply keeps the peer-to-peer kernels.  Collectives on buffers inside a bound range then use the
        switch on their own (multimem.st / multimem.ld_reduce), see include/bg_galvatron.h."""
        import torch.distributed as dist
        vmm, mc, gran = self.arena_mode()
        if not (vmm and mc):
            return {}
        regions = {}
        for buf in self._sym.values():
            # (a registered range lies inside memory of another group -- a unit's gradient buffer: a bind over it would cover that)
            if buf.registered or buf.group.size < 2 or buf.offsets is None or len(set(int(o) for o in buf.offsets)) != 1:
                continue
            ranks = tuple(buf.group.ranks)
            lo, hi = regions.get(ranks, (1 << 62, 0))
            regions[ranks] = (min(lo, buf.offset), max(hi, buf.offset + buf.nbytes))
        plan = []
        for ranks in sorted(regions):
            lo, hi = regions[ranks]
            lo = max(lo // gran * gran, self._first_aligned)
            hi = min((hi + gran - 1) // gran * gran, self.arena_bytes)
            plan.append((ranks, lo, hi - lo))
        ok = {ranks: True for ranks, _, _ in plan}
        outgoing, expected, created = [], 0, {}
        for ranks, lo, nbytes in plan:
            gid = self._gid_of_ranks(ranks)
            if self.rank == ranks[0]:
                fd = _i(-1)
                if lib().bg_group_mc_create(self._ctx, gid, int(nbytes), ctypes.byref(fd)) != 0:
                    ok[ranks] = False
                    fd = _i(os.open(os.devnull, os.O_RDONLY))      # the members still expect a descriptor
                created[ranks] = fd.value
                outgoing += [(r, ("mc", ranks, ok[ranks]), fd.value) for r in ranks[1:]]
            else:
                expected += 1
        got = self._fd_channel.exchange(outgoing, expected) if self.world > 1 else {}
        by_group = {tag[1]: (tag[2], fd) for (_src, tag), fd in got.items()}
        for ranks, lo, nbytes in plan:
            gid = self._gid_of_ranks(ranks)
            if self.rank == ranks[0]:
                if ok[ranks] and lib().bg_group_mc_join(self._ctx, gid, -1, int(nbytes)) != 0:
                    ok[ranks] = False
                os.close(created[ranks])
            else:
                good, fd = by_group[ranks]
                if not good or lib().bg_group_mc_join(self._ctx, gid, fd, int(nbytes)) != 0:
                    ok[ranks] = False
                os.close(fd)
        if self.world > 1:
            dist.barrier(group=pg)          # every device is in every object before anyone binds
        for ranks, lo, nbytes in plan:
            if ok[ranks] and lib().bg_group_mc_bind(self._ctx, self._gid_of_ranks(ranks), int(lo)) != 0:
                ok[ranks] = False
        if self.world > 1:
            every = [None] * self.world
            dist.all_gather_object(every, ok, group=pg)
        else:
            every = [ok]
        for ranks, lo, nbytes in plan:
            good = all(d.get(ranks, True) for d in every)
            if good:
                self._nvls[ranks] = (lo, nbytes)
            else:
                lib().bg_group_mc_disable(self._ctx, self._gid_of_ranks(ranks))
        return dict(self._nvls)

    def _gid_of_ranks(self, ranks):
        gid = self._gids.get(tuple(ranks))
        if gid is None:
            arr = (_i * len(ranks))(*ranks)
            out = _i()
            check(lib().bg_group_create(self._ctx, arr, len(ranks), ctypes.byref(out)))
            gid = self._gids[tuple(ranks)] = out.value
        return gid

    def close(self):
        if self._fd_channel is not None:
            self._fd_channel.close()
            self._fd_channel = None
        if self._ctx:
            self._arena_u8 = None
            check(lib().bg_ctx_destroy(self._ctx))
            self._ctx = _vp()

    # ---- groups ---------------------------------------------------------------------------------------
    def group_id(self, group):
        return self._gid_of_ranks(tuple(group.ranks))

    # ---- symmetric memory -----------------------------------------------------------------------------
    def alloc(self, nbytes):
        off = _sz()
        check(lib().bg_arena_alloc(self._ctx, int(nbytes), ctypes.byref(off)))
        return off.value, self._arena_u8[off.value: off.value + int(nbytes)]

    def sym_alloc(self, group, nbytes, tag="", align=256):
        """Allocate the calling rank's part of a symmetric buffer.  Members must call this in the same order
        per group (SPMD); peer offsets become known at the next ``exchange()``.  ``align``: offset AND size granularity
        (the multicast granularity for a buffer that NVLS binds)."""
        nbytes = (int(nbytes) + align - 1) // align * align
        if align > 256:
            o = _sz()
            check(lib().bg_arena_alloc_aligned(self._ctx, nbytes, int(align), ctypes.byref(o)))
            off, t = o.value, self._arena_u8[o.value: o.value + nbytes]
        else:
            off, t = self.alloc(nbytes)
        return self._add_sym(group, nbytes, off, t, registered=False)

    def sym_register(self, group, byte_offset, nbytes):
        """A symmetric buffer over an existing range ``[byte_offset, byte_offset + nbytes)`` of this rank's arena -- memory another
        buffer already owns, such as one parameter's slice of a unit's gradient buffer.  Same ordering rule as ``sym_alloc`` (it
        takes the group's next sequence number); peer offsets become known at the next ``exchange()``, which also refuses a
        registration whose size differs between the members.  Offset and size: whole 16-B vectors."""
        byte_offset, nbytes = int(byte_offset), int(nbytes)
        used = _sz()
        check(lib().bg_arena_info(self._ctx, None, None, ctypes.byref(used)))
        if byte_offset % 16 or nbytes % 16 or nbytes <= 0 or byte_offset + nbytes > used.value:
            raise BgError("sym_register: [%d, +%d) is not a 16-B aligned range of allocated arena memory" % (byte_offset, nbytes))
        return self._add_sym(group, nbytes, byte_offset, self._arena_u8[byte_offset: byte_offset + nbytes], registered=True)

    def _add_sym(self, group, nbytes, off, t, registered):
        ranks = tuple(group.ranks)
        seq = self._sym_seq.get(ranks, 0)
        self._sym_seq[ranks] = seq + 1
        key = (ranks, seq)
        buf = SymBuffer(self, group, nbytes, off, t, key, registered=registered)
        self._sym[key] = buf
        if group.size > 1:
            self._pending.append(buf)
        return buf

    def exchange(self, pg=None):
        """Collective over the whole job: learn the peers' offsets of every pending symmetric buffer (and check that every member
        registered the same number of bytes for a ``sym_register`` buffer)."""
        mine = {b.key: (b.offset, b.nbytes) for b in self._pending}
        if self._local_peers is not None:
            tables = {c.rank: {b.key: (b.offset, b.nbytes) for b in c._sym.values()} for c in self._local_peers}
        elif self.world == 1:
            tables = {self.rank: mine}
        else:
            import torch.distributed as dist
            gathered = [None] * self.world
            dist.all_gather_object(gathered, mine, group=pg)
            tables = dict(enumerate(gathered))
        for b in self._pending:
            offs = []
            for r in b.group.ranks:
                if b.key not in tables[r]:
                    raise BgError("rank %d did not allocate symmetric buffer %r (allocation order differs)" % (r, b.key))
                off, nbytes = tables[r][b.key]
                if b.registered and nbytes != b.nbytes:
                    raise BgError("registered symmetric buffer %r: %d bytes on rank %d, %d on rank %d -- the members' ranges must have "
                                  "the same size (tied embeddings: the same vocabulary sharding on both rows)"
                                  % (b.key, b.nbytes, self.rank, nbytes, r))
                offs.append(off)
            b.offsets = (_sz * len(offs))(*offs)
        self._pending = []

    # ---- collectives (async on the current or given torch stream) -------------------------------------
    @contextlib.contextmanager
    def _in_order(self, stream):
        """The stream a cross-rank kernel is launched on.  Round 1 chained every such kernel of a rank into one total order
        (its 256-thread / 128-register kernels could not share an SM, and two of them in flight on different streams could
        deadlock across ranks -- seen with ZeRO-3's concurrent all-gather and reduce-scatter at Llama-70B sizes).  The slim
        kernels (128 threads x <= 64 registers, one CTA per SM, no shared memory) are always co-resident, beside each other
        and beside a fused GEMM (three of them; two beside a plain GEMM's wider tile, which waits on no peer and always
        retires), so no ordering is imposed any more: collectives on different streams really overlap.
        ``HGB_SERIAL_COLLECTIVES=1`` restores the chain (debugging aid)."""
        import torch
        s = torch.cuda.current_stream() if stream is None else stream
        if not _SERIAL:
            yield _vp(s.cuda_stream)
            return
        last = self._last_coll
        if last is not None and last[0] != s.cuda_stream:
            s.wait_event(last[1])
        yield _vp(s.cuda_stream)
        if self._coll_events is None:
            self._coll_events = [torch.cuda.Event() for _ in range(8)]
        ev = self._coll_events[self._coll_i % 8]
        self._coll_i += 1
        ev.record(s)
        self._last_coll = (s.cuda_stream, ev)

    def barrier(self, group, lane=LANE_MISC, stream=None):
        with self._in_order(stream) as sp:
            check(lib().bg_barrier(self._ctx, self.group_id(group), lane, sp))

    def all_gather_cast(self, group, src, dst, shard_elems=None, lane=LANE_UNSHARD, stream=None, dst_dtype=None,
                        dst_byte_offset=0):
        """dst (SymBuffer) slot my_index <- cast(src) on every member."""
        import torch
        n = src.numel() if shard_elems is None else int(shard_elems)
        dd = torch.bfloat16 if dst_dtype is None else dst_dtype
        offs = dst.offs() if dst_byte_offset == 0 else dst.sub(dst_byte_offset)
        with self._in_order(stream) as sp:
            check(lib().bg_all_gather_cast(self._ctx, self.group_id(group), lane, _ptr(src), dtype_code(src.dtype), offs,
                                           dtype_code(dd), n, sp))

    def reduce_scatter_acc(self, group, src, src_dtype, dst, shard_elems=None, prescale=1.0, postscale=1.0,
                           accumulate=False, lane=LANE_REDUCE, stream=None, src_byte_offset=0):
        """dst[shard] = [dst +] sum_members(src_member[my slice]) * prescale * postscale."""
        n = dst.numel() if shard_elems is None else int(shard_elems)
        offs = src.offs() if src_byte_offset == 0 else src.sub(src_byte_offset)
        with self._in_order(stream) as sp:
            check(lib().bg_reduce_scatter_acc(self._ctx, self.group_id(group), lane, offs, dtype_code(src_dtype), _ptr(dst),
                                              dtype_code(dst.dtype), n, float(prescale), float(postscale),
                                              1 if accumulate else 0, sp))

    def reduce_scatter_adamw(self, group, src, src_dtype, param, exp_avg, exp_avg_sq, shard_elems, prescale, postscale, lr, beta1,
                             beta2, eps, weight_decay, step, lane=LANE_REDUCE, stream=None):
        with self._in_order(stream) as sp:
            check(lib().bg_reduce_scatter_adamw(self._ctx, self.group_id(group), lane, src.offs(), dtype_code(src_dtype), _ptr(param),
                                                _ptr(exp_avg), _ptr(exp_avg_sq), int(shard_elems), float(prescale), float(postscale),
                                                float(lr), float(beta1), float(beta2), float(eps), float(weight_decay), int(step),
                                                sp))

    def reduce_scatter_sumsq(self, group, src, src_dtype, shard_elems, prescale, postscale, partials, skip=(), dst=None,
                             lane=LANE_REDUCE, stream=None):
        """Norm pass: per-warp fp32 sums of squares of the reduced gradient into ``partials`` (fp32, whole tensor: the unused tail is
        zeroed), leaving out the shard-relative element ranges ``skip`` [(lo, hi)]; with ``dst`` also the reduced fp32 shard."""
        flat = [int(x) for r in skip for x in r]
        arr = (_sz * max(1, len(flat)))(*flat)
        with self._in_order(stream) as sp:
            check(lib().bg_reduce_scatter_sumsq(self._ctx, self.group_id(group), lane, src.offs(), dtype_code(src_dtype),
                                                _ptr(dst) if dst is not None else None, int(shard_elems), float(prescale),
                                                float(postscale), _ptr(partials), partials.numel(), arr, len(skip), sp))

    def reduce_scatter_adamw_clipped(self, group, src, src_dtype, param, exp_avg, exp_avg_sq, shard_elems, prescale, postscale, lr,
                                     beta1, beta2, eps, weight_decay, step, clip_coef, lane=LANE_REDUCE, stream=None):
        """``reduce_scatter_adamw`` with the gradient multiplied by the device scalar ``clip_coef`` (fp32 tensor, or None for 1)."""
        with self._in_order(stream) as sp:
            check(lib().bg_reduce_scatter_adamw_clipped(self._ctx, self.group_id(group), lane, src.offs(), dtype_code(src_dtype),
                                                        _ptr(param), _ptr(exp_avg), _ptr(exp_avg_sq), int(shard_elems), float(prescale),
                                                        float(postscale), float(lr), float(beta1), float(beta2), float(eps),
                                                        float(weight_decay), int(step),
                                                        _ptr(clip_coef) if clip_coef is not None else None, sp))

    def all_reduce(self, group, src, dst, elems=None, op=SUM, scale=1.0, lane=LANE_ACT, stream=None, src_byte_offset=0):
        n = dst.numel() if elems is None else int(elems)
        offs = src.offs() if src_byte_offset == 0 else src.sub(src_byte_offset)
        with self._in_order(stream) as sp:
            check(lib().bg_all_reduce(self._ctx, self.group_id(group), lane, offs, _ptr(dst), n, dtype_code(dst.dtype), op,
                                      float(scale), sp))

    def pair_sum_inplace(self, group, buf, dtype, elems=None, scale=1.0, lane=LANE_REDUCE, stream=None):
        """Both members' ``buf`` (SymBuffer of a two-member ``group``, first ``elems`` elements of ``dtype``) <- scale * (x0 + x1)."""
        import torch
        n = buf.nbytes // torch.empty((), dtype=dtype).element_size() if elems is None else int(elems)
        with self._in_order(stream) as sp:
            check(lib().bg_pair_sum_inplace(self._ctx, self.group_id(group), lane, buf.offs(), n, dtype_code(dtype), float(scale), sp))

    def all_to_all_rows(self, group, descs, dtype, lane=LANE_ACT, stream=None):
        """descs: list of dicts with keys src(SymBuffer) [src_byte_offset] dst(tensor) batch rows row_elems src_bs src_rs
        src_me_off dst_bs dst_rs dst_peer_off."""
        arr = (bg_a2a_desc * len(descs))()
        keep = []
        for i, d in enumerate(descs):
            offs = d["src"].offs() if d.get("src_byte_offset", 0) == 0 else d["src"].sub(d["src_byte_offset"])
            keep.append(offs)
            arr[i].src_offs = ctypes.cast(offs, _c.POINTER(_sz))
            arr[i].dst = d["dst"].data_ptr()
            for k in ("batch", "rows", "row_elems", "src_bs", "src_rs", "src_me_off", "dst_bs", "dst_rs", "dst_peer_off"):
                setattr(arr[i], k, int(d[k]))
        with self._in_order(stream) as sp:
            check(lib().bg_all_to_all_rows(self._ctx, self.group_id(group), lane, arr, len(descs), dtype_code(dtype),
                                           sp))

    def gemm_reduce_scatter(self, group, a, b, m, n, k, layout, partial, partial_byte_offset, flags_byte_offset, out,
                            lane=LANE_ACT, stream=None):
        """C = A op B reduce-scattered along M over ``group`` in one fused operation (partial tiles -> owner's HBM)."""
        with self._in_order(stream) as sp:
            check(lib().bg_gemm_reduce_scatter(self._ctx, self.group_id(group), lane, _ptr(a), _ptr(b), int(m), int(n), int(k), int(layout),
                                               partial.sub(partial_byte_offset), partial.sub(flags_byte_offset), _ptr(out),
                                               sp))

    def gemm_all_reduce(self, group, a, b, m, n, k, layout, buf, partial_byte_offset, flags_byte_offset, out_byte_offset,
                        lane=LANE_ACT, stream=None):
        """C = A op B summed over ``group``, complete in every member's ``buf`` at ``out_byte_offset`` (GEMM + all-reduce fused)."""
        with self._in_order(stream) as sp:
            check(lib().bg_gemm_all_reduce(self._ctx, self.group_id(group), lane, _ptr(a), _ptr(b), int(m), int(n), int(k), int(layout),
                                           buf.sub(partial_byte_offset), buf.sub(flags_byte_offset), buf.sub(out_byte_offset), sp))

    def all_gather_gemm(self, group, a_local, b, out, m, n, k, layout, buf, stage_byte_offset, flags_byte_offset, comm_stream,
                        lane=LANE_PUSH, stream=None):
        """out[M,N] = gather_M(a_local) op B: chunk-signalled push on ``comm_stream`` + GEMM consuming chunks as they land."""
        with self._in_order(stream) as sp:
            check(lib().bg_all_gather_gemm(self._ctx, self.group_id(group), lane, _ptr(a_local), buf.sub(stage_byte_offset),
                                           buf.sub(flags_byte_offset), _ptr(b), _ptr(out), int(m), int(n), int(k), int(layout), sp,
                                           _vp(comm_stream.cuda_stream)))

    def p2p_send(self, peer_rank, dst_offset, src, flag_id, stream=None):
        check(lib().bg_p2p_send(self._ctx, int(peer_rank), int(dst_offset), _ptr(src), src.numel() * src.element_size(),
                                int(flag_id), _stream_ptr(stream)))

    def p2p_wait(self, peer_rank, flag_id, stream=None):
        check(lib().bg_p2p_wait(self._ctx, int(peer_rank), int(flag_id), _stream_ptr(stream)))

    def p2p_release(self, peer_rank, flag_id, stream=None):
        check(lib().bg_p2p_release(self._ctx, int(peer_rank), int(flag_id), _stream_ptr(stream)))

    # ---- ring context parallelism: one hop to the next member of ``group`` (include/bg_galvatron.h, C15) ----
    def cp_ring_push(self, group, slot, parity, wait_free, k, v, stream=None):
        """k, v (bf16, same numel) -> the next member's ``slot`` (SymBuffer view offsets of the parity's [k | v] slot)."""
        check(lib().bg_cp_ring_push(self._ctx, self.group_id(group), int(parity), 1 if wait_free else 0, _ptr(k), _ptr(v), k.numel(),
                                    slot, _stream_ptr(stream)))

    def cp_ring_acc_push(self, group, slot, parity, wait_free, acc_in, dk, dv, batch, rows, row_elems, c_row0, c_rows, stream=None):
        """next member's fp32 [dK | dV] slot = acc_in (or 0) + the bf16 contribution rows c_row0 .. c_row0 + c_rows - 1."""
        check(lib().bg_cp_ring_acc_push(self._ctx, self.group_id(group), int(parity), 1 if wait_free else 0,
                                        _ptr(acc_in) if acc_in is not None else None, _ptr(dk) if dk is not None else None,
                                        _ptr(dv) if dv is not None else None, int(batch), int(rows), int(row_elems), int(c_row0),
                                        int(c_rows), slot, _stream_ptr(stream)))

    def cp_ring_wait(self, group, kind, parity, elems, stream=None):
        check(lib().bg_cp_ring_wait(self._ctx, self.group_id(group), int(kind), int(parity), int(elems), _stream_ptr(stream)))

    def cp_ring_release(self, group, kind, parity, elems, stream=None):
        check(lib().bg_cp_ring_release(self._ctx, self.group_id(group), int(kind), int(parity), int(elems), _stream_ptr(stream)))

    def error_flag(self):
        out = _i()
        check(lib().bg_ctx_error_flag(self._ctx, ctypes.byref(out)))
        return out.value

    def error_info(self):
        """The device-side timeout record: status, kind (1 signalling / 2 waiting for a peer, 3 fused-GEMM tile reducer),
        CTA, thread-or-tile, value last seen, and two kind-specific integers."""
        out = (_i * 8)()
        check(lib().bg_ctx_error_info(self._ctx, out))
        return list(out)


# ---- local ops (no communicator needed) ---------------------------------------------------------------------
def cast(src, dst, scale=1.0, accumulate=False, stream=None):
    check(lib().bg_cast(_ptr(src), dtype_code(src.dtype), _ptr(dst), dtype_code(dst.dtype), src.numel(), float(scale),
                        1 if accumulate else 0, _stream_ptr(stream)))


def adamw_clipped(param, exp_avg, exp_avg_sq, grad, lr, beta1, beta2, eps, weight_decay, step, clip_coef, stream=None):
    """AdamW on fp32 (param, exp_avg, exp_avg_sq) with the local fp32 ``grad`` multiplied by the device scalar ``clip_coef``."""
    check(lib().bg_adamw_clipped(_ptr(param), _ptr(exp_avg), _ptr(exp_avg_sq), _ptr(grad), grad.numel(), float(lr), float(beta1),
                                 float(beta2), float(eps), float(weight_decay), int(step),
                                 _ptr(clip_coef) if clip_coef is not None else None, _stream_ptr(stream)))


def lse_merge(blk_out, blk_lse, acc_out, acc_lse, final_out=None, row_off=0, init=False, stream=None):
    """Merge one attention block (out [b, sq_blk, n, d] bf16, lse [b, n, sq_blk] fp32) into the running fp32 (acc_out [b, s, n, d],
    acc_lse [b, n, s]) at query rows row_off..; ``final_out`` (bf16 [b, s, n, d]): also write the merged output there."""
    b, s, n, d = acc_out.shape
    for t in (blk_out, blk_lse, acc_out, acc_lse) + ((final_out,) if final_out is not None else ()):
        if not t.is_contiguous():
            raise BgError("lse_merge operands must be contiguous")
    check(lib().bg_lse_merge(_ptr(blk_out), _ptr(blk_lse), _ptr(acc_out), _ptr(acc_lse), _ptr(final_out) if final_out is not None else None,
                             b, s, blk_out.shape[1], n, d, int(row_off), 1 if init else 0, _stream_ptr(stream)))


def gemm_bf16_add(a, b, c, addend, m, n, k, layout, stream=None):
    """C = A op B + addend (residual add in the GEMM epilogue)."""
    check(lib().bg_gemm_bf16_add(_ptr(a), _ptr(b), _ptr(c), _ptr(addend), int(m), int(n), int(k), int(layout), _stream_ptr(stream)))


def gemm_bf16(a, b, c, m, n, k, layout, accumulate=False, stream=None):
    """layout 0: C=A[M,K]B[N,K]^T   1: C=A[M,K]B[K,N]   2: C=A[K,M]^T B[K,N]  (row-major bf16)."""
    check(lib().bg_gemm_bf16(_ptr(a), _ptr(b), _ptr(c), int(m), int(n), int(k), int(layout), 1 if accumulate else 0,
                             _stream_ptr(stream)))

// bg_comm.cu -- symmetric arena (cudaIpc or VMM), groups, device-side barrier, pipeline p2p and NVSwitch multicast setup.
// The collective kernels themselves live in bg_coll.cu.  sm_90a; NVLink 4 / NVSwitch peer loads & stores, no NCCL.
#include <math.h>
#include <stdarg.h>
#include <string.h>

#include "bg_ctx.cuh"

namespace bg {
thread_local std::string g_last_error;
std::atomic<unsigned long long> g_launches{0};
Tunables g_tun;

int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}
}  // namespace bg

using namespace bg;

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------

int bg_preload_coll();
int bg_preload_gemm();
int bg_preload_ops();
static __global__ void barrier_kernel(Sig s);
__global__ void p2p_raise_kernel(uint32_t* flag, unsigned long long timeout_ns, int* err);
__global__ void p2p_consume_kernel(uint32_t* flag, unsigned long long timeout_ns, int* err);

static void enumerate_slots(bg_ctx* c) {
    // every arithmetic progression of 2..BG_MAX_PEERS ranks inside [0, world): same table on all ranks
    int next = 0;
    for (int stride = 1; stride < c->world; ++stride)
        for (int size = 2; size <= BG_MAX_PEERS; ++size)
            for (int first = 0; first + (size - 1) * stride < c->world; ++first)
                c->slot_of[std::make_tuple(first, stride, size)] = next++;
}


// =================================================================================================================
// VMM arena + NVLS (NVSwitch multicast) all-reduce.  OPT-IN (bg_ctx_create_ex flag BG_CTX_VMM, HGB_NVLS=1 on the host side):
// the default arena is cudaMalloc + cudaIpc.  Multicast objects can only bind memory that was created with cuMemCreate, so
// this mode allocates the arena through the virtual-memory API and shares it (and the multicast objects) between the
// processes as POSIX file descriptors, which the host passes over a unix socket (SCM_RIGHTS).
// Replaces NCCL's NVLS all-reduce for the tensor-parallel reductions (mappings_group.py:19, layers.py:474-480):
// two-shot -- every member reduces ITS slice in the switch (multimem.ld_reduce) and broadcasts it (multimem.st).
// =================================================================================================================

namespace {

struct Drv {
    CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
    CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
    CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
    CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
    CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
    CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
    CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
    CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long) = nullptr;
    CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
    CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
    CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*) = nullptr;
    CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice) = nullptr;
    CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long) = nullptr;
    CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags) = nullptr;
    CUresult (*DeviceGet)(CUdevice*, int) = nullptr;
    CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice) = nullptr;
    CUresult (*GetErrorString)(CUresult, const char**) = nullptr;
    bool ok = false;
};

template <typename F>
bool drv_sym(const char* name, F* out) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
        cudaGetLastError();
        return false;
    }
    *out = reinterpret_cast<F>(p);
    return true;
}

Drv& drv() {
    static Drv d;
    static std::once_flag once;
    std::call_once(once, [] {
        bool ok = true;
        ok &= drv_sym("cuMemCreate", &d.MemCreate);
        ok &= drv_sym("cuMemRelease", &d.MemRelease);
        ok &= drv_sym("cuMemAddressReserve", &d.MemAddressReserve);
        ok &= drv_sym("cuMemAddressFree", &d.MemAddressFree);
        ok &= drv_sym("cuMemMap", &d.MemMap);
        ok &= drv_sym("cuMemUnmap", &d.MemUnmap);
        ok &= drv_sym("cuMemSetAccess", &d.MemSetAccess);
        ok &= drv_sym("cuMemExportToShareableHandle", &d.MemExportToShareableHandle);
        ok &= drv_sym("cuMemImportFromShareableHandle", &d.MemImportFromShareableHandle);
        ok &= drv_sym("cuMemGetAllocationGranularity", &d.MemGetAllocationGranularity);
        ok &= drv_sym("cuMulticastCreate", &d.MulticastCreate);
        ok &= drv_sym("cuMulticastAddDevice", &d.MulticastAddDevice);
        ok &= drv_sym("cuMulticastBindMem", &d.MulticastBindMem);
        ok &= drv_sym("cuMulticastGetGranularity", &d.MulticastGetGranularity);
        ok &= drv_sym("cuDeviceGet", &d.DeviceGet);
        ok &= drv_sym("cuDeviceGetAttribute", &d.DeviceGetAttribute);
        ok &= drv_sym("cuGetErrorString", &d.GetErrorString);
        d.ok = ok;
    });
    return d;
}

int drv_fail(const char* what, CUresult r) {
    const char* msg = nullptr;
    if (drv().GetErrorString) drv().GetErrorString(r, &msg);
    return fail(BG_ECUDA, "%s: %s (CUresult %d)", what, msg ? msg : "?", (int)r);
}
#define BG_DRV(expr)                                   \
    do {                                               \
        CUresult _r = (expr);                          \
        if (_r != CUDA_SUCCESS) return drv_fail(#expr, _r); \
    } while (0)

CUmemAllocationProp arena_prop(int device) {
    CUmemAllocationProp prop = {};
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = device;
    prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    return prop;
}

int map_rw(CUdeviceptr* va, size_t bytes, size_t align, CUmemGenericAllocationHandle h, int device) {
    Drv& d = drv();
    BG_DRV(d.MemAddressReserve(va, bytes, align, 0, 0));
    BG_DRV(d.MemMap(*va, bytes, 0, h, 0));
    CUmemAccessDesc acc = {};
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    acc.location.id = device;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    BG_DRV(d.MemSetAccess(*va, bytes, &acc, 1));
    return BG_OK;
}

}  // namespace

extern "C" int bg_abi_version(void) { return BG_ABI_VERSION; }
extern "C" const char* bg_last_error(void) { return g_last_error.c_str(); }
extern "C" unsigned long long bg_launch_count(void) { return g_launches.load(); }

static long long* tunable(const char* name) {
    if (!name) return nullptr;
    if (!strcmp(name, "comm_ctas")) return &g_tun.comm_ctas;
    if (!strcmp(name, "local_ctas")) return &g_tun.local_ctas;
    if (!strcmp(name, "timeout_ms")) return &g_tun.timeout_ms;
    if (!strcmp(name, "oneshot_bytes")) return &g_tun.oneshot_bytes;
    if (!strcmp(name, "nvls_min_bytes")) return &g_tun.nvls_min_bytes;
    if (!strcmp(name, "nvls_min_ranks")) return &g_tun.nvls_min_ranks;
    if (!strcmp(name, "nvls_gather")) return &g_tun.nvls_gather;
    if (!strcmp(name, "nvls_reduce")) return &g_tun.nvls_reduce;
    if (!strcmp(name, "nvls_bcast")) return &g_tun.nvls_bcast;
    return nullptr;
}
extern "C" int bg_set_tunable(const char* name, long long value) {
    long long* t = tunable(name);
    if (!t) return fail(BG_EINVAL, "unknown tunable %s", name ? name : "(null)");
    if (t == &g_tun.comm_ctas && (value < 1 || value > BG_MAX_CHANNELS))
        return fail(BG_EINVAL, "comm_ctas must be in [1,%d]", BG_MAX_CHANNELS);
    const bool flag = t == &g_tun.nvls_gather || t == &g_tun.nvls_reduce || t == &g_tun.nvls_bcast;
    if (value < (flag ? 0 : 1)) return fail(BG_EINVAL, "tunable %s must be positive", name);
    *t = value;
    return BG_OK;
}
extern "C" long long bg_get_tunable(const char* name) {
    long long* t = tunable(name);
    return t ? *t : -1;
}

extern "C" int bg_ctx_create_ex(int rank, int world, int device, size_t arena_bytes, unsigned flags, bg_ctx_t* out) {
    if (!out || world < 1 || world > BG_MAX_WORLD || rank < 0 || rank >= world)
        return fail(BG_EINVAL, "bg_ctx_create: bad rank/world %d/%d", rank, world);
    BG_CUDA(cudaSetDevice(device));
    BG_CUDA(cudaFree(0));   // the primary context exists before any driver-API call
    bg_ctx* c = new bg_ctx();
    c->rank = rank; c->world = world; c->device = device;
    memset(c->peer_base, 0, sizeof(c->peer_base));
    memset(c->peer_ipc, 0, sizeof(c->peer_ipc));
    enumerate_slots(c);
    size_t pad = c->slot_of.size() * kSlotBytes + (size_t)BG_MAX_WORLD * kP2PFlags * 2 * sizeof(uint32_t);
    pad = (pad + 4095) / 4096 * 4096;
    c->pad_bytes = pad;
    c->arena_bytes = pad + ((arena_bytes + 4095) / 4096 * 4096);
    if (flags & BG_CTX_VMM) {
        Drv& d = drv();
        int rc = BG_OK;
        if (!d.ok) rc = fail(BG_ECUDA, "the driver does not expose the virtual-memory / multicast entry points");
        CUmemAllocationProp prop = arena_prop(device);
        size_t gran = 0;
        CUdevice dev = 0;
        if (!rc && d.MemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) != CUDA_SUCCESS)
            rc = fail(BG_ECUDA, "cuMemGetAllocationGranularity failed");
        if (!rc && d.DeviceGet(&dev, device) == CUDA_SUCCESS)
            d.DeviceGetAttribute(&c->mc_supported, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev);
        if (!rc && c->mc_supported) {
            CUmulticastObjectProp mp = {};
            mp.numDevices = world > 1 ? (unsigned)world : 2u;
            mp.size = gran;
            mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
            size_t mg = 0;
            if (d.MulticastGetGranularity(&mg, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && mg) {
                c->mc_gran = mg;
                if (mg > gran) gran = mg;
            } else {
                c->mc_supported = 0;
            }
        }
        if (!rc) {
            c->vmm = true;
            c->vmm_gran = gran;
            c->arena_bytes = (c->arena_bytes + gran - 1) / gran * gran;
            CUresult r = d.MemCreate(&c->arena_handle, c->arena_bytes, &prop, 0);
            if (r != CUDA_SUCCESS) rc = drv_fail("cuMemCreate(arena)", r);
        }
        CUdeviceptr va = 0;
        if (!rc) rc = map_rw(&va, c->arena_bytes, c->vmm_gran, c->arena_handle, device);
        if (rc) { delete c; return rc; }
        c->arena = (char*)va;
    } else {
        cudaError_t e = cudaMalloc(&c->arena, c->arena_bytes);
        if (e != cudaSuccess) {
            size_t want = c->arena_bytes;
            delete c;
            return fail(BG_ENOMEM, "arena cudaMalloc(%zu): %s", want, cudaGetErrorString(e));
        }
    }
    BG_CUDA(cudaMemset(c->arena, 0, pad));
    {   // load every kernel of the library now: a lazily loaded kernel synchronises with the device on its FIRST launch, which
        // must never happen behind a kernel that is waiting for a peer (see bg_preload_coll)
        cudaFuncAttributes attr;
        BG_CUDA(cudaFuncGetAttributes(&attr, reinterpret_cast<const void*>(&barrier_kernel)));
        BG_CUDA(cudaFuncGetAttributes(&attr, reinterpret_cast<const void*>(&p2p_raise_kernel)));
        BG_CUDA(cudaFuncGetAttributes(&attr, reinterpret_cast<const void*>(&p2p_consume_kernel)));
        int rc = bg_preload_coll();
        if (!rc) rc = bg_preload_gemm();
        if (!rc) rc = bg_preload_ops();
        if (rc) { delete c; return rc; }
    }
    BG_CUDA(cudaHostAlloc(&c->err_host, 8 * sizeof(int), cudaHostAllocMapped));   // [0] status, [1..7] who/where
    for (int i = 0; i < 8; ++i) c->err_host[i] = 0;
    BG_CUDA(cudaHostGetDevicePointer(&c->err_dev, c->err_host, 0));
    BG_CUDA(cudaDeviceSynchronize());
    c->bump = pad;
    c->peer_base[rank] = c->arena;
    *out = c;
    return BG_OK;
}

extern "C" int bg_ctx_create(int rank, int world, int device, size_t arena_bytes, bg_ctx_t* out) {
    return bg_ctx_create_ex(rank, world, device, arena_bytes, 0u, out);
}

extern "C" int bg_ctx_destroy(bg_ctx_t c) {
    if (!c) return BG_OK;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    if (c->vmm) {
        Drv& d = drv();
        for (auto& kv : c->mc_of) {
            if (kv.second.va) { d.MemUnmap(kv.second.va, kv.second.bytes); d.MemAddressFree(kv.second.va, kv.second.bytes); }
            if (kv.second.mc) d.MemRelease(kv.second.mc);
        }
        for (int r = 0; r < c->world; ++r)
            if (r != c->rank && c->peer_handle[r]) {
                d.MemUnmap((CUdeviceptr)c->peer_base[r], c->arena_bytes);
                d.MemAddressFree((CUdeviceptr)c->peer_base[r], c->arena_bytes);
                d.MemRelease(c->peer_handle[r]);
            }
        if (c->arena) { d.MemUnmap((CUdeviceptr)c->arena, c->arena_bytes); d.MemAddressFree((CUdeviceptr)c->arena, c->arena_bytes); }
        if (c->arena_handle) d.MemRelease(c->arena_handle);
    } else {
        for (int r = 0; r < c->world; ++r)
            if (c->peer_ipc[r] && c->peer_base[r]) cudaIpcCloseMemHandle(c->peer_base[r]);
        if (c->arena) cudaFree(c->arena);
    }
    if (c->err_host) cudaFreeHost(c->err_host);
    for (auto e : c->events) cudaEventDestroy(e);
    delete c;
    return BG_OK;
}

extern "C" int bg_arena_info(bg_ctx_t c, void** base, size_t* bytes, size_t* used) {
    if (!c) return fail(BG_EINVAL, "null ctx");
    if (base) *base = c->arena;
    if (bytes) *bytes = c->arena_bytes;
    if (used) *used = c->bump;
    return BG_OK;
}

extern "C" int bg_arena_alloc(bg_ctx_t c, size_t bytes, size_t* offset) {
    if (!c || !offset) return fail(BG_EINVAL, "null arg");
    std::lock_guard<std::mutex> lk(c->mu);
    size_t off = (c->bump + 255) / 256 * 256;
    if (off + bytes > c->arena_bytes)
        return fail(BG_ENOMEM, "arena exhausted: want %zu at %zu of %zu (raise arena_bytes)", bytes, off, c->arena_bytes);
    c->bump = off + bytes;
    *offset = off;
    return BG_OK;
}

extern "C" int bg_arena_alloc_aligned(bg_ctx_t c, size_t bytes, size_t align, size_t* offset) {
    if (!c || !offset || !align) return fail(BG_EINVAL, "null arg");
    std::lock_guard<std::mutex> lk(c->mu);
    size_t off = (c->bump + align - 1) / align * align;
    if (off + bytes > c->arena_bytes)
        return fail(BG_ENOMEM, "arena exhausted: want %zu at %zu of %zu (raise arena_bytes)", bytes, off, c->arena_bytes);
    c->bump = off + bytes;
    *offset = off;
    return BG_OK;
}

extern "C" int bg_arena_mode(bg_ctx_t c, int* vmm, int* multicast, size_t* mc_granularity) {
    if (!c) return fail(BG_EINVAL, "null ctx");
    if (vmm) *vmm = c->vmm ? 1 : 0;
    if (multicast) *multicast = c->vmm ? c->mc_supported : 0;
    if (mc_granularity) *mc_granularity = c->mc_gran;
    return BG_OK;
}

extern "C" int bg_arena_export_fd(bg_ctx_t c, int* fd) {
    if (!c || !fd) return fail(BG_EINVAL, "null arg");
    if (!c->vmm) return fail(BG_EINVAL, "bg_arena_export_fd needs a BG_CTX_VMM context (cudaMalloc arenas use bg_arena_export)");
    BG_CUDA(cudaSetDevice(c->device));
    BG_DRV(drv().MemExportToShareableHandle(fd, c->arena_handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
    return BG_OK;
}

extern "C" int bg_arena_import_fd(bg_ctx_t c, int peer, int fd) {
    if (!c || peer < 0 || peer >= c->world || fd < 0) return fail(BG_EINVAL, "bad peer %d / fd %d", peer, fd);
    if (!c->vmm) return fail(BG_EINVAL, "bg_arena_import_fd needs a BG_CTX_VMM context");
    if (peer == c->rank) return BG_OK;
    BG_CUDA(cudaSetDevice(c->device));
    Drv& d = drv();
    BG_DRV(d.MemImportFromShareableHandle(&c->peer_handle[peer], (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
    CUdeviceptr va = 0;
    int rc = map_rw(&va, c->arena_bytes, c->vmm_gran, c->peer_handle[peer], c->device);   // every rank's arena has the same size
    if (rc) return rc;
    c->peer_base[peer] = (char*)va;
    return BG_OK;
}

extern "C" int bg_arena_export(bg_ctx_t c, void* handle64) {
    if (!c || !handle64) return fail(BG_EINVAL, "null arg");
    if (c->vmm) return fail(BG_EINVAL, "a BG_CTX_VMM arena is shared with bg_arena_export_fd");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    BG_CUDA(cudaSetDevice(c->device));
    BG_CUDA(cudaIpcGetMemHandle((cudaIpcMemHandle_t*)handle64, c->arena));
    return BG_OK;
}

extern "C" int bg_arena_import(bg_ctx_t c, int peer, const void* handle64) {
    if (!c || !handle64 || peer < 0 || peer >= c->world) return fail(BG_EINVAL, "bad peer %d", peer);
    if (peer == c->rank) return BG_OK;
    BG_CUDA(cudaSetDevice(c->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, sizeof(h));
    void* p = nullptr;
    BG_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    c->peer_base[peer] = (char*)p;
    c->peer_ipc[peer] = true;
    return BG_OK;
}

extern "C" int bg_arena_attach_local(bg_ctx_t c, int peer, bg_ctx_t other) {
    if (!c || !other || peer < 0 || peer >= c->world) return fail(BG_EINVAL, "bad peer %d", peer);
    if (other->device != c->device) {
        int can = 0;
        BG_CUDA(cudaDeviceCanAccessPeer(&can, c->device, other->device));
        if (!can) return fail(BG_ENOTMAPPED, "device %d cannot access %d", c->device, other->device);
        BG_CUDA(cudaSetDevice(c->device));
        cudaError_t e = cudaDeviceEnablePeerAccess(other->device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
            return fail(BG_ECUDA, "enable peer access: %s", cudaGetErrorString(e));
        cudaGetLastError();
    }
    c->peer_base[peer] = other->arena;
    return BG_OK;
}

extern "C" int bg_ctx_error_flag(bg_ctx_t c, int* flag) {
    if (!c || !flag) return fail(BG_EINVAL, "null arg");
    *flag = *c->err_host;
    return BG_OK;
}

extern "C" int bg_ctx_error_info(bg_ctx_t c, int* info8) {
    if (!c || !info8) return fail(BG_EINVAL, "null arg");
    for (int i = 0; i < 8; ++i) info8[i] = c->err_host[i];   // mapped host memory: readable after a device trap
    return BG_OK;
}

// ------------------------------------------------------------------------------------------------
// groups
// ------------------------------------------------------------------------------------------------
extern "C" int bg_group_create(bg_ctx_t c, const int* ranks, int n, int* gid) {
    if (!c || !ranks || !gid || n < 1) return fail(BG_EINVAL, "bg_group_create: bad args");
    if (n > BG_MAX_PEERS) return fail(BG_EGROUP, "group of %d ranks exceeds one NVSwitch domain (%d)", n, BG_MAX_PEERS);
    std::vector<int> key(ranks, ranks + n);
    std::lock_guard<std::mutex> lk(c->mu);
    auto it = c->gid_of.find(key);
    if (it != c->gid_of.end()) { *gid = it->second; return BG_OK; }
    Group g;
    g.n = n;
    for (int i = 0; i < n; ++i) {
        if (ranks[i] < 0 || ranks[i] >= c->world) return fail(BG_EGROUP, "rank %d outside world %d", ranks[i], c->world);
        if (i && ranks[i] <= ranks[i - 1]) return fail(BG_EGROUP, "rank list must be strictly increasing");
        g.ranks[i] = ranks[i];
        if (ranks[i] == c->rank) g.me = i;
    }
    if (g.me < 0) return fail(BG_EGROUP, "calling rank %d is not a member", c->rank);
    if (n >= 2) {
        int stride = ranks[1] - ranks[0];
        for (int i = 2; i < n; ++i)
            if (ranks[i] - ranks[i - 1] != stride) return fail(BG_EGROUP, "rank list is not an arithmetic progression");
        auto s = c->slot_of.find(std::make_tuple(ranks[0], stride, n));
        if (s == c->slot_of.end()) return fail(BG_EGROUP, "no signal slot for group");
        g.slot = s->second;
    }
    c->groups.push_back(g);
    *gid = (int)c->groups.size() - 1;
    c->gid_of[key] = *gid;
    return BG_OK;
}

extern "C" int bg_group_info(bg_ctx_t c, int gid, int* n, int* my_index, int* ranks_out) {
    if (!c || gid < 0 || gid >= (int)c->groups.size()) return fail(BG_EGROUP, "bad gid %d", gid);
    const Group& g = c->groups[gid];
    if (n) *n = g.n;
    if (my_index) *my_index = g.me;
    if (ranks_out) for (int i = 0; i < g.n; ++i) ranks_out[i] = g.ranks[i];
    return BG_OK;
}

// C mirror of the closed-form membership rules (comm_groups.py:71-236,382-409) for the bit-exact check
static int put_range(int* counts, int* ranks, int first, int stop, int step) {
    int k = 0;
    for (int r = first; r < stop; r += step) ranks[k++] = r;
    *counts = k;
    return k;
}
extern "C" int bg_build_groups(int rank, int world, int pp, int n_layers, const int* tp, const int* sp, const int* cp,
                               int* out_counts, int* out_ranks, int* pp_count, int* pp_ranks) {
    if (world < 1 || world > BG_MAX_WORLD || pp < 1 || world % pp || rank < 0 || rank >= world)
        return fail(BG_EINVAL, "bg_build_groups: bad world/pp/rank");
    const int per_stage = world / pp, base = rank / per_stage * per_stage, local = rank - base;
    for (int i = 0; i < n_layers; ++i) {
        const int t = tp[i], s = sp[i], c = cp[i], mul = t * s;
        if (t < 1 || s < 1 || c < 1 || (t != 1 && s != 1) || per_stage % (mul * c))
            return fail(BG_EINVAL, "layer %d: invalid tp/sp/cp %d/%d/%d", i, t, s, c);
        auto cnt = [&](int kind) { return out_counts + kind * n_layers + i; };
        auto rk = [&](int kind) { return out_ranks + ((size_t)kind * n_layers + i) * BG_MAX_WORLD; };
        put_range(cnt(0), rk(0), rank / t * t, rank / t * t + t, 1);                                   // tp
        put_range(cnt(1), rk(1), rank / s * s, rank / s * s + s, 1);                                   // sp
        int first = base + local / (mul * c) * (mul * c) + local % mul;
        put_range(cnt(2), rk(2), first, first + mul * c, mul);                                         // cp
        put_range(cnt(3), rk(3), base + local % (mul * c), base + per_stage, mul * c);                 // dp
        if (t == 1) put_range(cnt(4), rk(4), base, base + per_stage, 1);                               // sdp
        else put_range(cnt(4), rk(4), base + local % t, base + per_stage, t);
    }
    put_range(pp_count, pp_ranks, rank % per_stage, world, per_stage);
    return BG_OK;
}


int make_sig(bg_ctx* c, int gid, int lane, Sig* s, const Group** gout) {
    if (!c) return fail(BG_EINVAL, "null ctx");
    if (gid < 0 || gid >= (int)c->groups.size()) return fail(BG_EGROUP, "bad gid %d", gid);
    if (lane < 0 || lane >= BG_LANES) return fail(BG_EINVAL, "bad lane %d", lane);
    const Group& g = c->groups[gid];
    s->me = g.me; s->n = g.n;
    s->timeout_ns = (unsigned long long)g_tun.timeout_ms * 1000000ull;
    s->err = c->err_dev;
    s->site = 0;
    s->local = nullptr;
    for (int i = 0; i < BG_MAX_PEERS; ++i) s->peer[i] = nullptr;
    if (g.n > 1) {
        size_t off = (size_t)g.slot * kSlotBytes + (size_t)lane * BG_MAX_CHANNELS * BG_MAX_PEERS * sizeof(uint32_t);
        for (int i = 0; i < g.n; ++i) {
            char* base = c->peer_base[g.ranks[i]];
            if (!base) return fail(BG_ENOTMAPPED, "arena of rank %d is not mapped (bg_arena_import)", g.ranks[i]);
            s->peer[i] = (uint32_t*)(base + off);
        }
        s->local = s->peer[g.me];
    }
    if (gout) *gout = &g;
    return BG_OK;
}

int resolve(bg_ctx* c, const Group& g, const size_t* offs, size_t bytes, PeerPtrs* out) {
    if (!offs) return fail(BG_EINVAL, "null symmetric-offset array");
    for (int i = 0; i < BG_MAX_PEERS; ++i) out->p[i] = nullptr;
    for (int i = 0; i < g.n; ++i) {
        char* base = c->peer_base[g.ranks[i]];
        if (!base) return fail(BG_ENOTMAPPED, "arena of rank %d is not mapped", g.ranks[i]);
        if (offs[i] % 16) return fail(BG_EINVAL, "symmetric offset %zu not 16-B aligned", offs[i]);
        // (written so that no sum can wrap around: a huge `bytes` must not pass as a small one)
        if (offs[i] < c->pad_bytes || bytes > c->arena_bytes || offs[i] > c->arena_bytes - bytes)
            return fail(BG_EINVAL, "symmetric buffer [%zu,+%zu) outside arena", offs[i], bytes);
        out->p[i] = base + offs[i];
    }
    return BG_OK;
}

char* mc_ptr(bg_ctx* c, int gid, const Group& g, const size_t* offs, size_t bytes) {
    if (!c->vmm || g.n < 2 || g.n < g_tun.nvls_min_ranks || !offs) return nullptr;
    auto it = c->mc_of.find(gid);
    if (it == c->mc_of.end() || !it->second.bound) return nullptr;
    const bg_ctx::McGroup& m = it->second;
    for (int i = 1; i < g.n; ++i)
        if (offs[i] != offs[0]) return nullptr;
    if (offs[0] < m.arena_off || offs[0] + bytes > m.arena_off + m.bytes) return nullptr;
    return (char*)m.va + (offs[0] - m.arena_off);
}

int comm_grid(size_t work_items, int threads, int n) {
    long long cap = n == 1 ? g_tun.local_ctas : g_tun.comm_ctas;
    long long want = (long long)((work_items + threads - 1) / threads);
    if (want < 1) want = 1;
    return (int)(want < cap ? want : cap);
}

static __global__ void barrier_kernel(Sig s) { sync_peers<true, true, true>(s); }

extern "C" int bg_barrier(bg_ctx_t c, int gid, int lane, void* stream) {
    Sig s;
    int rc = make_sig(c, gid, lane, &s, nullptr);
    if (rc) return rc;
    BG_CUDA(cudaSetDevice(c->device));
    if (s.n == 1) return BG_OK;
    barrier_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(s);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

// ------------------------------------------------------------------------------------------------
// C11: pipeline p2p -- peer copy on the caller's (side) stream + device flags, no device-wide sync.
// Flags in every arena: F[other_rank][flag_id][2]; [0] "a message from other has landed here",
// [1] "other has consumed the message I sent".  A sender re-uses a slot only after the receiver's ack.
// ------------------------------------------------------------------------------------------------
__global__ void p2p_raise_kernel(uint32_t* flag, unsigned long long timeout_ns, int* err) {
    __threadfence_system();
    Sig s; s.timeout_ns = timeout_ns; s.err = err; s.me = -1; s.n = 0; s.site = 10;
    sig_spin_cas(flag, 0u, 1u, true, s);
}
__global__ void p2p_consume_kernel(uint32_t* flag, unsigned long long timeout_ns, int* err) {
    Sig s; s.timeout_ns = timeout_ns; s.err = err; s.me = -1; s.n = 0; s.site = 11;
    sig_spin_cas(flag, 1u, 0u, false, s);
}

static uint32_t* p2p_flag(bg_ctx* c, int owner_rank, int other_rank, int flag_id, int which) {
    char* base = c->peer_base[owner_rank];
    if (!base) return nullptr;
    size_t off = c->slot_of.size() * kSlotBytes + (((size_t)other_rank * kP2PFlags + flag_id) * 2 + which) * sizeof(uint32_t);
    return (uint32_t*)(base + off);
}

static int p2p_args(bg_ctx* c, int peer, int flag_id, const char* who) {
    if (!c || peer < 0 || peer >= c->world || peer == c->rank || flag_id < 0 || flag_id >= kP2PFlags)
        return fail(BG_EINVAL, "%s: bad peer/flag %d/%d", who, peer, flag_id);
    if (!c->peer_base[peer]) return fail(BG_ENOTMAPPED, "arena of rank %d is not mapped", peer);
    return BG_OK;
}

extern "C" int bg_p2p_send(bg_ctx_t c, int peer, size_t dst_off, const void* src, size_t bytes, int flag_id, void* stream) {
    int rc = p2p_args(c, peer, flag_id, "bg_p2p_send");
    if (rc) return rc;
    if (dst_off < c->pad_bytes || dst_off + bytes > c->arena_bytes) return fail(BG_EINVAL, "p2p destination outside arena");
    BG_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned long long to = (unsigned long long)g_tun.timeout_ms * 1000000ull;
    bool first;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        first = c->p2p_sent[peer][flag_id]++ == 0;
    }
    if (!first) {  // the receiver must have released the slot (bg_p2p_release) before it is overwritten
        p2p_consume_kernel<<<1, 1, 0, st>>>(p2p_flag(c, c->rank, peer, flag_id, 1), to, c->err_dev);
        BG_CHECK_LAUNCH();
    }
    if (bytes) BG_CUDA(cudaMemcpyAsync(c->peer_base[peer] + dst_off, src, bytes, cudaMemcpyDeviceToDevice, st));
    p2p_raise_kernel<<<1, 1, 0, st>>>(p2p_flag(c, peer, c->rank, flag_id, 0), to, c->err_dev);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_p2p_wait(bg_ctx_t c, int peer, int flag_id, void* stream) {
    int rc = p2p_args(c, peer, flag_id, "bg_p2p_wait");
    if (rc) return rc;
    BG_CUDA(cudaSetDevice(c->device));
    p2p_consume_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(p2p_flag(c, c->rank, peer, flag_id, 0),
                                                          (unsigned long long)g_tun.timeout_ms * 1000000ull, c->err_dev);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_p2p_release(bg_ctx_t c, int peer, int flag_id, void* stream) {
    int rc = p2p_args(c, peer, flag_id, "bg_p2p_release");
    if (rc) return rc;
    BG_CUDA(cudaSetDevice(c->device));
    p2p_raise_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(p2p_flag(c, peer, c->rank, flag_id, 1),
                                                        (unsigned long long)g_tun.timeout_ms * 1000000ull, c->err_dev);
    BG_CHECK_LAUNCH();
    return BG_OK;
}
// ---- NVLS: multicast object over one group's symmetric buffer ---------------------------------------------------------
static int mc_group(bg_ctx* c, int gid, const Group** gout) {
    if (!c) return fail(BG_EINVAL, "null ctx");
    if (gid < 0 || gid >= (int)c->groups.size()) return fail(BG_EGROUP, "bad gid %d", gid);
    if (!c->vmm || !c->mc_supported) return fail(BG_EINVAL, "NVLS needs a BG_CTX_VMM context on a multicast-capable device");
    *gout = &c->groups[gid];
    if ((*gout)->n < 2) return fail(BG_EINVAL, "NVLS needs a group of >= 2 ranks");
    return BG_OK;
}

extern "C" int bg_group_mc_create(bg_ctx_t c, int gid, size_t bytes, int* fd_out) {
    const Group* g;
    int rc = mc_group(c, gid, &g);
    if (rc) return rc;
    if (!fd_out || !bytes) return fail(BG_EINVAL, "null arg");
    BG_CUDA(cudaSetDevice(c->device));
    bg_ctx::McGroup& m = c->mc_of[gid];
    if (m.mc) return fail(BG_EINVAL, "group %d already has a multicast object", gid);
    CUmulticastObjectProp mp = {};
    mp.numDevices = (unsigned)g->n;
    mp.size = (bytes + c->mc_gran - 1) / c->mc_gran * c->mc_gran;
    mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    BG_DRV(drv().MulticastCreate(&m.mc, &mp));
    m.bytes = mp.size;
    BG_DRV(drv().MemExportToShareableHandle(fd_out, m.mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
    return BG_OK;
}

// fd >= 0: import the creator's object (every other member); then add this rank's device.  ALL members must have joined
// before any of them binds (host-side barrier).
extern "C" int bg_group_mc_join(bg_ctx_t c, int gid, int fd, size_t bytes) {
    const Group* g;
    int rc = mc_group(c, gid, &g);
    if (rc) return rc;
    BG_CUDA(cudaSetDevice(c->device));
    bg_ctx::McGroup& m = c->mc_of[gid];
    if (fd >= 0) {
        if (m.mc) return fail(BG_EINVAL, "group %d already has a multicast object", gid);
        BG_DRV(drv().MemImportFromShareableHandle(&m.mc, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
        m.bytes = (bytes + c->mc_gran - 1) / c->mc_gran * c->mc_gran;
    }
    if (!m.mc) return fail(BG_EINVAL, "group %d has no multicast object (create or import first)", gid);
    CUdevice dev = 0;
    BG_DRV(drv().DeviceGet(&dev, c->device));
    BG_DRV(drv().MulticastAddDevice(m.mc, dev));
    return BG_OK;
}

extern "C" int bg_group_mc_disable(bg_ctx_t c, int gid) {
    if (!c) return fail(BG_EINVAL, "null ctx");
    auto it = c->mc_of.find(gid);
    if (it != c->mc_of.end()) it->second.bound = false;      // collectives of this group keep the peer-to-peer kernels
    return BG_OK;
}

extern "C" int bg_group_mc_bind(bg_ctx_t c, int gid, size_t arena_offset) {
    const Group* g;
    int rc = mc_group(c, gid, &g);
    if (rc) return rc;
    BG_CUDA(cudaSetDevice(c->device));
    bg_ctx::McGroup& m = c->mc_of[gid];
    if (!m.mc || m.bound) return fail(BG_EINVAL, "group %d: multicast object missing or already bound", gid);
    if (arena_offset % c->mc_gran || arena_offset < c->pad_bytes || arena_offset + m.bytes > c->arena_bytes)
        return fail(BG_EINVAL, "NVLS buffer [%zu,+%zu) must be multicast-granularity (%zu) aligned inside the arena", arena_offset, m.bytes,
                    c->mc_gran);
    BG_DRV(drv().MulticastBindMem(m.mc, 0, c->arena_handle, arena_offset, m.bytes, 0));
    rc = map_rw(&m.va, m.bytes, c->mc_gran, m.mc, c->device);
    if (rc) return rc;
    m.arena_off = arena_offset;
    m.bound = true;
    return BG_OK;
}

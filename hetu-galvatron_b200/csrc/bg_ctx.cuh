// bg_ctx.cuh -- the per-rank context, groups, peer-pointer tables and the device-side cross-rank barrier shared by
// bg_comm.cu (arena / groups / p2p / multicast setup) and bg_coll.cu (the collective kernels).
#pragma once
#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include <cuda.h>

#include "bg_common.cuh"

struct Group {
    int n = 0, me = -1, slot = -1;
    int ranks[BG_MAX_PEERS];
};

struct bg_ctx {
    int rank = 0, world = 1, device = 0;
    char* arena = nullptr;
    size_t arena_bytes = 0, bump = 0, pad_bytes = 0;
    char* peer_base[BG_MAX_WORLD];
    bool peer_ipc[BG_MAX_WORLD];
    std::vector<Group> groups;
    std::map<std::vector<int>, int> gid_of;
    std::map<std::tuple<int, int, int>, int> slot_of;  // (first, stride, size) -> signal slot
    int* err_host = nullptr;                            // mapped pinned: device-side timeout report
    int* err_dev = nullptr;
    unsigned long long p2p_sent[BG_MAX_WORLD][64] = {};
    std::mutex mu;
    std::vector<cudaEvent_t> events;                    // ring used to order the compute and communication streams of fused ops
    size_t event_i = 0;
    // ---- VMM arena / NVLS multicast (opt-in) ----
    bool vmm = false;
    int mc_supported = 0;
    size_t vmm_gran = 0, mc_gran = 0;
    CUmemGenericAllocationHandle arena_handle = 0;
    CUmemGenericAllocationHandle peer_handle[BG_MAX_WORLD] = {};
    struct McGroup {
        CUmemGenericAllocationHandle mc = 0;
        CUdeviceptr va = 0;
        size_t bytes = 0, arena_off = 0;
        bool bound = false;
    };
    std::map<int, McGroup> mc_of;   // gid -> multicast object over the group's NVLS buffer
};

// signal pad: pad[slot][lane][channel][BG_MAX_PEERS] u32, followed by the p2p flags [BG_MAX_WORLD][P2P_FLAGS]
static constexpr size_t kSlotBytes = (size_t)BG_LANES * BG_MAX_CHANNELS * BG_MAX_PEERS * sizeof(uint32_t);
static constexpr int kP2PFlags = 64;

// ------------------------------------------------------------------------------------------------
// device-side cross-rank barrier (per CTA channel): CAS put 0->1 on the peer, CAS wait 1->0 locally
// ------------------------------------------------------------------------------------------------
struct Sig {
    uint32_t* local;               // my pad for (slot, lane): [channel][BG_MAX_PEERS]
    uint32_t* peer[BG_MAX_PEERS];  // the same region in every member's arena
    int me, n;
    unsigned long long timeout_ns;
    int* err;
    int site;                      // which kernel family launched with this Sig (goes into the timeout record, info8[7])
};

struct PeerPtrs {
    char* p[BG_MAX_PEERS];
};

__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ void sig_spin_cas(uint32_t* addr, uint32_t expect, uint32_t desired, bool release,
                                             const Sig& s) {
    unsigned long long t0 = 0;
    unsigned spins = 0;
    while (true) {
        uint32_t old;
        if (release)
            asm volatile("atom.global.release.sys.cas.b32 %0, [%1], %2, %3;" : "=r"(old) : "l"(addr), "r"(expect), "r"(desired) : "memory");
        else
            asm volatile("atom.global.acquire.sys.cas.b32 %0, [%1], %2, %3;" : "=r"(old) : "l"(addr), "r"(expect), "r"(desired) : "memory");
        if (old == expect) return;
        if ((++spins & 0xff) == 0) {
            unsigned long long now = gtimer();
            if (t0 == 0) t0 = now;
            else if (now - t0 > s.timeout_ns) {
                // who/where: kind 1 = signal a peer (its flag never drained), 2 = wait for a peer's signal
                if (atomicCAS(s.err + 1, 0, release ? 1 : 2) == 0) {
                    s.err[2] = (int)blockIdx.x; s.err[3] = (int)threadIdx.x; s.err[4] = (int)old; s.err[5] = s.me; s.err[6] = s.n; s.err[7] = s.site;
                }
                *s.err = BG_ETIMEOUT;
                __threadfence_system();
                __trap();
            }
        }
    }
}

// All threads of the CTA call this.
//   kSyncBefore: the whole CTA must have finished its prior loads/stores before the signal is raised
//   kFence:      this CTA wrote data that peers read after the barrier (make it visible at .sys scope)
//   kSyncAfter:  the whole CTA must wait for the barrier before continuing
template <bool kSyncBefore, bool kFence, bool kSyncAfter>
__device__ __forceinline__ void sync_peers(const Sig& s) {
    if (s.n == 1) return;
    if (kFence) __threadfence_system();
    if (kSyncBefore) __syncthreads();
    const int t = threadIdx.x;
    if (t < s.n && t != s.me) {
        sig_spin_cas(s.peer[t] + blockIdx.x * BG_MAX_PEERS + s.me, 0u, 1u, true, s);
        sig_spin_cas(s.local + blockIdx.x * BG_MAX_PEERS + t, 1u, 0u, false, s);
    }
    if (kSyncAfter) __syncthreads();
}

int make_sig(bg_ctx* c, int gid, int lane, Sig* s, const Group** gout);
int resolve(bg_ctx* c, const Group& g, const size_t* offs, size_t bytes, PeerPtrs* out);
int comm_grid(size_t work_items, int threads, int n);
// multicast (NVLS) address of a symmetric buffer: non-null when the group has a bound multicast region that covers
// [offs[i], offs[i]+bytes) and every member placed the buffer at the same arena offset
char* mc_ptr(bg_ctx* c, int gid, const Group& g, const size_t* offs, size_t bytes);

// Fused GEMM + collective kernels (bg_gemm.cu).  The tensor maps are encoded by *_maps before the entry point (bg_coll.cu)
// launches anything -- its entry barrier or push kernel -- so an operand the encoder rejects fails the call with no work queued
// and no peer left waiting.  *_launch then only launches.
struct FusedGemmMaps {
    CUtensorMap a, b, c;               // reduce-scatter: c unused; all-gather: a = the staging buffer [M][K]
    CUtensorMap peer[BG_MAX_PEERS];    // reduce-scatter: owner i's partial buffer; all-gather: peer[0] = the local shard
};
int bg_gemm_scatter_maps(FusedGemmMaps* maps, const void* a, const void* b, long long m, long long n, long long k, int layout, int p,
                         void* const* partial_ptrs);
int bg_gemm_scatter_launch(const FusedGemmMaps& maps, long long m, long long n, long long k, int layout, int p, int me,
                           void* const* partial_ptrs, uint32_t* const* flag_ptrs, void* out, void* const* bcast_ptrs, char* bcast_mc,
                           unsigned long long timeout_ns, int* err_dev, cudaStream_t st);
int bg_gemm_gather_maps(FusedGemmMaps* maps, const void* a_local, const void* a_staged, const void* b, void* c, long long m, long long n,
                        long long k, int layout, int p);
int bg_gemm_gather_launch(const FusedGemmMaps& maps, long long m, long long n, long long k, int layout, int p, int me,
                          const uint32_t* flags, uint32_t target, unsigned long long timeout_ns, int* err_dev, cudaStream_t st);

// bg_gemm.cu -- K1: bf16 GEMM on the Hopper tensor cores (wgmma.mma_async, fp32 accumulators in registers, operands staged
// by TMA with 128-B swizzle), persistent, warp-specialised.  Replaces the torch.matmul -> cuBLAS calls of
// galvatron/site_package/megatron/core/tensor_parallel/layers.py:417 (fwd), :462 (dgrad), :534 (wgrad).
//
//   tile            : BLOCK_M 128 x (128 | 256) x BLOCK_K 64, one CTA per SM; two consumer warpgroups, each issuing
//                     wgmma m64n128k16 (64 fp32 accumulators per thread) or m64n256k16 (128) on its 64 rows of the tile.
//                     The plain GEMM runs 256-wide tiles for N > 128 (half the shared-memory operand reads per FLOP of
//                     the 128-wide tile); the fused modes and plain GEMMs of N <= 128 run 128-wide tiles.
//   smem pipeline   : 128-wide: 5 stages x (A 16 KiB + B 16 KiB); 256-wide: 4 stages x (A 16 KiB + B 32 KiB);
//                     full/empty mbarriers (TMA <-> wgmma)
//   warps           : 0-7 = the two consumer warpgroups (wgmma, then the epilogue: registers -> swizzled smem -> TMA store),
//                     8 = TMA producer; 288 threads.  The producer fills the stages of the next tile while the consumers run
//                     the epilogue of this one.
//   residency       : slim collective CTAs (128 threads x 64 registers, no shared memory, bg_coll.cu) stay resident beside
//                     a running GEMM CTA: three beside a 128-wide CTA (<= 136 registers per thread, 193 KiB of shared
//                     memory), which every kernel that waits on peers needs; two beside a 256-wide plain CTA (<= 168
//                     registers, 209 KiB), which waits on nothing and always retires (DESIGN section 2)
//   layouts         : TN  C = A[M,K] * B[N,K]^T   (A, B K-major)
//                     NN  C = A[M,K] * B[K,N]     (B MN-major: TMA boxes of 64 N-elements x 64 K-rows)
//                     NT  C = A[K,M]^T * B[K,N]   (A, B MN-major)
//   edges           : TMA zero-fills out-of-bounds loads and clips stores, so M, N, K only need to be multiples of 8.
#include <stdlib.h>

#include "bg_ctx.cuh"

using namespace bg;

namespace {

constexpr int BLOCK_M = 128, BLOCK_N = 128, BLOCK_K = 64, WGMMA_K = 16;   // BLOCK_N: the fused modes' tile width
constexpr int WIDE_N = 256;                                    // the plain GEMM's tile width for N > BLOCK_N
constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
constexpr int kStoreCols = 64;                                 // columns per TMA store box (128 B)
constexpr int kStoreBytes = BLOCK_M * kStoreCols * 2;          // 16 KiB per staging buffer
constexpr int kEpiThreads = 256, kThreads = kEpiThreads + 32;  // two consumer warpgroups + one producer warp
constexpr int kProducerWarp = kEpiThreads / 32;
constexpr int kWgOffset = 8192;  // smem offset of consumer warpgroup 1's operand A: 64 K-major rows, or the 2nd 64-wide M chunk
constexpr int kGroupM = 16;      // tile raster of the fused modes: 16 m-blocks share each sweep over n (L2 reuse)

// Pipeline and residency of one tile width.  A kernel that waits on peers (the fused modes, every collective) must always be
// resident beside one CTA of each other collective that can be in flight: a 128-wide GEMM CTA leaves room for three slim
// CTAs.  A 256-wide plain GEMM CTA leaves room for two: it waits on nothing after launch, so a third collective CTA that
// cannot become resident beside it waits at most until it retires, and no cycle of waits passes through it.
template <int kBlockN>
struct Tile {
    static constexpr bool kWide = kBlockN == WIDE_N;
    static constexpr int kStages = kWide ? 4 : 5;
    static constexpr int kNumStoreBufs = kWide ? 1 : 2;
    static constexpr int kMaxRegs = kWide ? 168 : 136;         // 128 (64) fp32 accumulators per consumer thread
    static constexpr int kSlimCtas = kWide ? 2 : 3;
    static constexpr int kBBytes = kBlockN * BLOCK_K * 2, kStageBytes = kABytes + kBBytes;
    static constexpr int kSmemBytes = kStages * kStageBytes + kNumStoreBufs * kStoreBytes + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(kBlockN == BLOCK_N || kBlockN == WIDE_N, "tile width 128 or 256");
    static_assert(kSmemBytes <= 227 * 1024, "H100: at most 227 KiB of shared memory per block");
    static_assert(kThreads * kMaxRegs + kSlimCtas * 128 * 64 <= 65536, "a GEMM CTA and its slim collective CTAs share an SM's registers");
    // H100: 228 KiB of shared memory per SM, of which the driver reserves 1 KiB per resident CTA (also for a CTA that uses none)
    static_assert(kSmemBytes + 1024 + kSlimCtas * 1024 <= 228 * 1024, "a GEMM CTA and its slim collective CTAs share an SM's shared memory");
};
template struct Tile<BLOCK_N>;
template struct Tile<WIDE_N>;

enum Layout { kTN = 0, kNN = 1, kNT = 2 };

// ---- PTX wrappers ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(map), "r"(src), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kEpiThreads) : "memory"); }
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching the accumulators across an asynchronous wgmma (register dependences only)
template <int kNumAcc>
__device__ __forceinline__ void fence_acc(float* d) {
#pragma unroll
    for (int i = 0; i < kNumAcc; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] (+)= A[64 x 16] * B[16 x 128], both operands in shared memory; kTransA / kTransB = 1 for an MN-major operand
template <int kTransA, int kTransB>
__device__ __forceinline__ void wgmma_m64n128(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(kTransA), "n"(kTransB));
}

// D[64 x 256] (+)= A[64 x 16] * B[16 x 256]: as above, 128 accumulators per thread
template <int kTransA, int kTransB>
__device__ __forceinline__ void wgmma_m64n256(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, %131, %132;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(kTransA), "n"(kTransB));
}

// wgmma shared-memory matrix descriptor (cute::GMMA::GmmaDescriptor bit layout): start[0,14) lbo[16,30) sbo[32,46)
// base_offset[49,52)=0 (stages are 1024-B aligned) layout_type[62,64) (1 = SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

struct TileCoord { int m, n; };
// kMode: which collective is fused into the GEMM
enum { kPlain = 0, kScatterMode = 1, kGatherMode = 2 };

template <int kMode>
struct FuseParams {};

// Plain GEMM: how many m-blocks share each sweep over n (chosen per shape on the host, gemm_launch)
template <>
struct FuseParams<kPlain> {
    int group_m;
};

__device__ __forceinline__ TileCoord tile_of_virtual(int t, int m_blocks, int n_blocks, int group_m) {
    const int per_group = group_m * n_blocks;
    const int g = t / per_group, first_m = g * group_m;
    const int rows = min(group_m, m_blocks - first_m);
    const int r = t - g * per_group;
    return {first_m + r % rows, r / rows};
}

// Fused GEMM + reduce-scatter (C5/C8): instead of storing C locally, the epilogue TMA-stores every finished 128x128 partial
// tile straight into the HBM of the rank that owns those rows (peer store over NVLink) and bumps that rank's per-tile
// arrival counter; a small reducer kernel on the owner sums the p partials of a tile as soon as all have landed.  Transfer and
// math overlap tile by tile; no NCCL, no separate collective pass over the full activation.
template <>
struct FuseParams<kScatterMode> {
    CUtensorMap dst[BG_MAX_PEERS];      // owner o's partial buffer viewed as [p * rows_per_rank][N] (block r = source rank r)
    uint32_t* flags[BG_MAX_PEERS];      // owner o's arrival counters, one per local tile
    int p, me, rows_per_rank;
};

// Fused all-gather + GEMM (C7): A[M,K] is the concatenation of the members' [M/p, K] shards.  The rank's own rows are read
// from its local shard; every other 128-row block is read from the staging slot the owner's push kernel fills, as soon as that
// block's arrival counter shows all pushing CTAs have delivered it.  Blocks are walked in arrival order: block c of slot me,
// me+1, ..., me-1, then block c+1 of every slot, so the first sweep over N needs only the first block of every slot.
template <>
struct FuseParams<kGatherMode> {
    CUtensorMap a_local;                // [M/p][K]
    const uint32_t* flags;              // [p][blocks_per_rank] arrival counters in THIS rank's arena
    uint32_t target;                    // CTAs of the push kernel
    int p, me, blocks_per_rank;
    unsigned long long timeout_ns;
    int* err;
};

template <int kMode>
__device__ __forceinline__ int map_m(int mv, int m_blocks, const FuseParams<kMode>& fp) {
    if constexpr (kMode == kScatterMode) {
        // rank r walks the owners in the order r+1, r+2, ..., r (ring schedule): every owner receives from ONE peer at a time
        int m = mv + ((fp.me + 1) % fp.p) * (fp.rows_per_rank / BLOCK_M);
        return m >= m_blocks ? m - m_blocks : m;
    } else if constexpr (kMode == kGatherMode) {
        const int c = mv / fp.p, k = mv - c * fp.p;
        int slot = fp.me + k; if (slot >= fp.p) slot -= fp.p;
        return slot * fp.blocks_per_rank + c;
    } else {
        return mv;
    }
}
template <int kMode>
__device__ __forceinline__ TileCoord tile_of(int t, int m_blocks, int n_blocks, const FuseParams<kMode>& fp) {
    int group_m = kGroupM;
    if constexpr (kMode == kPlain) group_m = fp.group_m;
    TileCoord tc = tile_of_virtual(t, m_blocks, n_blocks, group_m);
    tc.m = map_m<kMode>(tc.m, m_blocks, fp);
    return tc;
}

template <int kLayout, int kMode = kPlain, int kBlockN = BLOCK_N>
__global__ void __maxnreg__(Tile<kBlockN>::kMaxRegs) gemm_bf16_kernel(const __grid_constant__ CUtensorMap map_a,
                                                                const __grid_constant__ CUtensorMap map_b,
                                                                const __grid_constant__ CUtensorMap map_c,
                                                                const __nv_bfloat16* __restrict__ c_old, int M, int N, int K,
                                                                int accumulate,
                                                                const __grid_constant__ FuseParams<kMode> sp) {
    static_assert(kMode == kPlain || kBlockN == BLOCK_N, "the fused modes wait on peers: they keep the three-slim-CTA tile");
    constexpr bool kScatter = kMode == kScatterMode, kGather = kMode == kGatherMode;
    constexpr bool kAMn = kLayout == kNT, kBMn = kLayout != kTN;
    constexpr int kStages = Tile<kBlockN>::kStages, kStageBytes = Tile<kBlockN>::kStageBytes;
    constexpr int kNumStoreBufs = Tile<kBlockN>::kNumStoreBufs;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_store = smem + kStages * kStageBytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_store + kNumStoreBufs * kStoreBytes);
    uint64_t* full_bar = bars;                       // [kStages]
    uint64_t* empty_bar = bars + kStages;            // [kStages]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m_blocks = (M + BLOCK_M - 1) / BLOCK_M, n_blocks = (N + kBlockN - 1) / kBlockN;
    const int num_tiles = m_blocks * n_blocks, k_blocks = (K + BLOCK_K - 1) / BLOCK_K;

    // Fused scatter: rank r walks the owners in the order r+1, r+2, ..., r (ring schedule, map_m), so at any moment every owner
    // receives from ONE peer instead of all p-1 at once (incast would serialise the job on one GPU's NVLink ingress), and
    // the rank's own rows -- which need no NVLink -- come last, when the links are draining.
    if constexpr (kScatter) {
        // Programmatic dependent launch: the tile reducer (next kernel in this stream) may be scheduled once EVERY CTA of
        // this grid is running.  It spins on tiles this grid (and the peers') produce, so it must never take an SM's
        // registers before the GEMM CTA of that SM is resident.
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    }
    if (warp == kProducerWarp && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_c) : "memory");
        // empty: one arrival per consumer warp once its wgmma reading the stage has retired
        for (int i = 0; i < kStages; ++i) { mbar_init(smem_u32(full_bar + i), 1); mbar_init(smem_u32(empty_bar + i), kEpiThreads / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kProducerWarp) {
        // ================= TMA producer =================
        if (elect_one()) {
            int stage = 0; uint32_t phase = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                const TileCoord tc = tile_of<kMode>(t, m_blocks, n_blocks, sp);
                const CUtensorMap* amap = &map_a;
                int a_row = tc.m * BLOCK_M;
                if constexpr (kGather) {
                    const int slot = tc.m / sp.blocks_per_rank, c = tc.m - slot * sp.blocks_per_rank;
                    if (slot == sp.me) {
                        amap = &sp.a_local; a_row = c * BLOCK_M;          // own rows: straight from the local shard
                    } else {
                        // the owner's push kernel counts this 128-row block in once per pushing CTA
                        const uint32_t* f = sp.flags + slot * sp.blocks_per_rank + c;
                        unsigned long long t0 = 0; unsigned spins = 0;
                        while (true) {
                            uint32_t v;
                            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
                            if (v >= sp.target) break;
                            if ((++spins & 0x3ff) == 0) {
                                unsigned long long now = gtimer();
                                if (t0 == 0) t0 = now;
                                else if (now - t0 > sp.timeout_ns) {
                                    if (atomicCAS(sp.err + 1, 0, 4) == 0) { sp.err[2] = (int)blockIdx.x; sp.err[3] = tc.m; sp.err[4] = (int)v; sp.err[5] = (int)sp.target; sp.err[6] = slot; }
                                    *sp.err = BG_ETIMEOUT; __threadfence_system(); __trap();
                                }
                            }
                        }
                        asm volatile("fence.proxy.async.global;" ::: "memory");   // the peer's stores (generic proxy) before my TMA reads (async proxy)
                    }
                }
                for (int kb = 0; kb < k_blocks; ++kb) {
                    mbar_wait(smem_u32(empty_bar + stage), phase ^ 1);
                    const uint32_t bar = smem_u32(full_bar + stage);
                    const uint32_t sa = smem_u32(smem + stage * kStageBytes), sb = sa + kABytes;
                    mbar_expect_tx(bar, kStageBytes);
                    if (kAMn) {  // A stored [K][M]: two boxes of 64 M-elements x 64 K-rows
#pragma unroll
                        for (int j = 0; j < BLOCK_M / 64; ++j) tma_load_2d(sa + j * (BLOCK_K * 128), &map_a, bar, tc.m * BLOCK_M + j * 64, kb * BLOCK_K);
                    } else {     // A stored [M][K]: one box of 64 K-elements x 128 rows
                        tma_load_2d(sa, amap, bar, kb * BLOCK_K, a_row);
                    }
                    if (kBMn) {  // B stored [K][N]: kBlockN/64 boxes of 64 N-elements x 64 K-rows
#pragma unroll
                        for (int j = 0; j < kBlockN / 64; ++j) tma_load_2d(sb + j * (BLOCK_K * 128), &map_b, bar, tc.n * kBlockN + j * 64, kb * BLOCK_K);
                    } else {     // B stored [N][K]: one box of 64 K-elements x kBlockN rows
                        tma_load_2d(sb, &map_b, bar, kb * BLOCK_K, tc.n * kBlockN);
                    }
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ================= consumers: wgmma main loop, then registers -> (+C) -> bf16 -> swizzled smem -> TMA store =================
        const int wg = warp >> 2;                              // rows [64*wg, 64*wg+64) of the tile
        const int frag_row = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // accumulator rows frag_row and frag_row + 8
        const int frag_col = (lane & 3) * 2;                   // accumulator columns frag_col, +1 of every 8-column group
        const bool issuer = threadIdx.x == 0;
        // K-major: 8-row groups 1024 B apart (SBO), K step 32 B inside the 128-B swizzle row
        // MN-major: 64-element MN chunks BLOCK_K*128 B apart (LBO), 8-k-row groups 1024 B apart (SBO), K step 16 rows
        constexpr uint32_t a_lbo = kAMn ? BLOCK_K * 128 : 0, b_lbo = kBMn ? BLOCK_K * 128 : 0;
        constexpr uint32_t a_kstep = kAMn ? WGMMA_K * 128 : WGMMA_K * 2, b_kstep = kBMn ? WGMMA_K * 128 : WGMMA_K * 2;
        float acc[kBlockN / 2];
#pragma unroll
        for (int i = 0; i < kBlockN / 2; ++i) acc[i] = 0.f;
        int stage = 0; uint32_t phase = 0;
        int buf = 0;
        uint32_t* prev_flag = nullptr;                // fused scatter: arrival counter of the tile whose stores are in flight
        for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
            const TileCoord tc = tile_of<kMode>(t, m_blocks, n_blocks, sp);
            int prev_stage = 0;
            for (int kb = 0; kb < k_blocks; ++kb) {
                mbar_wait(smem_u32(full_bar + stage), phase);
                const uint32_t sa = smem_u32(smem + stage * kStageBytes) + wg * kWgOffset;
                const uint32_t sb = smem_u32(smem + stage * kStageBytes) + kABytes;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BLOCK_K / WGMMA_K; ++k) {
                    const uint64_t da = make_smem_desc(sa + k * a_kstep, a_lbo, 1024);
                    const uint64_t db = make_smem_desc(sb + k * b_kstep, b_lbo, 1024);
                    if constexpr (kBlockN == WIDE_N) wgmma_m64n256<kAMn ? 1 : 0, kBMn ? 1 : 0>(acc, da, db, (kb | k) != 0);
                    else wgmma_m64n128<kAMn ? 1 : 0, kBMn ? 1 : 0>(acc, da, db, (kb | k) != 0);
                }
                wgmma_commit();
                wgmma_wait<1>();                               // k-block kb-1's wgmmas have retired: its stage is free
                if (kb > 0 && lane == 0) mbar_arrive(smem_u32(empty_bar + prev_stage));
                prev_stage = stage;
                if (++stage == kStages) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            fence_acc<kBlockN / 2>(acc);
            if (lane == 0) mbar_arrive(smem_u32(empty_bar + prev_stage));
#pragma unroll
            for (int c = 0; c < kBlockN / kStoreCols; ++c) {
                const int n0 = tc.n * kBlockN + c * kStoreCols;
                if (n0 >= N) break;  // whole chunk out of bounds (uniform across the CTA)
                float* v = acc + c * (kStoreCols / 2);         // 8 column groups x {row, row + 8} x 2 columns
                if (accumulate && Tile<kBlockN>::kWide) {
                    // 128 accumulators leave 40 registers: int row bounds and one base pointer per row
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int grow = tc.m * BLOCK_M + frag_row + 8 * h;
                        if (grow < M) {
                            const uint32_t* src = reinterpret_cast<const uint32_t*>(c_old + (long long)grow * N + n0 + frag_col);
#pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                if (n0 + j * 8 < N) {
                                    const float2 o = bf2_to_f2(src[j * 4]);
                                    v[j * 4 + 2 * h] += o.x;
                                    v[j * 4 + 2 * h + 1] += o.y;
                                }
                            }
                        }
                    }
                } else if (accumulate) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const long long grow = (long long)tc.m * BLOCK_M + frag_row + 8 * h;
                        if (grow < M) {
#pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                if (n0 + j * 8 < N) {
                                    const float2 o = bf2_to_f2(*reinterpret_cast<const uint32_t*>(c_old + grow * N + n0 + j * 8 + frag_col));
                                    v[j * 4 + 2 * h] += o.x;
                                    v[j * 4 + 2 * h + 1] += o.y;
                                }
                            }
                        }
                    }
                }
                // staging buffer `buf` must be free: the store issued kNumStoreBufs chunks ago has finished reading it
                if (issuer) tma_store_wait_read<kNumStoreBufs - 1>();
                epi_bar_sync();
                uint8_t* sbuf = smem_store + buf * kStoreBytes;
                if constexpr (Tile<kBlockN>::kWide) {
                    // The same swizzle as one XOR per store on a single row address (the buffer is 1024-B aligned, so bits 4-6
                    // of the address are the 16-B chunk).  The empty asm keeps the compiler from hoisting the eight chunk
                    // addresses out of the tile loop, which would cost eight registers.
                    uint32_t srow = smem_u32(sbuf) + frag_row * 128 + ((frag_row & 7) << 4) + frag_col * 2;
                    asm volatile("" : "+r"(srow));
#pragma unroll
                    for (int h = 0; h < 2; ++h) {   // row + 8: 1024 B further, same (row & 7)
#pragma unroll
                        for (int j = 0; j < 8; ++j)
                            asm volatile("st.shared.u32 [%0], %1;" ::"r"((srow + h * 1024) ^ (j << 4)),
                                         "r"(f2_to_bf2(v[j * 4 + 2 * h], v[j * 4 + 2 * h + 1])) : "memory");
                    }
                } else {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = frag_row + 8 * h;
#pragma unroll
                        for (int j = 0; j < 8; ++j)   // 128-B swizzle: 16-B chunk j of row r lives at chunk (j ^ (r & 7))
                            *reinterpret_cast<uint32_t*>(sbuf + row * 128 + ((j ^ (row & 7)) << 4) + frag_col * 2) =
                                f2_to_bf2(v[j * 4 + 2 * h], v[j * 4 + 2 * h + 1]);
                    }
                }
                fence_proxy_async();
                epi_bar_sync();
                if (issuer) {
                    if constexpr (kScatter) {
                        const int row0 = tc.m * BLOCK_M, owner = row0 / sp.rows_per_rank;
                        tma_store_2d(&sp.dst[owner], smem_u32(sbuf), n0, sp.me * sp.rows_per_rank + (row0 - owner * sp.rows_per_rank));
                    } else {
                        tma_store_2d(&map_c, smem_u32(sbuf), n0, tc.m * BLOCK_M);
                    }
                    tma_store_commit();
                }
                if constexpr (kNumStoreBufs > 1) buf ^= 1;
            }
            if constexpr (kScatter) {
                if (issuer) {
                    // Publish the PREVIOUS tile: every bulk group except this tile's (<= 2 chunks) has completed, so its peer
                    // stores are done -- no stall on this tile's NVLink latency.
                    if (prev_flag != nullptr) {
                        asm volatile("cp.async.bulk.wait_group %0;" ::"n"(kBlockN / kStoreCols) : "memory");
                        __threadfence_system();
                        asm volatile("red.release.sys.global.add.u32 [%0], 1;" ::"l"(prev_flag) : "memory");
                    }
                    const int row0 = tc.m * BLOCK_M, owner = row0 / sp.rows_per_rank;
                    prev_flag = sp.flags[owner] + ((row0 - owner * sp.rows_per_rank) / BLOCK_M) * n_blocks + tc.n;
                }
            }
        }
        if (issuer) {
            tma_store_wait_all<0>();
            if constexpr (kScatter) {
                if (prev_flag != nullptr) {
                    __threadfence_system();
                    asm volatile("red.release.sys.global.add.u32 [%0], 1;" ::"l"(prev_flag) : "memory");
                }
            }
        }
    }
}

// ---- host: tensor maps --------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    });
    return fn;
}

// 2-D row-major bf16 tensor [rows][cols] (cols contiguous); box = box_cols x box_rows, 128-B swizzle
int make_map(CUtensorMap* map, const void* ptr, long long rows, long long cols, int box_cols, int box_rows) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return fail(BG_ECUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_ERROR_INVALID_CONTEXT) {
        // a thread (e.g. the autograd engine's) whose first CUDA call is this driver-API encode has no context bound yet:
        // touching the runtime binds the device's primary context, then retry
        cudaFree(0);
        r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (r != CUDA_SUCCESS) return fail(BG_ECUDA, "cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld", (int)r, rows, cols);
    return BG_OK;
}

int g_num_sms = 0;

}  // namespace

int bg_preload_gemm();

static int gemm_setup() {
    if (g_num_sms == 0) {
        int dev = 0;
        BG_CUDA(cudaGetDevice(&dev));
        int sms = 0;
        BG_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
#define BG_SMEM(K, W) BG_CUDA(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, Tile<W>::kSmemBytes))
        BG_SMEM(gemm_bf16_kernel<kTN>, BLOCK_N); BG_SMEM(gemm_bf16_kernel<kNN>, BLOCK_N); BG_SMEM(gemm_bf16_kernel<kNT>, BLOCK_N);
        BG_SMEM((gemm_bf16_kernel<kTN, kPlain, WIDE_N>), WIDE_N); BG_SMEM((gemm_bf16_kernel<kNN, kPlain, WIDE_N>), WIDE_N);
        BG_SMEM((gemm_bf16_kernel<kNT, kPlain, WIDE_N>), WIDE_N);
        BG_SMEM((gemm_bf16_kernel<kTN, kScatterMode>), BLOCK_N); BG_SMEM((gemm_bf16_kernel<kNN, kScatterMode>), BLOCK_N);
        BG_SMEM((gemm_bf16_kernel<kNT, kScatterMode>), BLOCK_N);
        BG_SMEM((gemm_bf16_kernel<kTN, kGatherMode>), BLOCK_N); BG_SMEM((gemm_bf16_kernel<kNN, kGatherMode>), BLOCK_N);
#undef BG_SMEM
        g_num_sms = sms;
    }
    return BG_OK;
}



static int make_ab_maps(CUtensorMap* ma, CUtensorMap* mb, const void* a, const void* b, long long m, long long n, long long k, int layout,
                        int block_n = BLOCK_N) {
    // A: TN/NN stored [M][K] (K-major: box 64 K x 128 rows); NT stored [K][M] (MN-major: box 64 M x 64 K-rows)
    int rc = layout == kNT ? make_map(ma, a, k, m, 64, BLOCK_K) : make_map(ma, a, m, k, BLOCK_K, BLOCK_M);
    if (rc) return rc;
    // B: TN stored [N][K] (box 64 K x block_n rows); NN/NT stored [K][N] (box 64 N x 64 K-rows)
    return layout == kTN ? make_map(mb, b, n, k, BLOCK_K, block_n) : make_map(mb, b, k, n, 64, BLOCK_K);
}

static int gemm_launch(const void* a, const void* b, void* c, const void* addend, long long m, long long n, long long k, int layout, void* stream);

extern "C" int bg_gemm_bf16(const void* a, const void* b, void* c, long long m, long long n, long long k, int layout,
                            int accumulate, void* stream) {
    return gemm_launch(a, b, c, accumulate ? c : nullptr, m, n, k, layout, stream);
}

// C = A op B + addend: the residual add that follows a row-parallel projection (LlamaModel_tensor_parallel.py:83,100: out + residual)
// rides in the GEMM epilogue -- fp32 accumulator + bf16 addend, ONE rounding, no separate elementwise pass.
extern "C" int bg_gemm_bf16_add(const void* a, const void* b, void* c, const void* addend, long long m, long long n, long long k,
                                int layout, void* stream) {
    if (addend == nullptr || (uintptr_t)addend % 16) return fail(BG_EINVAL, "bg_gemm_bf16_add: addend must be a 16-B aligned [M][N] bf16 tensor");
    return gemm_launch(a, b, c, addend, m, n, k, layout, stream);
}

template <int kBlockN>
static int plain_launch(const void* a, const void* b, void* c, const void* addend, long long m, long long n, long long k, int layout, void* stream);

static int gemm_launch(const void* a, const void* b, void* c, const void* addend, long long m, long long n, long long k, int layout, void* stream) {
    if (layout < 0 || layout > 2) return fail(BG_EINVAL, "bg_gemm_bf16: layout %d", layout);
    if (m <= 0 || n <= 0 || k <= 0 || m % 8 || n % 8 || k % 8)
        return fail(BG_EINVAL, "bg_gemm_bf16: m,n,k (%lld,%lld,%lld) must be positive multiples of 8", m, n, k);
    if (((uintptr_t)a | (uintptr_t)b | (uintptr_t)c) % 16) return fail(BG_EINVAL, "bg_gemm_bf16: pointers must be 16-B aligned");
    // 256-wide tiles for every output wider than one 128-wide tile; at N <= 128 a 256-wide tile would compute half zeros
    return n > BLOCK_N ? plain_launch<WIDE_N>(a, b, c, addend, m, n, k, layout, stream)
                       : plain_launch<BLOCK_N>(a, b, c, addend, m, n, k, layout, stream);
}

template <int kBlockN>
static int plain_launch(const void* a, const void* b, void* c, const void* addend, long long m, long long n, long long k, int layout, void* stream) {
    CUtensorMap ma, mb, mc;
    int rc = make_ab_maps(&ma, &mb, a, b, m, n, k, layout, kBlockN);
    if (rc) return rc;
    rc = make_map(&mc, c, m, n, kStoreCols, BLOCK_M);
    if (rc) return rc;
    rc = gemm_setup();
    if (rc) return rc;
    const long long n_blocks = (n + kBlockN - 1) / kBlockN, tiles = ((m + BLOCK_M - 1) / BLOCK_M) * n_blocks;
    const int grid = (int)(tiles < g_num_sms ? tiles : g_num_sms);
    cudaStream_t st = (cudaStream_t)stream;
    const __nv_bfloat16* c_old = (const __nv_bfloat16*)addend;
    const int accumulate = addend != nullptr;
    constexpr int smem = Tile<kBlockN>::kSmemBytes;
    // Raster: m-blocks per sweep over n.  From a sweep of 1..64 with the 256-wide tile at the flagship shapes on H100 (DESIGN
    // section 4): outputs of <= 16 n-blocks (N <= 4096) run within 3.4 % of their best with 4, wider ones within 1.5 % with 16.
    // At N <= 128 (one n-block, the 128-wide tile) every group size walks the same order.  The raster orders tiles only; every
    // output element is the same.
    FuseParams<kPlain> plain;
    plain.group_m = n_blocks <= 16 ? 4 : 16;
    if (layout == kTN) gemm_bf16_kernel<kTN, kPlain, kBlockN><<<grid, kThreads, smem, st>>>(ma, mb, mc, c_old, (int)m, (int)n, (int)k, accumulate, plain);
    else if (layout == kNN) gemm_bf16_kernel<kNN, kPlain, kBlockN><<<grid, kThreads, smem, st>>>(ma, mb, mc, c_old, (int)m, (int)n, (int)k, accumulate, plain);
    else gemm_bf16_kernel<kNT, kPlain, kBlockN><<<grid, kThreads, smem, st>>>(ma, mb, mc, c_old, (int)m, (int)n, (int)k, accumulate, plain);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

// ---- fused GEMM + reduce-scatter / all-reduce ---------------------------------------------------------------------------------
namespace {

struct Bcast {
    char* out[BG_MAX_PEERS];     // every member's full [M][N] output (all-reduce), or all null (reduce-scatter)
    char* mc;                    // multicast address of that buffer (one multimem.st reaches every member), or null
    int on;
};

__device__ __forceinline__ void mm_st_16g(void* mc, const uint4& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(__uint_as_float(v.x)),
                 "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w)) : "memory");
}

// One CTA per local tile (grid-strided): wait until all p partial tiles have landed, sum them in fp32, write bf16 -- into the
// local [M/p][N] result (reduce-scatter) or into rows [me*M/p, ...) of EVERY member's [M][N] result (all-reduce: the second
// shot of the two-shot algorithm happens here, tile by tile, while the GEMMs are still producing).
__global__ void __launch_bounds__(128, 8) tile_reduce_kernel(const __nv_bfloat16* __restrict__ partial, uint32_t* __restrict__ flags,
                                                          __nv_bfloat16* __restrict__ out, int p, int me, int rows_per_rank, int N,
                                                          int n_blocks, int local_tiles, const __grid_constant__ Bcast bc,
                                                          unsigned long long timeout_ns, int* err) {
    for (int lt = blockIdx.x; lt < local_tiles; lt += gridDim.x) {
        if (threadIdx.x == 0) {
            unsigned long long t0 = 0;
            unsigned spins = 0;
            while (true) {
                uint32_t v;
                asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + lt) : "memory");
                if (v >= (uint32_t)p) break;
                if ((++spins & 0x3ff) == 0) {
                    unsigned long long now = gtimer();
                    if (t0 == 0) t0 = now;
                    else if (now - t0 > timeout_ns / 2) {     // (half: a missing tile is reported before the peers' barriers time out)
                        if (atomicCAS(err + 1, 0, 3) == 0) { err[2] = (int)blockIdx.x; err[3] = lt; err[4] = (int)v; err[5] = p; err[6] = local_tiles; }
                        *err = BG_ETIMEOUT; __threadfence_system(); __trap();
                    }
                }
            }
        }
        __syncthreads();
        const int mb = lt / n_blocks, nb = lt % n_blocks;
        const int row0 = mb * BLOCK_M, col0 = nb * BLOCK_N;
        const int cols = min(BLOCK_N, N - col0), rows = min(BLOCK_M, rows_per_rank - row0);
        const int vec_per_row = cols / 8;
        for (int i = threadIdx.x; i < rows * vec_per_row; i += blockDim.x) {
            const int r = i / vec_per_row, c = i - r * vec_per_row;
            const size_t off = (size_t)(row0 + r) * N + col0 + c * 8;
            uint4 in[BG_MAX_PEERS];
#pragma unroll
            for (int src = 0; src < BG_MAX_PEERS; ++src)
                if (src < p) in[src] = ld16_stream(partial + (size_t)src * rows_per_rank * N + off);
            float acc[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
            for (int src = 0; src < BG_MAX_PEERS; ++src)
                if (src < p) {
                    float f[8];
                    unpack8(in[src], f);
#pragma unroll
                    for (int e = 0; e < 8; ++e) acc[e] += f[e];
                }
            const uint4 o = pack8(acc);
            if (bc.on) {
                const size_t goff = ((size_t)me * rows_per_rank * N + off) * 2;
                if (bc.mc != nullptr) {
                    mm_st_16g(bc.mc + goff, o);
                } else {
                    for (int k = 0; k < p; ++k) {
                        int q = me + k; if (q >= p) q -= p;
                        st16(bc.out[q] + goff, o);
                    }
                }
            } else {
                st16(out + off, o);
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) flags[lt] = 0;   // ready for the next use (peers only write again after the next entry barrier)
    }
    // (all-reduce: the cross-rank exit barrier is the next kernel of the stream, bg_coll.cu)
    // programmatic dependent of the GEMM: do not complete (and release the stream) before the GEMM grid has
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

}  // namespace

// Internal entries used by bg_coll.cu (which owns contexts, groups and peer pointers and has validated the arguments: layout,
// dims, alignment, p >= 2, M % (p * 128)).  partial/flags: per-member pointers.  Both kernels go to ONE stream: the GEMM, then
// the reducer as its programmatic dependent (it starts when all GEMM CTAs are resident, not when they finish; tiles are handed
// over through the arrival counters).
int bg_gemm_scatter_maps(FusedGemmMaps* maps, const void* a, const void* b, long long m, long long n, long long k, int layout, int p,
                         void* const* partial_ptrs) {
    int rc = make_ab_maps(&maps->a, &maps->b, a, b, m, n, k, layout);
    if (rc) return rc;
    for (int i = 0; i < BG_MAX_PEERS; ++i) {
        if (i < p) { rc = make_map(&maps->peer[i], partial_ptrs[i], m, n, kStoreCols, BLOCK_M); if (rc) return rc; }
        else maps->peer[i] = maps->peer[0];
    }
    return gemm_setup();
}

int bg_gemm_scatter_launch(const FusedGemmMaps& maps, long long m, long long n, long long k, int layout, int p, int me,
                           void* const* partial_ptrs, uint32_t* const* flag_ptrs, void* out, void* const* bcast_ptrs, char* bcast_mc,
                           unsigned long long timeout_ns, int* err_dev, cudaStream_t st) {
    const int rows_per_rank = (int)(m / p);
    FuseParams<kScatterMode> sp;
    sp.p = p; sp.me = me; sp.rows_per_rank = rows_per_rank;
    for (int i = 0; i < BG_MAX_PEERS; ++i) {
        sp.flags[i] = i < p ? flag_ptrs[i] : nullptr;
        sp.dst[i] = maps.peer[i];
    }
    const int m_blocks = (int)((m + BLOCK_M - 1) / BLOCK_M), n_blocks = (int)((n + BLOCK_N - 1) / BLOCK_N);
    const long long tiles = (long long)m_blocks * n_blocks;
    const int grid = (int)(tiles < g_num_sms ? tiles : g_num_sms);
    const int local_tiles = (rows_per_rank / BLOCK_M) * n_blocks;
    const CUtensorMap& mc_unused = sp.dst[0];
    if (layout == kTN) gemm_bf16_kernel<kTN, kScatterMode><<<grid, kThreads, Tile<BLOCK_N>::kSmemBytes, st>>>(maps.a, maps.b, mc_unused, nullptr, (int)m, (int)n, (int)k, 0, sp);
    else if (layout == kNN) gemm_bf16_kernel<kNN, kScatterMode><<<grid, kThreads, Tile<BLOCK_N>::kSmemBytes, st>>>(maps.a, maps.b, mc_unused, nullptr, (int)m, (int)n, (int)k, 0, sp);
    else gemm_bf16_kernel<kNT, kScatterMode><<<grid, kThreads, Tile<BLOCK_N>::kSmemBytes, st>>>(maps.a, maps.b, mc_unused, nullptr, (int)m, (int)n, (int)k, 0, sp);
    BG_CHECK_LAUNCH();
    // one reducer CTA fits beside a GEMM CTA (registers); more CTAs than SMs only queue
    const int rgrid = local_tiles < g_num_sms ? local_tiles : g_num_sms;
    Bcast bc = {};
    if (bcast_ptrs != nullptr) {
        bc.on = 1; bc.mc = bcast_mc;
        for (int i = 0; i < p; ++i) bc.out[i] = (char*)bcast_ptrs[i];
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)rgrid); cfg.blockDim = dim3(128);   // slim: fits beside the GEMM CTA and two more collectives
    cfg.dynamicSmemBytes = 0; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    static const bool no_pdl = getenv("HGB_NO_PDL") != nullptr;      // debugging aid: launch the reducer as an ordinary kernel
    cfg.attrs = attr; cfg.numAttrs = no_pdl ? 0 : 1;
    BG_CUDA(cudaLaunchKernelEx(&cfg, tile_reduce_kernel, (const __nv_bfloat16*)partial_ptrs[me], (uint32_t*)flag_ptrs[me],
                               (__nv_bfloat16*)out, p, me, rows_per_rank, (int)n, n_blocks, local_tiles, bc, timeout_ns, err_dev));
    bg::g_launches.fetch_add(1, std::memory_order_relaxed);
    return BG_OK;
}

// Fused all-gather + GEMM: the consumer half (the push kernel is launched by bg_coll.cu on the communication stream).
int bg_gemm_gather_maps(FusedGemmMaps* maps, const void* a_local, const void* a_staged, const void* b, void* c, long long m, long long n,
                        long long k, int layout, int p) {
    int rc = make_ab_maps(&maps->a, &maps->b, a_staged, b, m, n, k, layout);
    if (rc) return rc;
    rc = make_map(&maps->c, c, m, n, kStoreCols, BLOCK_M);
    if (rc) return rc;
    rc = make_map(&maps->peer[0], a_local, m / p, k, BLOCK_K, BLOCK_M);
    if (rc) return rc;
    return gemm_setup();
}

int bg_gemm_gather_launch(const FusedGemmMaps& maps, long long m, long long n, long long k, int layout, int p, int me,
                          const uint32_t* flags, uint32_t target, unsigned long long timeout_ns, int* err_dev, cudaStream_t st) {
    FuseParams<kGatherMode> gp;
    gp.a_local = maps.peer[0];
    gp.flags = flags; gp.target = target; gp.p = p; gp.me = me; gp.blocks_per_rank = (int)(m / p / BLOCK_M);
    gp.timeout_ns = timeout_ns; gp.err = err_dev;
    const long long tiles = (m / BLOCK_M) * ((n + BLOCK_N - 1) / BLOCK_N);
    const int grid = (int)(tiles < g_num_sms ? tiles : g_num_sms);
    if (layout == kTN) gemm_bf16_kernel<kTN, kGatherMode><<<grid, kThreads, Tile<BLOCK_N>::kSmemBytes, st>>>(maps.a, maps.b, maps.c, nullptr, (int)m, (int)n, (int)k, 0, gp);
    else gemm_bf16_kernel<kNN, kGatherMode><<<grid, kThreads, Tile<BLOCK_N>::kSmemBytes, st>>>(maps.a, maps.b, maps.c, nullptr, (int)m, (int)n, (int)k, 0, gp);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

// loads every kernel of this file and sets the dynamic shared-memory limits (see bg_preload_coll in bg_coll.cu)
int bg_preload_gemm() {
    int rc = gemm_setup();
    if (rc) return rc;
    cudaFuncAttributes attr;
    BG_CUDA(cudaFuncGetAttributes(&attr, reinterpret_cast<const void*>(&tile_reduce_kernel)));
    return BG_OK;
}

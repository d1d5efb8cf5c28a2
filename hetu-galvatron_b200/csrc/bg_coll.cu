// bg_coll.cu -- the peer-memory collectives (SURVEY 2.3 rows C1-C3, C5-C10, C12-C14, C16) as SLIM kernels.
//
// Every cross-rank kernel here is 128 threads x <= 64 registers with no shared memory (8,192 registers per CTA), launched with
// at most one CTA per SM ("comm_ctas", default 132).  A 128-wide wgmma GEMM CTA (every fused GEMM, and plain GEMMs of N <= 128)
// takes 36,864 registers and 193 KiB of the shared memory of its SM, so up to three collectives (e.g. ZeRO-3's prefetch
// all-gather, the gradient reduce-scatter and a tensor-parallel exchange) are resident BESIDE it, and beside each other: a
// collective never has to wait for a different kernel of its own rank to leave the SMs before its peers can see it arrive.
// A 256-wide plain GEMM CTA (48,384 registers, 209 KiB) leaves room for two; a third waits at most until that GEMM, which
// waits on nothing, retires (bg_gemm.cu, DESIGN section 2).  That removes the cross-rank deadlock
// of round 1's 256-thread / 128-register kernels (two of them could not share an SM; rank A ran the all-gather and rank B the
// reduce-scatter, each waiting for the peer kernel that could not become resident) without serialising the collectives on the
// host.  Bandwidth: a peer load takes ~2,000 cycles (~1.8 us) over NVSwitch; 132 x 128 threads x 8 x 16 B = 2.2 MB in
// flight covers 450 GB/s x 1.8 us = 0.8 MB (Little), so the slim kernels keep the NVLink pipe full.
//
// With a multicast-bound buffer (NVLS, BG_CTX_VMM) the same kernels use the switch: multimem.st replicates an all-gather
// store to every member (one store instead of p), multimem.ld_reduce returns the sum over the members (one load instead of p).
#include <math.h>

#include "bg_ctx.cuh"

using namespace bg;

namespace {

constexpr int kThreads = 128;
#define BG_SLIM __launch_bounds__(128, 8)
constexpr int kUnroll = 4;        // 16-B vectors per thread per iteration in the push kernels
constexpr int kInFlight = 8;      // 16-B NVLink loads in flight per thread in the pull kernels

__global__ void coll_barrier_kernel(const __grid_constant__ Sig s) { sync_peers<true, true, true>(s); }

__device__ __forceinline__ uint4 mm_ld_reduce_bf16(const void* mc) {   // sum over every member's copy, fp32 accumulation in the switch
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    return v;
}
__device__ __forceinline__ uint4 mm_ld_reduce_f32(const void* mc) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    return v;
}
__device__ __forceinline__ void mm_st_16(void* mc, const uint4& v) {    // one store, lands in every member's copy
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(__uint_as_float(v.x)),
                 "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w)) : "memory");
}

// ------------------------------------------------------------------------------------------------
// C1: all-gather (push) fused with cast
// ------------------------------------------------------------------------------------------------
template <typename SrcT, typename DstT>
struct Cvt;
template <> struct Cvt<float, __nv_bfloat16> {  // 8 elements: 32 B in, 16 B out
    static constexpr int kElems = 8;
    __device__ static void load(const float* src, size_t i, uint4* regs) {
        regs[0] = ld16_stream(src + i);
        regs[1] = ld16_stream(src + i + 4);
    }
    __device__ static uint4 convert(const uint4* regs) {
        uint4 o;
        o.x = f2_to_bf2(__uint_as_float(regs[0].x), __uint_as_float(regs[0].y));
        o.y = f2_to_bf2(__uint_as_float(regs[0].z), __uint_as_float(regs[0].w));
        o.z = f2_to_bf2(__uint_as_float(regs[1].x), __uint_as_float(regs[1].y));
        o.w = f2_to_bf2(__uint_as_float(regs[1].z), __uint_as_float(regs[1].w));
        return o;
    }
    static constexpr int kRegs = 2;
};
template <> struct Cvt<__nv_bfloat16, __nv_bfloat16> {
    static constexpr int kElems = 8;
    static constexpr int kRegs = 1;
    __device__ static void load(const __nv_bfloat16* src, size_t i, uint4* regs) { regs[0] = ld16_stream(src + i); }
    __device__ static uint4 convert(const uint4* regs) { return regs[0]; }
};
template <> struct Cvt<float, float> {
    static constexpr int kElems = 4;
    static constexpr int kRegs = 1;
    __device__ static void load(const float* src, size_t i, uint4* regs) { regs[0] = ld16_stream(src + i); }
    __device__ static uint4 convert(const uint4* regs) { return regs[0]; }
};

// kSignal (the all-gather half of the fused all-gather + GEMM, C7): the shard is pushed chunk by chunk; after a chunk every CTA
// bumps the chunk's arrival counter on every receiver (release at .sys scope), and the consumer -- the GEMM's TMA producer --
// starts on a chunk as soon as its counter reaches the number of pushing CTAs.  No exit barrier.  (The rank's own slot is
// written too -- the GEMM reads the local shard in place, but the wgrad GEMM of the layer wants the complete gathered operand.)
struct AgSignal {
    uint32_t* flag[BG_MAX_PEERS];   // receiver q's counters: [source member][chunk]
    size_t chunk_vecs;
    int n_chunks, split;            // a chunk is complete when `split` units have been counted in
};

template <typename SrcT, typename DstT, bool kSignal>
__global__ void BG_SLIM all_gather_push_kernel(const __grid_constant__ PeerPtrs dst, char* __restrict__ dst_mc, const SrcT* __restrict__ src,
                                               size_t shard_elems, const __grid_constant__ AgSignal sg, const __grid_constant__ Sig s) {
    using C = Cvt<SrcT, DstT>;
    sync_peers<false, false, true>(s);  // every member has finished consuming its dst (it reached this kernel)
    const size_t nvec = shard_elems / C::kElems;
    const size_t dst_base = (size_t)s.me * shard_elems * sizeof(DstT);
    if (!kSignal) {
        const size_t stride = (size_t)gridDim.x * blockDim.x;
        for (size_t v0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v0 < nvec; v0 += stride * kUnroll) {
            uint4 regs[kUnroll][C::kRegs];
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                size_t v = v0 + u * stride;
                if (v < nvec) C::load(src, v * C::kElems, regs[u]);
            }
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                size_t v = v0 + u * stride;
                if (v < nvec) {
                    uint4 o = C::convert(regs[u]);
                    if (dst_mc != nullptr) {
                        mm_st_16(dst_mc + dst_base + v * 16, o);       // replicated by the switch
                    } else {
                        for (int k = 0; k < s.n; ++k) {
                            int p = s.me + k; if (p >= s.n) p -= s.n;  // stagger targets across senders
                            st16(dst.p[p] + dst_base + v * 16, o);
                        }
                    }
                }
            }
        }
        sync_peers<true, true, false>(s);  // my stores are visible everywhere; everyone's shard has landed here
        return;
    }
    // kSignal: a chunk (one 128-row block of the GEMM) is cut into `split` units; a unit is pushed by ONE CTA, which then makes its
    // stores visible (one .sys fence per unit, not per chunk and grid) and counts the unit in on every receiver.  Units are dealt
    // out in chunk order, so block c of every slot is complete before block c+1.
    const size_t unit_vecs = sg.chunk_vecs / sg.split;
    const int n_units = sg.n_chunks * sg.split;
    for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
        const size_t u0 = (size_t)unit * unit_vecs, u1 = u0 + unit_vecs;
        for (size_t v0 = u0 + threadIdx.x; v0 < u1; v0 += (size_t)blockDim.x * kUnroll) {
            uint4 regs[kUnroll][C::kRegs];
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                size_t v = v0 + (size_t)u * blockDim.x;
                if (v < u1) C::load(src, v * C::kElems, regs[u]);
            }
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                size_t v = v0 + (size_t)u * blockDim.x;
                if (v < u1) {
                    uint4 o = C::convert(regs[u]);
                    for (int k = 0; k < s.n; ++k) {
                        int p = s.me + k; if (p >= s.n) p -= s.n;
                        st16(dst.p[p] + dst_base + v * 16, o);
                    }
                }
            }
        }
        __threadfence_system();
        __syncthreads();
        const int t = threadIdx.x;
        if (t < s.n && t != s.me)
            asm volatile("red.release.sys.global.add.u32 [%0], 1;" ::"l"(sg.flag[t] + (size_t)s.me * sg.n_chunks + unit / sg.split) : "memory");
    }
}

// ------------------------------------------------------------------------------------------------
// C2: reduce-scatter (pull) fused with prescale/postscale, cast and accumulate -- or with the AdamW step (SURVEY 8f-3)
// ------------------------------------------------------------------------------------------------
template <bool kSrcBf16>
__device__ __forceinline__ void rs_accumulate(const uint4& v, float* acc, float w) {
    if (kSrcBf16) {
        float f[8];
        unpack8(v, f);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(f[i], w, acc[i]);
    } else {
        acc[0] = fmaf(__uint_as_float(v.x), w, acc[0]); acc[1] = fmaf(__uint_as_float(v.y), w, acc[1]);
        acc[2] = fmaf(__uint_as_float(v.z), w, acc[2]); acc[3] = fmaf(__uint_as_float(v.w), w, acc[3]);
    }
}

struct AdamArgs {
    float lr, beta1, beta2, eps, weight_decay, bias_corr1, bias_corr2_sqrt;
};
struct RsOut {
    void* dst;                    // kEpi 0: fp32 shard, 1: bf16 shard, 2 / 4: fp32 parameter shard (AdamW), 3: fp32 shard or null
    float* exp_avg;
    float* exp_avg_sq;
    int accumulate;
    AdamArgs a;
    const float* clip_coef;       // kEpiAdamWClip: the gradient is (sum prescale * x) * (postscale * *clip_coef); null: 1
    // kEpiSumSq: one fp32 sum of squares of the reduced gradient per warp, in warp order; the entries from 4 * gridDim.x up to
    // n_partials are zeroed.  Shard-relative element ranges [skip_lo, skip_hi) are left out of the sum.
    float* partials;
    int n_partials, n_skip;
    unsigned long long skip_lo[BG_MAX_SKIP], skip_hi[BG_MAX_SKIP];
};
// kEpiAdamWClip is kEpiAdamW with the clip coefficient folded into postscale at kernel start: its own instances, so the code of
// the unclipped ones (and their register allocation) stays as it is
enum { kEpiF32 = 0, kEpiBf16 = 1, kEpiAdamW = 2, kEpiSumSq = 3, kEpiAdamWClip = 4 };
constexpr int kWarps = kThreads / 32;

template <int E, int kEpi>
__device__ __forceinline__ void rs_epilogue(const RsOut& o, size_t v, float* acc, float postscale, double& sq) {
    if (kEpi == kEpiSumSq) {
        // the norm pass: squares accumulate in fp64 (a thread's sum runs over thousands of elements).  Range bounds are multiples
        // of 8 elements, so a vector is either inside a skip range or outside all of them.  With a destination the reduced shard
        // is written as well, with the bits of kEpiF32 (accumulate 0).
#pragma unroll
        for (int i = 0; i < E; ++i) acc[i] *= postscale;
        const unsigned long long e = (unsigned long long)v * E;
        bool skip = false;
        for (int r = 0; r < o.n_skip; ++r) skip |= e >= o.skip_lo[r] && e < o.skip_hi[r];
        if (!skip) {
#pragma unroll
            for (int i = 0; i < E; ++i) sq = fma((double)acc[i], (double)acc[i], sq);
        }
        if (o.dst != nullptr) {
            float4* d = reinterpret_cast<float4*>(o.dst) + v * (E / 4);
#pragma unroll
            for (int q = 0; q < E / 4; ++q) d[q] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
        }
    } else if (kEpi == kEpiBf16) {
#pragma unroll
        for (int i = 0; i < E; ++i) acc[i] *= postscale;
        uint4* d = reinterpret_cast<uint4*>(o.dst) + v;
        if (o.accumulate) {
            float old[8];
            unpack8(*d, old);
#pragma unroll
            for (int i = 0; i < E; ++i) acc[i] += old[i];
        }
        st16(d, pack8(acc));
    } else if (kEpi == kEpiF32) {
        float4* d = reinterpret_cast<float4*>(o.dst) + v * (E / 4);
#pragma unroll
        for (int q = 0; q < E / 4; ++q) {
            float4 r = make_float4(acc[4 * q] * postscale, acc[4 * q + 1] * postscale, acc[4 * q + 2] * postscale, acc[4 * q + 3] * postscale);
            if (o.accumulate) {
                float4 old = d[q];
                r.x += old.x; r.y += old.y; r.z += old.z; r.w += old.w;
            }
            d[q] = r;
        }
    } else {
        // the reduced gradient never touches HBM: it updates (param, exp_avg, exp_avg_sq) from registers.  Same update rule as
        // torch.optim.AdamW / apex FusedAdam(adam_w_mode=True) (galvatron/core/runtime/utils.py:137-150).
        const AdamArgs& a = o.a;
        const float step_size = a.lr / a.bias_corr1, decay = 1.f - a.lr * a.weight_decay;
        float4* pp = reinterpret_cast<float4*>(o.dst) + v * (E / 4);
        float4* pm = reinterpret_cast<float4*>(o.exp_avg) + v * (E / 4);
        float4* pv = reinterpret_cast<float4*>(o.exp_avg_sq) + v * (E / 4);
#pragma unroll
        for (int q = 0; q < E / 4; ++q) {
            float4 w = pp[q], m = pm[q], vv = pv[q];
            float* wf = reinterpret_cast<float*>(&w); float* mf = reinterpret_cast<float*>(&m); float* vf = reinterpret_cast<float*>(&vv);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float gi = acc[4 * q + i] * postscale;
                mf[i] = a.beta1 * mf[i] + (1.f - a.beta1) * gi;
                vf[i] = a.beta2 * vf[i] + (1.f - a.beta2) * gi * gi;
                const float denom = sqrtf(vf[i]) / a.bias_corr2_sqrt + a.eps;
                wf[i] = wf[i] * decay - step_size * mf[i] / denom;
            }
            pp[q] = w; pm[q] = m; pv[q] = vv;
        }
    }
}

// PMAX = 2, 4 or 8 >= group size: V = 8 / PMAX vectors x PMAX loads (the rank's own copy + the peers in ring order) are in flight
// per thread.  (Keeping only peer loads in flight and reading the own copy one vector ahead was measured SLOWER at p = 2: the
// serialised local loads, 7 x ~700 cycles, outlast the peer latency.)  kMc: the source is multicast-bound -- ONE
// multimem.ld_reduce per vector returns the members' sum (fp32 accumulation in the switch, rounded to the source dtype).
template <int PMAX, int kEpi>
struct RsPlan {
    // (the AdamW epilogue keeps 12 more registers of optimizer state live, the sum-of-squares epilogue its fp64 sum and the skip
    // test: half the vectors in flight below 8 peers)
    static constexpr bool kHalf = kEpi == kEpiAdamW || kEpi == kEpiAdamWClip || kEpi == kEpiSumSq;
    static constexpr int V = (kHalf && PMAX < 8 ? kInFlight / 2 : kInFlight) / PMAX;
    static constexpr int V_MC = kHalf ? 4 : 8;
};

template <int PMAX, bool kSrcBf16, int kEpi, bool kMc>
__global__ void BG_SLIM reduce_scatter_pull_kernel(const __grid_constant__ PeerPtrs src, const char* __restrict__ src_mc, const __grid_constant__ RsOut o,
                                                   size_t shard_elems, float prescale, float postscale, const __grid_constant__ Sig s) {
    constexpr int E = kSrcBf16 ? 8 : 4;  // elements per 16-B source vector
    constexpr int NL = kMc ? 1 : PMAX;
    constexpr int V = kMc ? RsPlan<PMAX, kEpi>::V_MC : RsPlan<PMAX, kEpi>::V;
    sync_peers<false, false, true>(s);  // every member's src is complete (its producer kernels finished before this one)
    const size_t nvec = shard_elems / E;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const size_t slice_off = (size_t)s.me * shard_elems * (kSrcBf16 ? 2 : 4);
    if (kEpi == kEpiAdamWClip && o.clip_coef != nullptr) postscale *= *o.clip_coef;
    double sq = 0.0;
    for (size_t v0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v0 < nvec; v0 += stride * V) {
        uint4 in[V][NL];
        // issue every load of this iteration before consuming any
#pragma unroll
        for (int u = 0; u < V; ++u) {
            const size_t v = v0 + u * stride;
            if (kMc) {
                if (v < nvec) in[u][0] = kSrcBf16 ? mm_ld_reduce_bf16(src_mc + slice_off + v * 16) : mm_ld_reduce_f32(src_mc + slice_off + v * 16);
            } else {
#pragma unroll
                for (int k = 0; k < NL; ++k) {
                    if (k < s.n && v < nvec) {
                        int q = s.me + k; if (q >= s.n) q -= s.n;       // own copy, then ring order: every source serves one reader at a time
                        const char* a = src.p[q] + slice_off + v * 16;
                        in[u][k] = k == 0 ? ld16_stream(a) : ld16_peer(a);
                    }
                }
            }
        }
#pragma unroll
        for (int u = 0; u < V; ++u) {
            const size_t v = v0 + u * stride;
            if (v >= nvec) break;
            float acc[E];
#pragma unroll
            for (int i = 0; i < E; ++i) acc[i] = 0.f;
            // fixed summation order (own slice, then the peers in ring order): run-to-run deterministic.  Each rank's contribution
            // is scaled by `prescale` before the sum, as the reference pre-divides (_runtime_utils.py:852).
#pragma unroll
            for (int k = 0; k < NL; ++k)
                if (kMc || k < s.n) rs_accumulate<kSrcBf16>(in[u][k], acc, prescale);
            rs_epilogue<E, kEpi>(o, v, acc, postscale, sq);
        }
    }
    if (kEpi == kEpiSumSq) {        // warp sums in a fixed order, one entry per warp, the rest of the slot zeroed
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, off);
        if ((threadIdx.x & 31) == 0) o.partials[blockIdx.x * kWarps + threadIdx.x / 32] = (float)sq;
        if (blockIdx.x == 0)
            for (int i = gridDim.x * kWarps + threadIdx.x; i < o.n_partials; i += blockDim.x) o.partials[i] = 0.f;
    }
    sync_peers<true, false, false>(s);  // every member has finished reading my src: it may be overwritten
}

// The clipped AdamW step on a local fp32 gradient (pooled ZeRO-3 units keep theirs in an fp32 shard until the step): the
// epilogue of the reduce-scatter above, with the gradient loaded instead of reduced.
__global__ void BG_SLIM adamw_local_kernel(const float* __restrict__ grad, const __grid_constant__ RsOut o, size_t n) {
    const float coef = o.clip_coef != nullptr ? *o.clip_coef : 1.f;
    double unused = 0.0;
    for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < n / 4; v += (size_t)gridDim.x * blockDim.x) {
        const float4 g = reinterpret_cast<const float4*>(grad)[v];
        float acc[4] = {g.x, g.y, g.z, g.w};
        rs_epilogue<4, kEpiAdamW>(o, v, acc, coef, unused);
    }
}

template <bool kSrcBf16, int kEpi>
void launch_rs(int n, bool mc, int grid, cudaStream_t st, const PeerPtrs& src, const char* src_mc, const RsOut& o, size_t shard_elems,
               float prescale, float postscale, const Sig& s) {
#define BG_RS(P, MC) reduce_scatter_pull_kernel<P, kSrcBf16, kEpi, MC><<<grid, kThreads, 0, st>>>(src, src_mc, o, shard_elems, prescale, postscale, s)
    if (mc) BG_RS(2, true);
    else if (n <= 2) BG_RS(2, false);
    else if (n <= 4) BG_RS(4, false);
    else BG_RS(8, false);
#undef BG_RS
}

// ------------------------------------------------------------------------------------------------
// C3/C5/C6/C13: all-reduce, one-shot (small) and two-shot (large)
// ------------------------------------------------------------------------------------------------
template <bool kBf16, bool kMax>
__device__ __forceinline__ void ar_combine(const uint4& v, float* acc, bool first) {
    constexpr int E = kBf16 ? 8 : 4;
    float f[E];
    if (kBf16) unpack8(v, f);
    else { f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y); f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w); }
#pragma unroll
    for (int i = 0; i < E; ++i) acc[i] = first ? f[i] : (kMax ? fmaxf(acc[i], f[i]) : acc[i] + f[i]);
}

template <bool kBf16>
__device__ __forceinline__ uint4 ar_pack(const float* acc, float scale) {
    if (kBf16) {
        float t[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) t[i] = acc[i] * scale;
        return pack8(t);
    }
    uint4 o;
    o.x = __float_as_uint(acc[0] * scale); o.y = __float_as_uint(acc[1] * scale);
    o.z = __float_as_uint(acc[2] * scale); o.w = __float_as_uint(acc[3] * scale);
    return o;
}

// one-shot: every member reads all n buffers in full
template <int PMAX, bool kBf16, bool kMax>
__global__ void BG_SLIM all_reduce_oneshot_kernel(const __grid_constant__ PeerPtrs src, void* __restrict__ dst, size_t nvec, float scale,
                                                  const __grid_constant__ Sig s) {
    constexpr int E = kBf16 ? 8 : 4;
    sync_peers<false, false, true>(s);
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
        uint4 in[PMAX];
#pragma unroll
        for (int p = 0; p < PMAX; ++p)
            if (p < s.n) in[p] = (p == s.me) ? ld16_stream(src.p[p] + v * 16) : ld16_peer(src.p[p] + v * 16);
        float acc[E];
#pragma unroll
        for (int p = 0; p < PMAX; ++p)
            if (p < s.n) ar_combine<kBf16, kMax>(in[p], acc, p == 0);
        st16(reinterpret_cast<uint4*>(dst) + v, ar_pack<kBf16>(acc, scale));
    }
    sync_peers<true, false, false>(s);
}

// two-shot: reduce my slice into my own src (peer-visible), barrier, gather every member's reduced slice.
// Vector v of a slice is always handled by the same (CTA, thread) on every member, so the per-CTA channel
// barrier between the two phases is sufficient.
template <int PMAX, bool kBf16, bool kMax>
__global__ void BG_SLIM all_reduce_twoshot_kernel(const __grid_constant__ PeerPtrs src, void* __restrict__ dst, size_t slice_vec, float scale,
                                                  const __grid_constant__ Sig s) {
    constexpr int E = kBf16 ? 8 : 4;
    constexpr int V = kInFlight / PMAX;
    sync_peers<false, false, true>(s);
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const size_t my0 = (size_t)s.me * slice_vec;
    for (size_t v0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v0 < slice_vec; v0 += stride * V) {
        uint4 in[V][PMAX];
#pragma unroll
        for (int u = 0; u < V; ++u) {
            const size_t v = v0 + u * stride;
#pragma unroll
            for (int p = 0; p < PMAX; ++p)
                if (p < s.n && v < slice_vec)
                    in[u][p] = (p == s.me) ? ld16_stream(src.p[p] + (my0 + v) * 16) : ld16_peer(src.p[p] + (my0 + v) * 16);
        }
#pragma unroll
        for (int u = 0; u < V; ++u) {
            const size_t v = v0 + u * stride;
            if (v >= slice_vec) break;
            float acc[E];
#pragma unroll
            for (int p = 0; p < PMAX; ++p)
                if (p < s.n) ar_combine<kBf16, kMax>(in[u][p], acc, p == 0);
            uint4 o = ar_pack<kBf16>(acc, scale);
            st16(src.p[s.me] + (my0 + v) * 16, o);
            st16(reinterpret_cast<uint4*>(dst) + my0 + v, o);
        }
    }
    sync_peers<true, true, true>(s);
    // gather every member's reduced slice (vector v of a slice is handled by the same CTA on every member)
    for (size_t v0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v0 < slice_vec; v0 += stride * V) {
        uint4 in[V][PMAX];
#pragma unroll
        for (int u = 0; u < V; ++u) {
            const size_t v = v0 + u * stride;
#pragma unroll
            for (int k = 1; k < PMAX; ++k)
                if (k < s.n && v < slice_vec) {
                    int p = s.me + k; if (p >= s.n) p -= s.n;
                    in[u][k] = ld16_peer(src.p[p] + ((size_t)p * slice_vec + v) * 16);
                }
        }
#pragma unroll
        for (int u = 0; u < V; ++u) {
            const size_t v = v0 + u * stride;
            if (v >= slice_vec) break;
#pragma unroll
            for (int k = 1; k < PMAX; ++k)
                if (k < s.n) {
                    int p = s.me + k; if (p >= s.n) p -= s.n;
                    st16(reinterpret_cast<uint4*>(dst) + (size_t)p * slice_vec + v, in[u][k]);
                }
        }
    }
    sync_peers<true, false, false>(s);
}

// Two-shot all-reduce through the switch, in place on the group's multicast-bound buffer, then a local copy to dst.
//   phase 1: member r owns vectors [r*per, (r+1)*per): ld_reduce pulls the SUM of all members' values (one NVLink read of the
//            reduced data instead of p-1 reads), scale, multimem.st pushes the result into every member's buffer
//   phase 2: after the barrier every member's buffer holds the full result; copy it out (local HBM)
// NVLink bytes per GPU: N/p received + N/p sent through the switch's reduction / replication, vs 2(p-1)/p*N for the P2P two-shot.
template <bool kBf16>
__global__ void BG_SLIM all_reduce_nvls_kernel(char* mc, const char* local, char* dst, size_t vecs, float scale, const __grid_constant__ Sig s) {
    sync_peers<false, false, true>(s);   // every member's input is complete (its producers precede this kernel in its stream)
    const size_t per = (vecs + s.n - 1) / s.n;
    const size_t lo = per * s.me, hi = lo + per < vecs ? lo + per : vecs;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    constexpr int kU = kInFlight;        // in-switch reductions in flight per thread
    for (size_t v0 = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x; v0 < hi; v0 += stride * kU) {
        uint4 val[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const size_t v = v0 + (size_t)u * stride;
            if (v < hi) val[u] = kBf16 ? mm_ld_reduce_bf16(mc + v * 16) : mm_ld_reduce_f32(mc + v * 16);
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const size_t v = v0 + (size_t)u * stride;
            if (v < hi) {
                uint4 out = val[u];
                if (scale != 1.0f) {
                    if (kBf16) {
                        float f[8];
                        unpack8(out, f);
#pragma unroll
                        for (int e = 0; e < 8; ++e) f[e] *= scale;
                        out = pack8(f);
                    } else {
                        out.x = __float_as_uint(__uint_as_float(out.x) * scale); out.y = __float_as_uint(__uint_as_float(out.y) * scale);
                        out.z = __float_as_uint(__uint_as_float(out.z) * scale); out.w = __float_as_uint(__uint_as_float(out.w) * scale);
                    }
                }
                mm_st_16(mc + v * 16, out);
            }
        }
    }
    sync_peers<true, true, true>(s);     // my stores are visible everywhere and everyone's slice has landed here
    if (dst != nullptr) {
        for (size_t v0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v0 < vecs; v0 += stride * kU) {
            uint4 val[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u)
                if (v0 + (size_t)u * stride < vecs) val[u] = ld16_stream(local + (v0 + (size_t)u * stride) * 16);
#pragma unroll
            for (int u = 0; u < kU; ++u)
                if (v0 + (size_t)u * stride < vecs) st16(dst + (v0 + (size_t)u * stride) * 16, val[u]);
        }
        // the buffer may be refilled by the next call's producers only after every member has finished reading it: the next
        // call's entry barrier cannot give that (it waits for producers, not consumers), so leave through a barrier
        sync_peers<true, false, false>(s);
    }
}

// ------------------------------------------------------------------------------------------------
// C14: in-place sum of a two-member group's copies (the tied word-embedding gradient of the first and the last pipeline stage)
// ------------------------------------------------------------------------------------------------
// Member m owns the vector range [lo, hi) (half of the buffer); CTA c of member m reads it from both members' regions, forms
// scale * (x0 + x1) in fp32 -- member order fixed, one rounding, so both copies end bit-identical -- and stores it into both.  No
// member reads a range another member writes, so one entry and one exit barrier per CTA channel are the whole protocol: both
// members launch the same grid (it depends on the element count only), and vector v of a range is always handled by CTA c.
template <bool kBf16>
__global__ void BG_SLIM pair_sum_kernel(const __grid_constant__ PeerPtrs buf, size_t lo, size_t hi, float scale, const __grid_constant__ Sig s) {
    constexpr int E = kBf16 ? 8 : 4;
    constexpr int U = kInFlight / 2;     // two loads per vector: 8 in flight per thread
    sync_peers<false, false, true>(s);   // both regions are complete (each member's producers precede this kernel in its stream)
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t v0 = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x; v0 < hi; v0 += stride * U) {
        uint4 x0[U], x1[U];                // member 0's copy, member 1's copy
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t v = v0 + u * stride;
            if (v < hi) {
                if (s.me == 0) {
                    x0[u] = ld16_stream(buf.p[0] + v * 16);
                    x1[u] = ld16_peer(buf.p[1] + v * 16);
                } else {
                    x0[u] = ld16_peer(buf.p[0] + v * 16);
                    x1[u] = ld16_stream(buf.p[1] + v * 16);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const size_t v = v0 + u * stride;
            if (v >= hi) break;
            float acc[E];
            ar_combine<kBf16, false>(x0[u], acc, true);
            ar_combine<kBf16, false>(x1[u], acc, false);
            const uint4 o = ar_pack<kBf16>(acc, scale);
            st16(buf.p[0] + v * 16, o);
            st16(buf.p[1] + v * 16, o);
        }
    }
    sync_peers<true, true, false>(s);    // my stores are visible at the peer, and the peer's have landed here
}

// ------------------------------------------------------------------------------------------------
// C10: Ulysses all-to-all fused with the head/seq transpose (pull; up to 4 tensors per launch)
// ------------------------------------------------------------------------------------------------
constexpr int kMaxA2A = 4;
struct A2ADev {
    PeerPtrs src;
    char* dst;
    long long batch, rows, row_vec;           // row_vec = 16-B vectors per row
    long long src_bs, src_rs, src_me_off;     // in 16-B vectors
    long long dst_bs, dst_rs, dst_peer_off;   // in 16-B vectors
    long long total_vec;                      // batch * rows * row_vec * n
};
struct A2AArgs {
    A2ADev t[kMaxA2A];
    int n_tensors;
};

// element i of a (batch, rows, row_vec) block -> vector offsets in the source (peer q's buffer) and in my destination
struct A2AIdx { long long src, dst; };
__device__ __forceinline__ A2AIdx a2a_index(const A2ADev& d, unsigned i, int me, int q) {
    const unsigned row_vec = (unsigned)d.row_vec, rows = (unsigned)d.rows;
    const unsigned c = i % row_vec, r = i / row_vec;
    const unsigned row = r % rows, b = r / rows;
    A2AIdx x;
    x.src = (long long)b * d.src_bs + (long long)row * d.src_rs + (long long)me * d.src_me_off + c;
    x.dst = (long long)b * d.dst_bs + (long long)row * d.dst_rs + (long long)q * d.dst_peer_off + c;
    return x;
}

// One source at a time (ring order: rank r reads from r+1, r+2, ...: every source serves ONE reader at a time), 8 peer loads in
// flight per thread; the block the rank keeps for itself is a plain local copy.  Indices are recomputed for the store instead of
// being kept in registers across the loads.
__global__ void BG_SLIM all_to_all_rows_kernel(const __grid_constant__ A2AArgs a, const __grid_constant__ Sig s) {
    sync_peers<false, false, true>(s);
    constexpr int U = kInFlight;
    const unsigned stride = gridDim.x * blockDim.x, t0 = blockIdx.x * blockDim.x + threadIdx.x;
    for (int ti = 0; ti < a.n_tensors; ++ti) {
        const A2ADev& d = a.t[ti];
        const unsigned per_peer = (unsigned)(d.batch * d.rows * d.row_vec);
        for (int k = 0; k < s.n; ++k) {
            int q = s.me + k; if (q >= s.n) q -= s.n;
            const char* sp = d.src.p[q];
            for (unsigned i0 = t0; i0 < per_peer; i0 += stride * U) {
                uint4 regs[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const unsigned i = i0 + u * stride;
                    if (i < per_peer) {
                        const char* ad = sp + a2a_index(d, i, s.me, q).src * 16;
                        regs[u] = k == 0 ? ld16_stream(ad) : ld16_peer(ad);
                    }
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const unsigned i = i0 + u * stride;
                    if (i < per_peer) st16(d.dst + a2a_index(d, i, s.me, q).dst * 16, regs[u]);
                }
            }
        }
    }
    sync_peers<true, false, false>(s);
}

// ------------------------------------------------------------------------------------------------
// C15: ring context parallelism -- one hop of K/V (bf16) or of the dK/dV accumulators (fp32) to the next cp member.
// Flags: lane BG_LANE_RING of the group's pad, [channel][8] u32 per member: index kind*4 + parity = "a block arrived in my
// slot[parity]" (raised by the previous member), kind*4 + 2 + parity = "the next member freed its slot[parity]" (raised by it).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int ring_next(const Sig& s) { return s.me + 1 == s.n ? 0 : s.me + 1; }
__device__ __forceinline__ int ring_prev(const Sig& s) { return s.me == 0 ? s.n - 1 : s.me - 1; }

// CTA-uniform: thread 0 waits for the receiver's "free" flag of this channel, the CTA stores its vector range, then thread 0 raises
// the receiver's "arrived" flag after every thread's stores are visible at .sys scope
__device__ __forceinline__ void ring_enter(const Sig& s, int kind, int parity, int wait_free) {
    if (wait_free && threadIdx.x == 0) sig_spin_cas(s.local + blockIdx.x * BG_MAX_PEERS + kind * 4 + 2 + parity, 1u, 0u, false, s);
    __syncthreads();
}
__device__ __forceinline__ void ring_leave(const Sig& s, int kind, int parity) {
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) sig_spin_cas(s.peer[ring_next(s)] + blockIdx.x * BG_MAX_PEERS + kind * 4 + parity, 0u, 1u, true, s);
}

// [k | v] -> the next member's slot; CTA b pushes the b-th contiguous range of the 2 * nvec 16-B vectors
__global__ void BG_SLIM cp_ring_push_kernel(const uint4* __restrict__ k, const uint4* __restrict__ v, uint4* __restrict__ dst,
                                           size_t nvec, int parity, int wait_free, const __grid_constant__ Sig s) {
    ring_enter(s, 0, parity, wait_free);
    const size_t total = 2 * nvec, per = (total + gridDim.x - 1) / gridDim.x;
    const size_t lo = (size_t)blockIdx.x * per, hi = lo + per < total ? lo + per : total;
    for (size_t i0 = lo + threadIdx.x; i0 < hi; i0 += (size_t)kThreads * kUnroll) {
        uint4 regs[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const size_t i = i0 + (size_t)u * kThreads;
            if (i < hi) regs[u] = ld16_stream(i < nvec ? k + i : v + (i - nvec));
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const size_t i = i0 + (size_t)u * kThreads;
            if (i < hi) st16(dst + i, regs[u]);
        }
    }
    ring_leave(s, 0, parity);
}

struct RingAcc {
    const float* acc_in;                 // this member's received accumulators [dK | dV] (nullptr at the first step)
    const __nv_bfloat16* contrib[2];     // the step's dK, dV rows [batch][c_rows][row_elems]
    float* dst;                          // the next member's slot [dK | dV]
    long long rows, row_elems, c_row0, c_rows;
    size_t units;                        // 8-element units per tensor
};

// next = acc_in + contribution, in that order, per element: the sum over the ring has one fixed order (owner, owner + 1, ...)
__global__ void BG_SLIM cp_ring_acc_push_kernel(const __grid_constant__ RingAcc a, int parity, int wait_free, const __grid_constant__ Sig s) {
    ring_enter(s, 1, parity, wait_free);
    const size_t total = 2 * a.units, per = (total + gridDim.x - 1) / gridDim.x;
    const size_t lo = (size_t)blockIdx.x * per, hi = lo + per < total ? lo + per : total;
    const long long blk = a.rows * a.row_elems;
    for (size_t u = lo + threadIdx.x; u < hi; u += kThreads) {
        float f[8];
        if (a.acc_in) {
            const uint4 x = ld16_stream(a.acc_in + u * 8), y = ld16_stream(a.acc_in + u * 8 + 4);
            f[0] = __uint_as_float(x.x); f[1] = __uint_as_float(x.y); f[2] = __uint_as_float(x.z); f[3] = __uint_as_float(x.w);
            f[4] = __uint_as_float(y.x); f[5] = __uint_as_float(y.y); f[6] = __uint_as_float(y.z); f[7] = __uint_as_float(y.w);
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) f[i] = 0.f;
        }
        const int t = u >= a.units;
        const long long e = (long long)(u - (t ? a.units : 0)) * 8;
        const long long bi = e / blk, rem = e - bi * blk, row = rem / a.row_elems;
        if (row >= a.c_row0 && row < a.c_row0 + a.c_rows) {
            float c[8];
            unpack8(ld16_stream(a.contrib[t] + ((bi * a.c_rows + row - a.c_row0) * a.row_elems + (rem - row * a.row_elems))), c);
#pragma unroll
            for (int i = 0; i < 8; ++i) f[i] += c[i];
        }
        st16(a.dst + u * 8, make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3])));
        st16(a.dst + u * 8 + 4, make_uint4(__float_as_uint(f[4]), __float_as_uint(f[5]), __float_as_uint(f[6]), __float_as_uint(f[7])));
    }
    ring_leave(s, 1, parity);
}

// consumer side, on the stream of the kernels that read the slot: wait for every channel's "arrived" flag ...
__global__ void BG_SLIM cp_ring_wait_kernel(int kind, int parity, int channels, const __grid_constant__ Sig s) {
    for (int ch = threadIdx.x; ch < channels; ch += kThreads)
        sig_spin_cas(s.local + ch * BG_MAX_PEERS + kind * 4 + parity, 1u, 0u, false, s);
}
// ... and, once those kernels are done with it, hand the slot back to the previous member
__global__ void BG_SLIM cp_ring_release_kernel(int kind, int parity, int channels, const __grid_constant__ Sig s) {
    __threadfence_system();
    for (int ch = threadIdx.x; ch < channels; ch += kThreads)
        sig_spin_cas(s.peer[ring_prev(s)] + ch * BG_MAX_PEERS + kind * 4 + 2 + parity, 0u, 1u, true, s);
}

}  // namespace

// Every kernel of this file is loaded up front (bg_ctx_create): with CUDA's lazy module loading the FIRST launch of a kernel
// synchronises with the device, and a launch that has to wait for a peer-waiting kernel already in flight (virtual ranks on one
// device; a second stream of the same rank) would stall behind it.
int bg_preload_coll() {
#define K(f) reinterpret_cast<const void*>(&f)
    const void* kernels[] = {
        K(coll_barrier_kernel),
        K(all_to_all_rows_kernel),
        K(cp_ring_push_kernel),
        K(cp_ring_acc_push_kernel),
        K(cp_ring_wait_kernel),
        K(cp_ring_release_kernel),
        K(all_reduce_nvls_kernel<true>),
        K(all_reduce_nvls_kernel<false>),
        K(pair_sum_kernel<true>),
        K(pair_sum_kernel<false>),
        K((all_gather_push_kernel<float, __nv_bfloat16, true>)),
        K((all_gather_push_kernel<float, __nv_bfloat16, false>)),
        K((all_gather_push_kernel<__nv_bfloat16, __nv_bfloat16, true>)),
        K((all_gather_push_kernel<__nv_bfloat16, __nv_bfloat16, false>)),
        K((all_gather_push_kernel<float, float, true>)),
        K((all_gather_push_kernel<float, float, false>)),
        K((reduce_scatter_pull_kernel<2, true, kEpiF32, false>)),
        K((reduce_scatter_pull_kernel<4, true, kEpiF32, false>)),
        K((reduce_scatter_pull_kernel<8, true, kEpiF32, false>)),
        K((reduce_scatter_pull_kernel<2, true, kEpiF32, true>)),
        K((reduce_scatter_pull_kernel<2, true, kEpiBf16, false>)),
        K((reduce_scatter_pull_kernel<4, true, kEpiBf16, false>)),
        K((reduce_scatter_pull_kernel<8, true, kEpiBf16, false>)),
        K((reduce_scatter_pull_kernel<2, true, kEpiBf16, true>)),
        K((reduce_scatter_pull_kernel<2, true, kEpiAdamW, false>)),
        K((reduce_scatter_pull_kernel<4, true, kEpiAdamW, false>)),
        K((reduce_scatter_pull_kernel<8, true, kEpiAdamW, false>)),
        K((reduce_scatter_pull_kernel<2, true, kEpiAdamW, true>)),
        K((reduce_scatter_pull_kernel<2, false, kEpiF32, false>)),
        K((reduce_scatter_pull_kernel<4, false, kEpiF32, false>)),
        K((reduce_scatter_pull_kernel<8, false, kEpiF32, false>)),
        K((reduce_scatter_pull_kernel<2, false, kEpiF32, true>)),
        K((reduce_scatter_pull_kernel<2, false, kEpiAdamW, false>)),
        K((reduce_scatter_pull_kernel<4, false, kEpiAdamW, false>)),
        K((reduce_scatter_pull_kernel<8, false, kEpiAdamW, false>)),
        K((reduce_scatter_pull_kernel<2, false, kEpiAdamW, true>)),
        K((reduce_scatter_pull_kernel<2, true, kEpiSumSq, false>)),
        K((reduce_scatter_pull_kernel<4, true, kEpiSumSq, false>)),
        K((reduce_scatter_pull_kernel<8, true, kEpiSumSq, false>)),
        K((reduce_scatter_pull_kernel<2, true, kEpiSumSq, true>)),
        K((reduce_scatter_pull_kernel<2, false, kEpiSumSq, false>)),
        K((reduce_scatter_pull_kernel<4, false, kEpiSumSq, false>)),
        K((reduce_scatter_pull_kernel<8, false, kEpiSumSq, false>)),
        K((reduce_scatter_pull_kernel<2, false, kEpiSumSq, true>)),
        K((reduce_scatter_pull_kernel<2, true, kEpiAdamWClip, false>)),
        K((reduce_scatter_pull_kernel<4, true, kEpiAdamWClip, false>)),
        K((reduce_scatter_pull_kernel<8, true, kEpiAdamWClip, false>)),
        K((reduce_scatter_pull_kernel<2, true, kEpiAdamWClip, true>)),
        K((reduce_scatter_pull_kernel<2, false, kEpiAdamWClip, false>)),
        K((reduce_scatter_pull_kernel<4, false, kEpiAdamWClip, false>)),
        K((reduce_scatter_pull_kernel<8, false, kEpiAdamWClip, false>)),
        K((reduce_scatter_pull_kernel<2, false, kEpiAdamWClip, true>)),
        K(adamw_local_kernel),
        K((all_reduce_oneshot_kernel<2, true, true>)),
        K((all_reduce_oneshot_kernel<2, true, false>)),
        K((all_reduce_oneshot_kernel<2, false, true>)),
        K((all_reduce_oneshot_kernel<2, false, false>)),
        K((all_reduce_oneshot_kernel<4, true, true>)),
        K((all_reduce_oneshot_kernel<4, true, false>)),
        K((all_reduce_oneshot_kernel<4, false, true>)),
        K((all_reduce_oneshot_kernel<4, false, false>)),
        K((all_reduce_oneshot_kernel<8, true, true>)),
        K((all_reduce_oneshot_kernel<8, true, false>)),
        K((all_reduce_oneshot_kernel<8, false, true>)),
        K((all_reduce_oneshot_kernel<8, false, false>)),
        K((all_reduce_twoshot_kernel<2, true, true>)),
        K((all_reduce_twoshot_kernel<2, true, false>)),
        K((all_reduce_twoshot_kernel<2, false, true>)),
        K((all_reduce_twoshot_kernel<2, false, false>)),
        K((all_reduce_twoshot_kernel<4, true, true>)),
        K((all_reduce_twoshot_kernel<4, true, false>)),
        K((all_reduce_twoshot_kernel<4, false, true>)),
        K((all_reduce_twoshot_kernel<4, false, false>)),
        K((all_reduce_twoshot_kernel<8, true, true>)),
        K((all_reduce_twoshot_kernel<8, true, false>)),
        K((all_reduce_twoshot_kernel<8, false, true>)),
        K((all_reduce_twoshot_kernel<8, false, false>))};
#undef K
    for (const void* k : kernels) {
        cudaFuncAttributes attr;
        BG_CUDA(cudaFuncGetAttributes(&attr, k));
    }
    return BG_OK;
}

// =================================================================================================================
// entry points
// =================================================================================================================
// Every plain collective entry below makes its context-free checks (dtypes, whole 16-B vectors, local pointer alignment,
// descriptor fields) before make_sig, then the group and arena checks; a call that fails any of them has launched nothing.

// bytes = count * unit of a symmetric buffer, refused as resolve() refuses a buffer outside the arena when the product exceeds the
// arena -- checked before it is formed, so an absurd count cannot wrap it to a small size that resolve() would accept
static int sym_bytes(const bg_ctx* c, size_t count, size_t unit, size_t* bytes) {
    if (unit != 0 && count > c->arena_bytes / unit)
        return fail(BG_EINVAL, "symmetric buffer of %zu x %zu B outside arena", count, unit);
    *bytes = count * unit;
    return BG_OK;
}

static int launch_all_gather(bg_ctx_t c, int gid, int lane, const void* src, int src_dtype, const size_t* dst_offs, int dst_dtype,
                             size_t shard_elems, const AgSignal* sg, void* stream) {
    if (!(src_dtype == BG_F32 && dst_dtype == BG_BF16) && !(src_dtype == BG_BF16 && dst_dtype == BG_BF16) &&
        !(src_dtype == BG_F32 && dst_dtype == BG_F32))
        return fail(BG_EUNSUPPORTED, "all_gather_cast %d->%d", src_dtype, dst_dtype);
    const size_t dsz = dst_dtype == BG_BF16 ? 2 : 4;
    const int per = (src_dtype == BG_F32 && dst_dtype == BG_F32) ? 4 : 8;
    if (shard_elems % per) return fail(BG_EINVAL, "shard_elems %zu must be a multiple of %d (pad the flat buffer)", shard_elems, per);
    if ((uintptr_t)src % 16) return fail(BG_EINVAL, "src not 16-B aligned");
    Sig s; const Group* g;
    int rc = make_sig(c, gid, lane, &s, &g);
    if (rc) return rc;
    size_t bytes;
    rc = sym_bytes(c, shard_elems, (size_t)g->n * dsz, &bytes);
    if (rc) return rc;
    PeerPtrs dst;
    rc = resolve(c, *g, dst_offs, bytes, &dst);
    if (rc) return rc;
    if (shard_elems == 0) return BG_OK;
    s.site = sg ? 12 : 1;
    BG_CUDA(cudaSetDevice(c->device));
    char* mc = (sg == nullptr && g_tun.nvls_gather) ? mc_ptr(c, gid, *g, dst_offs, bytes) : nullptr;
    if (mc && shard_elems * dsz < (size_t)g_tun.nvls_min_bytes) mc = nullptr;
    int grid = comm_grid(shard_elems / per / kUnroll + 1, kThreads, g->n);
    cudaStream_t st = (cudaStream_t)stream;
    AgSignal none = {};
#define BG_AG(S, D)                                                                                                            \
    do {                                                                                                                       \
        if (sg) all_gather_push_kernel<S, D, true><<<grid, kThreads, 0, st>>>(dst, nullptr, (const S*)src, shard_elems, *sg, s); \
        else all_gather_push_kernel<S, D, false><<<grid, kThreads, 0, st>>>(dst, mc, (const S*)src, shard_elems, none, s);     \
    } while (0)
    if (src_dtype == BG_F32 && dst_dtype == BG_BF16) BG_AG(float, __nv_bfloat16);
    else if (src_dtype == BG_BF16 && dst_dtype == BG_BF16) BG_AG(__nv_bfloat16, __nv_bfloat16);
    else BG_AG(float, float);
#undef BG_AG
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_all_gather_cast(bg_ctx_t c, int gid, int lane, const void* src, int src_dtype, const size_t* dst_offs,
                                  int dst_dtype, size_t shard_elems, void* stream) {
    return launch_all_gather(c, gid, lane, src, src_dtype, dst_offs, dst_dtype, shard_elems, nullptr, stream);
}

static int launch_reduce_scatter(bg_ctx_t c, int gid, int lane, const size_t* src_offs, int src_dtype, int epi, RsOut o,
                                 size_t shard_elems, float prescale, float postscale, void* stream) {
    if (src_dtype != BG_BF16 && src_dtype != BG_F32) return fail(BG_EUNSUPPORTED, "reduce_scatter src dtype %d", src_dtype);
    const int per = src_dtype == BG_BF16 ? 8 : 4;
    const size_t ssz = src_dtype == BG_BF16 ? 2 : 4;
    if (shard_elems % per) return fail(BG_EINVAL, "shard_elems %zu must be a multiple of %d", shard_elems, per);
    if ((uintptr_t)o.dst % 16) return fail(BG_EINVAL, "dst not 16-B aligned");
    Sig s; const Group* g;
    int rc = make_sig(c, gid, lane, &s, &g);
    if (rc) return rc;
    size_t bytes;
    rc = sym_bytes(c, shard_elems, (size_t)g->n * ssz, &bytes);
    if (rc) return rc;
    PeerPtrs src;
    rc = resolve(c, *g, src_offs, bytes, &src);
    if (rc) return rc;
    if (shard_elems == 0) return BG_OK;
    s.site = 2;
    BG_CUDA(cudaSetDevice(c->device));
    const char* mc = g_tun.nvls_reduce ? mc_ptr(c, gid, *g, src_offs, bytes) : nullptr;
    if (mc && shard_elems * ssz < (size_t)g_tun.nvls_min_bytes) mc = nullptr;
    const bool half = epi == kEpiAdamW || epi == kEpiAdamWClip || epi == kEpiSumSq;
    const int pmax = g->n <= 2 ? 2 : g->n <= 4 ? 4 : 8;
    const int in_flight_vecs = mc ? (half ? 4 : 8) : (half && pmax < 8 ? kInFlight / 2 : kInFlight) / pmax;
    int grid = comm_grid(shard_elems / per / in_flight_vecs + 1, kThreads, g->n);
    if (o.partials != nullptr && (long long)grid * kWarps > o.n_partials)
        return fail(BG_EINVAL, "sum-of-squares partials: %d entries, the launch needs %d", o.n_partials, grid * kWarps);
    cudaStream_t st = (cudaStream_t)stream;
    const bool bf = src_dtype == BG_BF16;
#define BG_RS_EPI(B, E) launch_rs<B, E>(g->n, mc != nullptr, grid, st, src, mc, o, shard_elems, prescale, postscale, s)
    if (bf && epi == kEpiF32) BG_RS_EPI(true, kEpiF32);
    else if (bf && epi == kEpiBf16) BG_RS_EPI(true, kEpiBf16);
    else if (bf && epi == kEpiAdamW) BG_RS_EPI(true, kEpiAdamW);
    else if (bf && epi == kEpiSumSq) BG_RS_EPI(true, kEpiSumSq);
    else if (bf && epi == kEpiAdamWClip) BG_RS_EPI(true, kEpiAdamWClip);
    else if (!bf && epi == kEpiF32) BG_RS_EPI(false, kEpiF32);
    else if (!bf && epi == kEpiAdamW) BG_RS_EPI(false, kEpiAdamW);
    else if (!bf && epi == kEpiSumSq) BG_RS_EPI(false, kEpiSumSq);
    else if (!bf && epi == kEpiAdamWClip) BG_RS_EPI(false, kEpiAdamWClip);
    else return fail(BG_EUNSUPPORTED, "reduce_scatter %d -> epilogue %d", src_dtype, epi);
#undef BG_RS_EPI
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_reduce_scatter_acc(bg_ctx_t c, int gid, int lane, const size_t* src_offs, int src_dtype, void* dst,
                                     int dst_dtype, size_t shard_elems, float prescale, float postscale, int accumulate,
                                     void* stream) {
    RsOut o = {};
    o.dst = dst; o.accumulate = accumulate;
    if (dst_dtype != BG_F32 && dst_dtype != BG_BF16) return fail(BG_EUNSUPPORTED, "reduce_scatter dst dtype %d", dst_dtype);
    if (dst_dtype == BG_BF16 && src_dtype != BG_BF16) return fail(BG_EUNSUPPORTED, "reduce_scatter %d->%d", src_dtype, dst_dtype);
    return launch_reduce_scatter(c, gid, lane, src_offs, src_dtype, dst_dtype == BG_F32 ? kEpiF32 : kEpiBf16, o, shard_elems, prescale,
                                 postscale, stream);
}

// The checks of the three AdamW entries, before any launch.  The hyperparameters are checked as the fp32 values the kernels use
// (torch.optim.AdamW's constructor checks, in fp32): beta1 = 1 would make bias_corr1 0 and every parameter inf or NaN.
static int adam_out(float* param, float* exp_avg, float* exp_avg_sq, float lr, float beta1, float beta2, float eps,
                    float weight_decay, long long step, RsOut* o) {
    if (param == nullptr || exp_avg == nullptr || exp_avg_sq == nullptr)
        return fail(BG_EINVAL, "adamw: param, exp_avg and exp_avg_sq must be non-null");
    if (((uintptr_t)param | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) % 16) return fail(BG_EINVAL, "optimizer state not 16-B aligned");
    if (step < 1) return fail(BG_EINVAL, "adam step must be >= 1");
    if (!(lr >= 0.f && isfinite(lr))) return fail(BG_EINVAL, "adamw: lr %g must be finite and >= 0", lr);
    if (!(eps >= 0.f && isfinite(eps))) return fail(BG_EINVAL, "adamw: eps %g must be finite and >= 0", eps);
    if (!(weight_decay >= 0.f && isfinite(weight_decay)))
        return fail(BG_EINVAL, "adamw: weight_decay %g must be finite and >= 0", weight_decay);
    if (!(beta1 >= 0.f && beta1 < 1.f)) return fail(BG_EINVAL, "adamw: beta1 %g outside [0, 1)", beta1);
    if (!(beta2 >= 0.f && beta2 < 1.f)) return fail(BG_EINVAL, "adamw: beta2 %g outside [0, 1)", beta2);
    o->dst = param; o->exp_avg = exp_avg; o->exp_avg_sq = exp_avg_sq;
    o->a.lr = lr; o->a.beta1 = beta1; o->a.beta2 = beta2; o->a.eps = eps; o->a.weight_decay = weight_decay;
    o->a.bias_corr1 = (float)(1.0 - pow((double)beta1, (double)step));
    o->a.bias_corr2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
    return BG_OK;
}

extern "C" int bg_reduce_scatter_adamw(bg_ctx_t c, int gid, int lane, const size_t* src_offs, int src_dtype, float* param,
                                       float* exp_avg, float* exp_avg_sq, size_t shard_elems, float prescale, float postscale,
                                       float lr, float beta1, float beta2, float eps, float weight_decay, long long step,
                                       void* stream) {
    RsOut o = {};
    int rc = adam_out(param, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, weight_decay, step, &o);
    if (rc) return rc;
    return launch_reduce_scatter(c, gid, lane, src_offs, src_dtype, kEpiAdamW, o, shard_elems, prescale, postscale, stream);
}

extern "C" int bg_reduce_scatter_adamw_clipped(bg_ctx_t c, int gid, int lane, const size_t* src_offs, int src_dtype, float* param,
                                               float* exp_avg, float* exp_avg_sq, size_t shard_elems, float prescale,
                                               float postscale, float lr, float beta1, float beta2, float eps, float weight_decay,
                                               long long step, const float* clip_coef, void* stream) {
    RsOut o = {};
    int rc = adam_out(param, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, weight_decay, step, &o);
    if (rc) return rc;
    o.clip_coef = clip_coef;
    return launch_reduce_scatter(c, gid, lane, src_offs, src_dtype, kEpiAdamWClip, o, shard_elems, prescale, postscale, stream);
}

extern "C" int bg_reduce_scatter_sumsq(bg_ctx_t c, int gid, int lane, const size_t* src_offs, int src_dtype, float* dst,
                                       size_t shard_elems, float prescale, float postscale, float* partials, int n_partials,
                                       const size_t* skip, int n_skip, void* stream) {
    if (partials == nullptr || n_partials < 1) return fail(BG_EINVAL, "sum-of-squares partials missing");
    if (n_skip < 0 || n_skip > BG_MAX_SKIP) return fail(BG_EINVAL, "%d skip ranges (at most %d)", n_skip, BG_MAX_SKIP);
    RsOut o = {};
    o.dst = dst; o.partials = partials; o.n_partials = n_partials; o.n_skip = n_skip;
    for (int r = 0; r < n_skip; ++r) {
        if (skip[2 * r] % 8 || skip[2 * r + 1] % 8 || skip[2 * r] > skip[2 * r + 1])
            return fail(BG_EINVAL, "skip range [%zu, %zu) is not 8-element aligned", skip[2 * r], skip[2 * r + 1]);
        if (skip[2 * r + 1] > shard_elems)
            return fail(BG_EINVAL, "skip range [%zu, %zu) ends past the shard of %zu elements", skip[2 * r], skip[2 * r + 1], shard_elems);
        o.skip_lo[r] = skip[2 * r]; o.skip_hi[r] = skip[2 * r + 1];
    }
    if (dst != nullptr && (uintptr_t)dst % 16) return fail(BG_EINVAL, "dst not 16-B aligned");
    return launch_reduce_scatter(c, gid, lane, src_offs, src_dtype, kEpiSumSq, o, shard_elems, prescale, postscale, stream);
}

extern "C" int bg_adamw_clipped(float* param, float* exp_avg, float* exp_avg_sq, const float* grad, size_t n, float lr, float beta1,
                                float beta2, float eps, float weight_decay, long long step, const float* clip_coef, void* stream) {
    RsOut o = {};
    int rc = adam_out(param, exp_avg, exp_avg_sq, lr, beta1, beta2, eps, weight_decay, step, &o);
    if (rc) return rc;
    if (n % 4 || (uintptr_t)grad % 16) return fail(BG_EINVAL, "adamw: %zu elements / gradient alignment (need multiples of 4, 16 B)", n);
    if (n > 0 && grad == nullptr) return fail(BG_EINVAL, "adamw: null grad");
    if (n == 0) return BG_OK;
    o.clip_coef = clip_coef;
    const int grid = comm_grid(n / 4, kThreads, 1);
    adamw_local_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(grad, o, n);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_all_reduce(bg_ctx_t c, int gid, int lane, const size_t* src_offs, void* dst, size_t elems, int dtype,
                             int redop, float scale, void* stream) {
    if (dtype != BG_BF16 && dtype != BG_F32) return fail(BG_EUNSUPPORTED, "all_reduce dtype %d", dtype);
    if (redop != BG_SUM && redop != BG_MAX) return fail(BG_EUNSUPPORTED, "all_reduce op %d", redop);
    const int per = dtype == BG_BF16 ? 8 : 4;
    const size_t esz = dtype == BG_BF16 ? 2 : 4;
    if (elems % per) return fail(BG_EINVAL, "all_reduce elems %zu must be a multiple of %d (pad)", elems, per);
    if ((uintptr_t)dst % 16) return fail(BG_EINVAL, "dst not 16-B aligned");
    Sig s; const Group* g;
    int rc = make_sig(c, gid, lane, &s, &g);
    if (rc) return rc;
    size_t bytes;
    rc = sym_bytes(c, elems, esz, &bytes);
    if (rc) return rc;
    PeerPtrs src;
    rc = resolve(c, *g, src_offs, bytes, &src);
    if (rc) return rc;
    if (elems == 0) return BG_OK;
    s.site = 3;
    BG_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = (cudaStream_t)stream;
    const size_t nvec = elems / per;
    // large sums on a multicast-bound buffer are reduced and replicated inside the switch
    if (redop == BG_SUM && g->n > 1 && bytes >= (size_t)g_tun.nvls_min_bytes) {
        char* mc = mc_ptr(c, gid, *g, src_offs, bytes);
        if (mc != nullptr) {
            const int grid = comm_grid((nvec + g->n - 1) / g->n / kInFlight + 1, kThreads, g->n);
            if (dtype == BG_BF16) all_reduce_nvls_kernel<true><<<grid, kThreads, 0, st>>>(mc, src.p[g->me], (char*)dst, nvec, scale, s);
            else all_reduce_nvls_kernel<false><<<grid, kThreads, 0, st>>>(mc, src.p[g->me], (char*)dst, nvec, scale, s);
            BG_CHECK_LAUNCH();
            return BG_OK;
        }
    }
    const bool twoshot = g->n > 1 && bytes > (size_t)g_tun.oneshot_bytes && nvec % g->n == 0;
    const bool bf = dtype == BG_BF16, mx = redop == BG_MAX;
#define BG_AR_P(KERNEL, P, NV)                                                                            \
    do {                                                                                                  \
        if (bf && !mx) KERNEL<P, true, false><<<grid, kThreads, 0, st>>>(src, dst, (NV), scale, s);       \
        else if (bf && mx) KERNEL<P, true, true><<<grid, kThreads, 0, st>>>(src, dst, (NV), scale, s);    \
        else if (!bf && !mx) KERNEL<P, false, false><<<grid, kThreads, 0, st>>>(src, dst, (NV), scale, s); \
        else KERNEL<P, false, true><<<grid, kThreads, 0, st>>>(src, dst, (NV), scale, s);                 \
    } while (0)
#define BG_AR_DISPATCH(KERNEL, NV, PER_ITER)                                  \
    do {                                                                      \
        int grid = comm_grid((NV) / (PER_ITER) + 1, kThreads, g->n);          \
        if (g->n <= 2) BG_AR_P(KERNEL, 2, NV);                                \
        else if (g->n <= 4) BG_AR_P(KERNEL, 4, NV);                           \
        else BG_AR_P(KERNEL, 8, NV);                                          \
    } while (0)
    if (twoshot) BG_AR_DISPATCH(all_reduce_twoshot_kernel, nvec / g->n, kInFlight / (g->n <= 2 ? 2 : g->n <= 4 ? 4 : 8));
    else BG_AR_DISPATCH(all_reduce_oneshot_kernel, nvec, 1);
#undef BG_AR_DISPATCH
#undef BG_AR_P
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_pair_sum_inplace(bg_ctx_t c, int gid, int lane, const size_t* offs, size_t elems, int dtype, float scale, void* stream) {
    if (dtype != BG_BF16 && dtype != BG_F32) return fail(BG_EUNSUPPORTED, "bg_pair_sum_inplace dtype %d", dtype);
    const int per = dtype == BG_BF16 ? 8 : 4;
    if (elems % per) return fail(BG_EINVAL, "bg_pair_sum_inplace: elems %zu is not a whole number of 16-B vectors (%d elements)", elems, per);
    Sig s; const Group* g;
    int rc = make_sig(c, gid, lane, &s, &g);
    if (rc) return rc;
    if (g->n != 2) return fail(BG_EINVAL, "bg_pair_sum_inplace: group of %d member(s), needs exactly 2", g->n);
    size_t bytes;
    rc = sym_bytes(c, elems, dtype == BG_BF16 ? 2 : 4, &bytes);
    if (rc) return rc;
    PeerPtrs buf;
    rc = resolve(c, *g, offs, bytes, &buf);
    if (rc) return rc;
    if (elems == 0) return BG_OK;
    s.site = 17;
    BG_CUDA(cudaSetDevice(c->device));
    const size_t nvec = elems / per, half = (nvec + 1) / 2;
    const size_t lo = g->me == 0 ? 0 : half, hi = g->me == 0 ? half : nvec;
    const int grid = comm_grid(half / (kInFlight / 2) + 1, kThreads, g->n);     // the same on both members
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == BG_BF16) pair_sum_kernel<true><<<grid, kThreads, 0, st>>>(buf, lo, hi, scale, s);
    else pair_sum_kernel<false><<<grid, kThreads, 0, st>>>(buf, lo, hi, scale, s);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_all_to_all_rows(bg_ctx_t c, int gid, int lane, const bg_a2a_desc* descs, int n_descs, int dtype,
                                  void* stream) {
    if (!descs || n_descs < 1 || n_descs > kMaxA2A) return fail(BG_EINVAL, "1..%d tensors per all_to_all launch", kMaxA2A);
    if (dtype != BG_BF16 && dtype != BG_F32) return fail(BG_EUNSUPPORTED, "all_to_all dtype %d", dtype);
    const long long esz = dtype == BG_BF16 ? 2 : 4, per = 16 / esz;
    for (int i = 0; i < n_descs; ++i) {
        const bg_a2a_desc& d = descs[i];
        if (d.batch < 0 || d.rows < 0 || d.row_elems < 0 || d.src_bs < 0 || d.src_rs < 0 || d.src_me_off < 0 || d.dst_bs < 0 ||
            d.dst_rs < 0 || d.dst_peer_off < 0)
            return fail(BG_EINVAL, "all_to_all: negative extent or stride");
        if (d.row_elems % per || d.src_bs % per || d.src_rs % per || d.src_me_off % per || d.dst_bs % per ||
            d.dst_rs % per || d.dst_peer_off % per)
            return fail(BG_EINVAL, "all_to_all: strides/row length must be multiples of %lld elements", per);
        if ((uintptr_t)d.dst % 16) return fail(BG_EINVAL, "all_to_all dst not 16-B aligned");
        // the kernel indexes a tensor's vectors of one peer with 32-bit counters
        const unsigned long long lim = 1ull << 32, b = d.batch, r = d.rows, v = d.row_elems / per;
        if (b && r && v && (b >= lim || r >= lim || v >= lim || b * r >= lim || b * r * v >= lim))
            return fail(BG_EINVAL, "all_to_all: more than 2^32 16-B vectors per peer");
    }
    Sig s; const Group* g;
    int rc = make_sig(c, gid, lane, &s, &g);
    if (rc) return rc;
    A2AArgs a;
    a.n_tensors = n_descs;
    size_t max_vec = 0;
    for (int i = 0; i < n_descs; ++i) {
        const bg_a2a_desc& d = descs[i];
        // extent of the peer's source that may be touched (none for an empty tensor); 128-bit, so huge strides cannot wrap it
        // under the arena size
        const bool empty = d.batch == 0 || d.rows == 0 || d.row_elems == 0;
        const unsigned __int128 span = empty ? 0 : (unsigned __int128)(d.batch - 1) * d.src_bs + (unsigned __int128)(d.rows - 1) * d.src_rs +
                                                       (unsigned __int128)(g->n - 1) * d.src_me_off + d.row_elems;
        const unsigned __int128 bytes = span * esz;
        rc = resolve(c, *g, d.src_offs, bytes > (unsigned __int128)SIZE_MAX ? SIZE_MAX : (size_t)bytes, &a.t[i].src);
        if (rc) return rc;
        a.t[i].dst = (char*)d.dst;
        a.t[i].batch = d.batch; a.t[i].rows = d.rows; a.t[i].row_vec = d.row_elems / per;
        a.t[i].src_bs = d.src_bs / per; a.t[i].src_rs = d.src_rs / per; a.t[i].src_me_off = d.src_me_off / per;
        a.t[i].dst_bs = d.dst_bs / per; a.t[i].dst_rs = d.dst_rs / per; a.t[i].dst_peer_off = d.dst_peer_off / per;
        a.t[i].total_vec = d.batch * d.rows * a.t[i].row_vec * g->n;
        if ((size_t)(a.t[i].total_vec / g->n) > max_vec) max_vec = (size_t)(a.t[i].total_vec / g->n);
    }
    s.site = 6;
    BG_CUDA(cudaSetDevice(c->device));
    int grid = comm_grid(max_vec / kInFlight + 1, kThreads, g->n);
    all_to_all_rows_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(a, s);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

// ------------------------------------------------------------------------------------------------
// C15: ring context parallelism
// ------------------------------------------------------------------------------------------------
// channels of a hop: a function of the per-tensor element count only, so a push and its wait / release agree
static int ring_channels(int kind, size_t elems) {
    const size_t work = kind == 0 ? 2 * elems / 8 / kUnroll : 2 * elems / 8;
    return comm_grid(work + 1, kThreads, 2);
}

static int ring_sig(bg_ctx_t c, int gid, int parity, Sig* s, const Group** g, int site) {
    int rc = make_sig(c, gid, BG_LANE_RING, s, g);
    if (rc) return rc;
    if ((*g)->n < 2) return fail(BG_EINVAL, "cp ring: group of %d member(s)", (*g)->n);
    if (parity != 0 && parity != 1) return fail(BG_EINVAL, "cp ring: parity %d", parity);
    s->site = site;
    BG_CUDA(cudaSetDevice(c->device));
    return BG_OK;
}

extern "C" int bg_cp_ring_push(bg_ctx_t c, int gid, int parity, int wait_free, const void* k, const void* v, size_t elems,
                               const size_t* slot_offs, void* stream) {
    Sig s; const Group* g;
    int rc = ring_sig(c, gid, parity, &s, &g, 13);
    if (rc) return rc;
    if (elems % 8 || (uintptr_t)k % 16 || (uintptr_t)v % 16) return fail(BG_EINVAL, "bg_cp_ring_push: elems %% 8, 16-B aligned k / v");
    PeerPtrs dst;
    rc = resolve(c, *g, slot_offs, 2 * elems * 2, &dst);
    if (rc) return rc;
    const int next = g->me + 1 == g->n ? 0 : g->me + 1;
    cp_ring_push_kernel<<<ring_channels(0, elems), kThreads, 0, (cudaStream_t)stream>>>(
        (const uint4*)k, (const uint4*)v, (uint4*)dst.p[next], elems / 8, parity, wait_free, s);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_cp_ring_acc_push(bg_ctx_t c, int gid, int parity, int wait_free, const float* acc_in, const void* dk, const void* dv,
                                   long long batch, long long rows, long long row_elems, long long c_row0, long long c_rows,
                                   const size_t* slot_offs, void* stream) {
    Sig s; const Group* g;
    int rc = ring_sig(c, gid, parity, &s, &g, 16);
    if (rc) return rc;
    if (batch < 1 || rows < 1 || row_elems < 8 || row_elems % 8 || c_row0 < 0 || c_rows < 0 || c_row0 + c_rows > rows)
        return fail(BG_EINVAL, "bg_cp_ring_acc_push: bad shape (%lld, %lld, %lld) rows %lld+%lld", batch, rows, row_elems, c_row0, c_rows);
    if ((uintptr_t)acc_in % 16 || (uintptr_t)dk % 16 || (uintptr_t)dv % 16 || (c_rows && (!dk || !dv)))
        return fail(BG_EINVAL, "bg_cp_ring_acc_push: 16-B aligned operands");
    const size_t elems = (size_t)(batch * rows * row_elems);
    PeerPtrs dst;
    rc = resolve(c, *g, slot_offs, 2 * elems * 4, &dst);
    if (rc) return rc;
    RingAcc a;
    a.acc_in = acc_in;
    a.contrib[0] = (const __nv_bfloat16*)dk; a.contrib[1] = (const __nv_bfloat16*)dv;
    a.dst = (float*)dst.p[g->me + 1 == g->n ? 0 : g->me + 1];
    a.rows = rows; a.row_elems = row_elems; a.c_row0 = c_row0; a.c_rows = c_rows;
    a.units = elems / 8;
    cp_ring_acc_push_kernel<<<ring_channels(1, elems), kThreads, 0, (cudaStream_t)stream>>>(a, parity, wait_free, s);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_cp_ring_wait(bg_ctx_t c, int gid, int kind, int parity, size_t elems, void* stream) {
    Sig s; const Group* g;
    int rc = ring_sig(c, gid, parity, &s, &g, 14);
    if (rc) return rc;
    if (kind != 0 && kind != 1) return fail(BG_EINVAL, "bg_cp_ring_wait: kind %d", kind);
    cp_ring_wait_kernel<<<1, kThreads, 0, (cudaStream_t)stream>>>(kind, parity, ring_channels(kind, elems), s);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_cp_ring_release(bg_ctx_t c, int gid, int kind, int parity, size_t elems, void* stream) {
    Sig s; const Group* g;
    int rc = ring_sig(c, gid, parity, &s, &g, 15);
    if (rc) return rc;
    if (kind != 0 && kind != 1) return fail(BG_EINVAL, "bg_cp_ring_release: kind %d", kind);
    cp_ring_release_kernel<<<1, kThreads, 0, (cudaStream_t)stream>>>(kind, parity, ring_channels(kind, elems), s);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

// ------------------------------------------------------------------------------------------------
// fused GEMM + collective entry points (kernels in bg_gemm.cu)
// ------------------------------------------------------------------------------------------------
// The checks every fused GEMM entry makes before it touches the context: layout in [0, max_layout], m, n, k positive multiples
// of 8 (TMA needs 16-B row strides), and the local operands 16-B aligned (TMA bases; the tile reducer's 16-B stores into out).
static int fused_gemm_args(const char* who, int layout, int max_layout, long long m, long long n, long long k, const void* p0,
                           const void* p1, const void* p2, const char* names) {
    if (layout < 0 || layout > max_layout) return fail(BG_EINVAL, "%s: layout %d", who, layout);
    if (m <= 0 || n <= 0 || k <= 0 || m % 8 || n % 8 || k % 8)
        return fail(BG_EINVAL, "%s: m,n,k (%lld,%lld,%lld) must be positive multiples of 8", who, m, n, k);
    if (((uintptr_t)p0 | (uintptr_t)p1 | (uintptr_t)p2) % 16) return fail(BG_EINVAL, "%s: %s must be 16-B aligned", who, names);
    return BG_OK;
}

// ... and the checks that need the group: at least two members, and M split into whole 128-row blocks per member
static int fused_gemm_group(const char* who, const Group& g, long long m) {
    if (g.n < 2) return fail(BG_EINVAL, "%s needs a group of >= 2 ranks (use bg_gemm_bf16)", who);
    if (m % ((long long)g.n * 128)) return fail(BG_EINVAL, "%s: M=%lld must be a multiple of p*128", who, m);
    return BG_OK;
}

static size_t scatter_flag_count(long long m, long long n, int p) { return (size_t)((m / p + 127) / 128) * ((n + 127) / 128); }

// C5/C8 fused: GEMM whose epilogue reduce-scatters over the group (wgmma tiles -> peer HBM -> tile reducer)
extern "C" int bg_gemm_reduce_scatter(bg_ctx_t c, int gid, int lane, const void* a, const void* b, long long m, long long n,
                                      long long k, int layout, const size_t* partial_offs, const size_t* flag_offs, void* out,
                                      void* stream) {
    static const char* who = "bg_gemm_reduce_scatter";
    int rc = fused_gemm_args(who, layout, 2, m, n, k, a, b, out, "a, b and out");
    if (rc) return rc;
    Sig s; const Group* g;
    rc = make_sig(c, gid, lane, &s, &g);
    if (rc) return rc;
    rc = fused_gemm_group(who, *g, m);
    if (rc) return rc;
    PeerPtrs partial, flags;
    rc = resolve(c, *g, partial_offs, (size_t)m * n * 2, &partial);
    if (rc) return rc;
    rc = resolve(c, *g, flag_offs, scatter_flag_count(m, n, g->n) * sizeof(uint32_t), &flags);
    if (rc) return rc;
    BG_CUDA(cudaSetDevice(c->device));
    void* pp[BG_MAX_PEERS]; uint32_t* fp[BG_MAX_PEERS];
    for (int i = 0; i < BG_MAX_PEERS; ++i) { pp[i] = partial.p[i]; fp[i] = (uint32_t*)flags.p[i]; }
    FusedGemmMaps maps;
    rc = bg_gemm_scatter_maps(&maps, a, b, m, n, k, layout, g->n, pp);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    // Entry barrier: every member's previous use of the partial buffers and counters (its last reducer, earlier in this same
    // stream) has drained before any peer may store into them again.
    s.site = 7;
    coll_barrier_kernel<<<1, 32, 0, st>>>(s);
    BG_CHECK_LAUNCH();
    return bg_gemm_scatter_launch(maps, m, n, k, layout, g->n, g->me, pp, fp, out, nullptr, nullptr,
                                  (unsigned long long)g_tun.timeout_ms * 1000000ull, c->err_dev, st);
}

// C5/C6 fused: GEMM + ALL-REDUCE.  Two-shot with both shots inside the fused operation: the GEMM epilogue scatters partial tiles
// to their owners (as above), the owner's tile reducer sums a tile as soon as its p partials have landed and immediately
// broadcasts the result rows into EVERY member's `out` buffer (peer stores, or one multimem.st when `out` is multicast-bound);
// the reducers leave through a cross-rank barrier, so `out` is complete on every member in stream order.
extern "C" int bg_gemm_all_reduce(bg_ctx_t c, int gid, int lane, const void* a, const void* b, long long m, long long n, long long k,
                                  int layout, const size_t* partial_offs, const size_t* flag_offs, const size_t* out_offs, void* stream) {
    static const char* who = "bg_gemm_all_reduce";
    int rc = fused_gemm_args(who, layout, 2, m, n, k, a, b, nullptr, "a and b");
    if (rc) return rc;
    Sig s; const Group* g;
    rc = make_sig(c, gid, lane, &s, &g);
    if (rc) return rc;
    rc = fused_gemm_group(who, *g, m);
    if (rc) return rc;
    PeerPtrs partial, flags, outs;
    rc = resolve(c, *g, partial_offs, (size_t)m * n * 2, &partial);
    if (rc) return rc;
    rc = resolve(c, *g, flag_offs, scatter_flag_count(m, n, g->n) * sizeof(uint32_t), &flags);
    if (rc) return rc;
    rc = resolve(c, *g, out_offs, (size_t)m * n * 2, &outs);
    if (rc) return rc;
    BG_CUDA(cudaSetDevice(c->device));
    void* pp[BG_MAX_PEERS]; uint32_t* fp[BG_MAX_PEERS]; void* op[BG_MAX_PEERS];
    for (int i = 0; i < BG_MAX_PEERS; ++i) { pp[i] = partial.p[i]; fp[i] = (uint32_t*)flags.p[i]; op[i] = outs.p[i]; }
    FusedGemmMaps maps;
    rc = bg_gemm_scatter_maps(&maps, a, b, m, n, k, layout, g->n, pp);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    s.site = 7;
    coll_barrier_kernel<<<1, 32, 0, st>>>(s);     // previous users of partial / out / counters have drained on every member
    BG_CHECK_LAUNCH();
    s.site = 8;                                   // the reducers' exit barrier
    char* mc = g_tun.nvls_bcast ? mc_ptr(c, gid, *g, out_offs, (size_t)m * n * 2) : nullptr;
    rc = bg_gemm_scatter_launch(maps, m, n, k, layout, g->n, g->me, pp, fp, outs.p[g->me], op, mc,
                                (unsigned long long)g_tun.timeout_ms * 1000000ull, c->err_dev, st);
    if (rc) return rc;
    // Exit barrier, behind the reducer in the stream: my rows are in every member's result (the reducer grid has completed, its
    // stores are flushed; the barrier's release makes them visible at .sys scope) and every member's rows are in mine.
    coll_barrier_kernel<<<1, 32, 0, st>>>(s);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

// C7 fused: ALL-GATHER + GEMM.  C[M,N] = gather_M(A_local) op B: the slim push kernel (comm_stream, beside the GEMM) sends the
// local M/p rows of A to every member's staging buffer in 128-row chunks and counts each chunk in on the receiver; the GEMM's
// TMA producer takes the rank's own rows straight from a_local and every remote 128-row block from the staging slot as soon as
// its counter is complete, walking the blocks in arrival order.  The counters are cleared behind the GEMM.
extern "C" int bg_all_gather_gemm(bg_ctx_t c, int gid, int lane, const void* a_local, const size_t* stage_offs, const size_t* flag_offs,
                                  const void* b, void* out, long long m, long long n, long long k, int layout, void* stream,
                                  void* comm_stream) {
    static const char* who = "bg_all_gather_gemm";
    int rc = fused_gemm_args(who, layout, 1, m, n, k, a_local, b, out, "a_local, b and c");
    if (rc) return rc;
    Sig s; const Group* g;
    rc = make_sig(c, gid, lane, &s, &g);
    if (rc) return rc;
    rc = fused_gemm_group(who, *g, m);
    if (rc) return rc;
    const int p = g->n;
    const long long rows_local = m / p;
    const int n_chunks = (int)(rows_local / 128);
    PeerPtrs stage, flags;
    rc = resolve(c, *g, stage_offs, (size_t)m * k * 2, &stage);
    if (rc) return rc;
    rc = resolve(c, *g, flag_offs, (size_t)p * n_chunks * sizeof(uint32_t), &flags);
    if (rc) return rc;
    BG_CUDA(cudaSetDevice(c->device));
    FusedGemmMaps maps;
    rc = bg_gemm_gather_maps(&maps, a_local, stage.p[g->me], b, out, m, n, k, layout, p);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream, cs = (cudaStream_t)comm_stream;
    cudaEvent_t ev_in, ev_out;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        if (c->events.empty()) {
            c->events.resize(16);
            for (auto& e : c->events) BG_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        }
        ev_in = c->events[c->event_i++ % c->events.size()];
        ev_out = c->events[c->event_i++ % c->events.size()];
    }
    BG_CUDA(cudaEventRecord(ev_in, st));                 // a_local is produced by the work already in `stream`
    BG_CUDA(cudaStreamWaitEvent(cs, ev_in, 0));
    s.site = 12;
    AgSignal sg = {};
    for (int i = 0; i < p; ++i) sg.flag[i] = (uint32_t*)flags.p[i];
    sg.chunk_vecs = (size_t)128 * k * 2 / 16;
    sg.n_chunks = n_chunks;
    // a chunk is cut into `split` units (each pushed and counted in by one CTA) so that all CTAs of the push kernel are busy
    // from the first chunk on: the largest power of two with n_chunks * split <= comm_ctas, at least 8 rows per unit
    sg.split = 1;
    while (sg.split < 16 && (long long)n_chunks * sg.split * 2 <= g_tun.comm_ctas) sg.split *= 2;
    const size_t shard_elems = (size_t)rows_local * k;
    int grid = (int)((long long)n_chunks * sg.split < g_tun.comm_ctas ? (long long)n_chunks * sg.split : g_tun.comm_ctas);
    {
        PeerPtrs dst = stage;
        all_gather_push_kernel<__nv_bfloat16, __nv_bfloat16, true><<<grid, kThreads, 0, cs>>>(dst, nullptr, (const __nv_bfloat16*)a_local,
                                                                                             shard_elems, sg, s);
        BG_CHECK_LAUNCH();
    }
    BG_CUDA(cudaEventRecord(ev_out, cs));
    rc = bg_gemm_gather_launch(maps, m, n, k, layout, p, g->me, (const uint32_t*)flags.p[g->me], (uint32_t)sg.split,
                               (unsigned long long)g_tun.timeout_ms * 1000000ull, c->err_dev, st);
    if (rc) return rc;
    BG_CUDA(cudaMemsetAsync(flags.p[g->me], 0, (size_t)p * n_chunks * sizeof(uint32_t), st));   // peers count again only after the next entry barrier
    BG_CUDA(cudaStreamWaitEvent(st, ev_out, 0));          // a_local may be reused once the push has read it
    return BG_OK;
}

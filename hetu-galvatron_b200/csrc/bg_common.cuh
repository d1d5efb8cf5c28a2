// Shared helpers for the bg_galvatron C-ABI library (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <string>

#include "bg_galvatron.h"

namespace bg {

extern thread_local std::string g_last_error;
extern std::atomic<unsigned long long> g_launches;

int fail(int code, const char* fmt, ...);

#define BG_CUDA(expr)                                                                            \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess) return bg::fail(BG_ECUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
    } while (0)

#define BG_CHECK_LAUNCH()                                                                  \
    do {                                                                                   \
        cudaError_t _e = cudaGetLastError();                                               \
        if (_e != cudaSuccess) return bg::fail(BG_ECUDA, "launch: %s", cudaGetErrorString(_e)); \
        bg::g_launches.fetch_add(1, std::memory_order_relaxed);                            \
    } while (0)

struct Tunables {
    long long comm_ctas = 132;     // CTAs of a cross-rank kernel (<= BG_MAX_CHANNELS): ONE slim CTA (128 thr x <= 64 regs) per SM
    long long local_ctas = 132 * 8;  // CTAs of a purely local streaming kernel
    long long timeout_ms = 60000;  // device-side barrier timeout
    long long oneshot_bytes = 512 * 1024;
    long long nvls_min_bytes = 1 << 20;  // below this the peer-to-peer kernels win (latency)
    long long nvls_min_ranks = 4;        // groups smaller than this keep the peer-to-peer kernels (measured at p = 2: no gain from the switch)
    long long nvls_gather = 0;     // all-gather stores through the switch (multimem.st) when the buffer is multicast-bound: off, p peer
                                   // stores are the default path
    long long nvls_bcast = 1;      // the fused GEMM + all-reduce reducer writes a summed tile into every member's copy with ONE multimem.st
    long long nvls_reduce = 1;     // reduce-scatter loads are reduced in the switch (multimem.ld_reduce) when the buffer is multicast-bound
};
extern Tunables g_tun;

// ---- 16-byte vector access -------------------------------------------------------------------
__device__ __forceinline__ uint4 ld16_stream(const void* p) {  // local HBM, read once
    uint4 v;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint4 ld16_peer(const void* p) {  // peer HBM over NVLink (never via stale L1)
    uint4 v;
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st16(void* p, const uint4& v) {
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st16_stream(void* p, const uint4& v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w) : "memory");
}

__device__ __forceinline__ float2 bf2_to_f2(uint32_t u) {
    float2 f;
    f.x = __uint_as_float(u << 16);
    f.y = __uint_as_float(u & 0xffff0000u);
    return f;
}
__device__ __forceinline__ uint32_t f2_to_bf2(float a, float b) {  // round-to-nearest-even, as Tensor.to()
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
    float2 a = bf2_to_f2(v.x), b = bf2_to_f2(v.y), c = bf2_to_f2(v.z), d = bf2_to_f2(v.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float* f) {
    uint4 v;
    v.x = f2_to_bf2(f[0], f[1]); v.y = f2_to_bf2(f[2], f[3]); v.z = f2_to_bf2(f[4], f[5]); v.w = f2_to_bf2(f[6], f[7]);
    return v;
}

// ---- Philox4x32-10 (Salmon et al., SC'11; the generator of curand_philox4x32_x.h) -----------------------------------------
// Counter-based: the output is a pure function of (counter, key), so a dropout mask needs no state and no stored bits.
__host__ __device__ __forceinline__ uint32_t philox_mulhi(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}
__host__ __device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        if (i) { k.x += 0x9E3779B9u; k.y += 0xBB67AE85u; }
        const uint32_t hi0 = philox_mulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = philox_mulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    }
    return c;
}

}  // namespace bg

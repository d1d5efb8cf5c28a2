// bg_ops.cu -- local fused elementwise / row kernels that sit next to the collectives on the layer path
// (SURVEY 2.3 rows K5 RMSNorm, K6 swiglu, K9 RoPE + the split/transposes of transformer.py:731-867,
//  a10 vocab-parallel cross-entropy).  All HBM-bound: 16-B vector access, fp32 math, one rounding to bf16.
#include "bg_common.cuh"
#include <type_traits>

using namespace bg;

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// block-wide all-reduce through shared memory; safe to call repeatedly
template <bool kMax>
__device__ __forceinline__ float block_reduce(float v, float* smem) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
    v = kMax ? warp_max(v) : warp_sum(v);
    __syncthreads();
    if (lane == 0) smem[warp] = v;
    __syncthreads();
    float r = (lane < nwarp) ? smem[lane] : (kMax ? -INFINITY : 0.f);
    r = kMax ? warp_max(r) : warp_sum(r);
    return r;
}

// the 8 fp32 column partials of 16-B vector c in row `row` of a [rows][nvec * 8] partial array, as two float4 stores
__device__ __forceinline__ void store_partial8(float* base, size_t row, int nvec, int c, const float acc[8]) {
    float4* p = reinterpret_cast<float4*>(base + (row * nvec + c) * 8);
    p[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    p[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// the 8 bias columns of 16-B vector c (bf16 or fp32 bias); a null bias gives zeros
template <bool kBiasF32>
__device__ __forceinline__ void load_bias8(const void* bias, int c, float out[8]) {
    if (bias == nullptr) {
#pragma unroll
        for (int i = 0; i < 8; ++i) out[i] = 0.f;
    } else if (kBiasF32) {
        const float4* bp = reinterpret_cast<const float4*>(bias) + 2 * c;
        const float4 b0 = __ldg(bp), b1 = __ldg(bp + 1);
        out[0] = b0.x; out[1] = b0.y; out[2] = b0.z; out[3] = b0.w; out[4] = b1.x; out[5] = b1.y; out[6] = b1.z; out[7] = b1.w;
    } else {
        unpack8(__ldg(reinterpret_cast<const uint4*>(bias) + c), out);
    }
}

// f[k] = keep bit k ? f[k] * scale : 0, the product rounded once (no FMA contraction with what follows)
__device__ __forceinline__ void apply_keep8(float f[8], unsigned keep, float scale) {
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = (keep >> k) & 1u ? __fmul_rn(f[k], scale) : 0.f;
}

int local_grid(size_t items, int threads) {
    long long want = (long long)((items + threads - 1) / threads);
    if (want < 1) want = 1;
    return (int)(want < g_tun.local_ctas ? want : g_tun.local_ctas);
}

// ---------------------------------------------------------------------------------------------
// cast / scale / accumulate:  dst = [dst +] src * scale
// ---------------------------------------------------------------------------------------------
template <bool kSrcBf16, bool kDstBf16>
__global__ void __launch_bounds__(kThreads) cast_kernel(const void* __restrict__ src, void* __restrict__ dst, size_t nvec8,
                                                        float scale, int accumulate) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec8; v += stride) {
        float f[8];
        if (kSrcBf16) {
            unpack8(ld16_stream(reinterpret_cast<const uint4*>(src) + v), f);
        } else {
            uint4 a = ld16_stream(reinterpret_cast<const uint4*>(src) + 2 * v), b = ld16_stream(reinterpret_cast<const uint4*>(src) + 2 * v + 1);
            f[0] = __uint_as_float(a.x); f[1] = __uint_as_float(a.y); f[2] = __uint_as_float(a.z); f[3] = __uint_as_float(a.w);
            f[4] = __uint_as_float(b.x); f[5] = __uint_as_float(b.y); f[6] = __uint_as_float(b.z); f[7] = __uint_as_float(b.w);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) f[i] *= scale;
        if (kDstBf16) {
            uint4* d = reinterpret_cast<uint4*>(dst) + v;
            if (accumulate) {
                float o[8];
                unpack8(*d, o);
#pragma unroll
                for (int i = 0; i < 8; ++i) f[i] += o[i];
            }
            st16(d, pack8(f));
        } else {
            float4* d = reinterpret_cast<float4*>(dst) + 2 * v;
            float4 lo = make_float4(f[0], f[1], f[2], f[3]), hi = make_float4(f[4], f[5], f[6], f[7]);
            if (accumulate) {
                float4 a = d[0], b = d[1];
                lo.x += a.x; lo.y += a.y; lo.z += a.z; lo.w += a.w;
                hi.x += b.x; hi.y += b.y; hi.z += b.z; hi.w += b.w;
            }
            d[0] = lo; d[1] = hi;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// RMSNorm (flash_attn.ops.rms_norm semantics: fp32 math, y = x * rstd * w, one rounding)
// ---------------------------------------------------------------------------------------------
constexpr int kMaxVpt = 4;  // register-resident row up to 256 * 8 * 4 = 8192 columns

// VPT = 16-B vectors per thread (1, 2 or 4: the row stays in registers); the NEXT row of the CTA is requested before the current
// one is reduced, so the loads of a CTA never drain while it sits in the two block-wide barriers.
template <int VPT>
__global__ void __launch_bounds__(kThreads) rmsnorm_fwd_kernel(const uint4* __restrict__ x, const uint4* __restrict__ w,
                                                               uint4* __restrict__ y, float* __restrict__ rstd_out,
                                                               long long rows, int nvec, float eps) {
    __shared__ float smem[32];
    uint4 cur[VPT], nxt[VPT];
    long long r = blockIdx.x;
    if (r < rows) {
#pragma unroll
        for (int j = 0; j < VPT; ++j) {
            const int v = threadIdx.x + j * kThreads;
            if (v < nvec) cur[j] = ld16_stream(x + r * nvec + v);
        }
    }
    for (; r < rows; r += gridDim.x) {
        const long long rn = r + gridDim.x;
        if (rn < rows) {
#pragma unroll
            for (int j = 0; j < VPT; ++j) {
                const int v = threadIdx.x + j * kThreads;
                if (v < nvec) nxt[j] = ld16_stream(x + rn * nvec + v);
            }
        }
        float ss = 0.f;
#pragma unroll
        for (int j = 0; j < VPT; ++j) {
            const int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
                float f[8];
                unpack8(cur[j], f);
#pragma unroll
                for (int i = 0; i < 8; ++i) ss += f[i] * f[i];
            }
        }
        ss = block_reduce<false>(ss, smem);
        const float rstd = rsqrtf(ss / (float)(nvec * 8) + eps);
        if (threadIdx.x == 0 && rstd_out) rstd_out[r] = rstd;
#pragma unroll
        for (int j = 0; j < VPT; ++j) {
            const int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
                float f[8], g[8];
                unpack8(cur[j], f);
                unpack8(__ldg(w + v), g);
#pragma unroll
                for (int i = 0; i < 8; ++i) f[i] = f[i] * rstd * g[i];
                st16(y + r * nvec + v, pack8(f));
            }
        }
#pragma unroll
        for (int j = 0; j < VPT; ++j) cur[j] = nxt[j];
    }
}

// dx = rstd * (dy*w - xhat * mean(dy*w*xhat)),  dw_partial[cta] = sum over the CTA's rows of dy * xhat
template <int VPT>
__global__ void __launch_bounds__(kThreads) rmsnorm_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x,
                                                               const uint4* __restrict__ w, const float* __restrict__ rstd_in,
                                                               uint4* __restrict__ dx, float* __restrict__ dw_partial,
                                                               long long rows, int nvec) {
    __shared__ float smem[32];
    float dw[VPT][8];
#pragma unroll
    for (int j = 0; j < VPT; ++j)
#pragma unroll
        for (int i = 0; i < 8; ++i) dw[j][i] = 0.f;
    uint4 cx[VPT], cg[VPT], nx[VPT], ng[VPT];
    long long r = blockIdx.x;
    if (r < rows) {
#pragma unroll
        for (int j = 0; j < VPT; ++j) {
            const int v = threadIdx.x + j * kThreads;
            if (v < nvec) { cx[j] = ld16_stream(x + r * nvec + v); cg[j] = ld16_stream(dy + r * nvec + v); }
        }
    }
    for (; r < rows; r += gridDim.x) {
        const long long rn = r + gridDim.x;
        if (rn < rows) {
#pragma unroll
            for (int j = 0; j < VPT; ++j) {
                const int v = threadIdx.x + j * kThreads;
                if (v < nvec) { nx[j] = ld16_stream(x + rn * nvec + v); ng[j] = ld16_stream(dy + rn * nvec + v); }
            }
        }
        const float rstd = rstd_in[r];
        float dot = 0.f;
#pragma unroll
        for (int j = 0; j < VPT; ++j) {
            const int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
                float xh[8], g[8], wv[8];
                unpack8(cx[j], xh);
                unpack8(cg[j], g);
                unpack8(__ldg(w + v), wv);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    xh[i] *= rstd;
                    dw[j][i] += g[i] * xh[i];
                    dot += g[i] * wv[i] * xh[i];
                }
            }
        }
        dot = block_reduce<false>(dot, smem) / (float)(nvec * 8);
#pragma unroll
        for (int j = 0; j < VPT; ++j) {     // second pass over the packed registers (cheaper than keeping xhat and g*w unpacked)
            const int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
                float xh[8], g[8], wv[8], o[8];
                unpack8(cx[j], xh);
                unpack8(cg[j], g);
                unpack8(__ldg(w + v), wv);
#pragma unroll
                for (int i = 0; i < 8; ++i) o[i] = rstd * (g[i] * wv[i] - xh[i] * rstd * dot);
                st16(dx + r * nvec + v, pack8(o));
            }
        }
#pragma unroll
        for (int j = 0; j < VPT; ++j) { cx[j] = nx[j]; cg[j] = ng[j]; }
    }
#pragma unroll
    for (int j = 0; j < VPT; ++j) {
        const int v = threadIdx.x + j * kThreads;
        if (v < nvec) store_partial8(dw_partial, blockIdx.x, nvec, v, dw[j]);
    }
}

// ---------------------------------------------------------------------------------------------
// LayerNorm with bias (GPT / BERT families: torch.nn.LayerNorm in gpt_hf/GPTModel_tensor_parallel.py:34,56 and
// bert_hf/BertModel_tensor_parallel.py): fp32 math, y = (x - mean) * rstd * w + b, one rounding.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) layernorm_fwd_kernel(const uint4* __restrict__ x, const uint4* __restrict__ w,
                                                                 const uint4* __restrict__ b, uint4* __restrict__ y,
                                                                 float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                                 long long rows, int nvec, float eps) {
    __shared__ float smem[32];
    const float inv_n = 1.f / (float)(nvec * 8);
    for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
        const uint4* xr = x + r * nvec;
        uint4 xv[kMaxVpt];
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < kMaxVpt; ++j) {
            int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
                xv[j] = ld16_stream(xr + v);
                float f[8];
                unpack8(xv[j], f);
#pragma unroll
                for (int i = 0; i < 8; ++i) s += f[i];
            }
        }
        const float mean = block_reduce<false>(s, smem) * inv_n;
        float ss = 0.f;               // two-pass variance on the register-resident row (no cancellation)
#pragma unroll
        for (int j = 0; j < kMaxVpt; ++j) {
            int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
                float f[8];
                unpack8(xv[j], f);
#pragma unroll
                for (int i = 0; i < 8; ++i) ss += (f[i] - mean) * (f[i] - mean);
            }
        }
        const float rstd = rsqrtf(block_reduce<false>(ss, smem) * inv_n + eps);
        if (threadIdx.x == 0) { mean_out[r] = mean; rstd_out[r] = rstd; }
#pragma unroll
        for (int j = 0; j < kMaxVpt; ++j) {
            int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
                float f[8], g[8], c[8];
                unpack8(xv[j], f);
                unpack8(__ldg(w + v), g);
                unpack8(__ldg(b + v), c);
#pragma unroll
                for (int i = 0; i < 8; ++i) f[i] = (f[i] - mean) * rstd * g[i] + c[i];
                st16(y + r * nvec + v, pack8(f));
            }
        }
    }
}

// dx = rstd * (g - mean(g) - xhat * mean(g * xhat)) with g = dy * w;  dw_partial[cta] = sum dy * xhat, db_partial[cta] = sum dy
__global__ void __launch_bounds__(kThreads) layernorm_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x,
                                                                 const uint4* __restrict__ w, const float* __restrict__ mean_in,
                                                                 const float* __restrict__ rstd_in, uint4* __restrict__ dx,
                                                                 float* __restrict__ dw_partial, float* __restrict__ db_partial,
                                                                 long long rows, int nvec) {
    __shared__ float smem[32];
    // one 16-B vector per thread per pass keeps the accumulators in registers for rows up to kThreads * 8 * kMaxVpt columns
    float dw[kMaxVpt][8], db[kMaxVpt][8];
#pragma unroll
    for (int j = 0; j < kMaxVpt; ++j)
#pragma unroll
        for (int i = 0; i < 8; ++i) { dw[j][i] = 0.f; db[j][i] = 0.f; }
    const float inv_n = 1.f / (float)(nvec * 8);
    for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
        const float mean = mean_in[r], rstd = rstd_in[r];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < kMaxVpt; ++j) {
            int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
                float xh[8], g[8], wv[8];
                unpack8(ld16_stream(x + r * nvec + v), xh);
                unpack8(ld16_stream(dy + r * nvec + v), g);
                unpack8(__ldg(w + v), wv);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    xh[i] = (xh[i] - mean) * rstd;
                    dw[j][i] += g[i] * xh[i];
                    db[j][i] += g[i];
                    const float gw = g[i] * wv[i];
                    s1 += gw;
                    s2 += gw * xh[i];
                }
            }
        }
        s1 = block_reduce<false>(s1, smem) * inv_n;
        s2 = block_reduce<false>(s2, smem) * inv_n;
#pragma unroll
        for (int j = 0; j < kMaxVpt; ++j) {
            int v = threadIdx.x + j * kThreads;
            if (v < nvec) {       // re-read (L2-resident) instead of holding xhat and g*w for the whole row in registers
                float xh[8], g[8], wv[8], o[8];
                unpack8(ld16_stream(x + r * nvec + v), xh);
                unpack8(ld16_stream(dy + r * nvec + v), g);
                unpack8(__ldg(w + v), wv);
#pragma unroll
                for (int i = 0; i < 8; ++i) o[i] = rstd * (g[i] * wv[i] - s1 - (xh[i] - mean) * rstd * s2);
                st16(dx + r * nvec + v, pack8(o));
            }
        }
    }
#pragma unroll
    for (int j = 0; j < kMaxVpt; ++j) {
        int v = threadIdx.x + j * kThreads;
        if (v < nvec) {
            store_partial8(dw_partial, blockIdx.x, nvec, v, dw[j]);
            store_partial8(db_partial, blockIdx.x, nvec, v, db[j]);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// bias + activation:  y = act(x + b);  backward: dx = dy * act'(x + b)   (dbias = column sums of dx, the caller's)
// ---------------------------------------------------------------------------------------------
// GeLU, tanh form (Megatron's bias_gelu_impl: transformer.py:150-160 with bias_gelu_fusion; HF "gelu_new")
struct GeluTanh {
    __device__ static __forceinline__ float value(float v) { return v * 0.5f * (1.f + tanhf(0.79788456f * v * (1.f + 0.044715f * v * v))); }
    __device__ static __forceinline__ float grad(float v) {
        const float t = tanhf(0.79788456f * v * (1.f + 0.044715f * v * v));
        return 0.5f * v * ((1.f - t * t) * (0.79788456f + 0.1070322243f * v * v)) + 0.5f * (1.f + t);
    }
};
// GeLU, exact erf form (HF BERT "gelu")
struct GeluErf {
    __device__ static __forceinline__ float value(float v) { return v * 0.5f * (1.f + erff(v * 0.70710678f)); }
    __device__ static __forceinline__ float grad(float v) {
        return 0.5f * (1.f + erff(v * 0.70710678f)) + v * 0.3989422804f * __expf(-0.5f * v * v);
    }
};
// tanh (the ViT pooler: vit_hf pooler = dense + tanh)
struct Tanh {
    __device__ static __forceinline__ float value(float v) { return tanhf(v); }
    __device__ static __forceinline__ float grad(float v) {
        const float t = tanhf(v);
        return 1.f - t * t;
    }
};

template <class Act, bool kBackward>
__global__ void __launch_bounds__(kThreads) bias_act_kernel(const uint4* __restrict__ x, const uint4* __restrict__ bias,
                                                            const uint4* __restrict__ dy, uint4* __restrict__ out,
                                                            long long rows, int cvec) {
    const size_t total = (size_t)rows * cvec, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const size_t c = i % cvec;
        float f[8], b[8];
        unpack8(ld16_stream(x + i), f);
        if (bias != nullptr) {
            unpack8(__ldg(bias + c), b);
#pragma unroll
            for (int k = 0; k < 8; ++k) f[k] += b[k];
        }
        if (kBackward) {
            float d[8];
            unpack8(ld16_stream(dy + i), d);
#pragma unroll
            for (int k = 0; k < 8; ++k) f[k] = d[k] * Act::grad(f[k]);
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) f[k] = Act::value(f[k]);
        }
        st16(out + i, pack8(f));
    }
}

// ---------------------------------------------------------------------------------------------
// bias + dropout + residual add of the GPT / BERT blocks (the reference's F.dropout sites, GPTModel_tensor_parallel.py:31-59,
// BertModel_tensor_parallel.py:29-55):  y = residual + keep * scale * (x + bias),  dx = keep * scale * dy.
// Element (row r, column j) of a local [s_loc, b_loc, h] SBH tensor is token t = seq_base + r / b_loc of sample
// sample_base + r % b_loc; it is kept iff  Philox4x32-10(ctr = (j / 4, t, sample, iteration), key = (seed, site)).word[j % 4]
// >= threshold.  The mask depends on global coordinates only -- not on the launch geometry, the rank or the parallel layout --
// and backward regenerates it (nothing stored).
// ---------------------------------------------------------------------------------------------
struct DropoutCoords {
    long long b_loc, seq_base;
    union {
        long long sample_base;          // row r is sample sample_base + r % b_loc
        const uint32_t* sample_ids;     // IdMask: row r is sample sample_ids[r % b_loc]
    };
    uint32_t threshold, seed, iteration, site;
    float scale;
};

// keep bits of the 8 columns starting at column 8 * c of row r
__device__ __forceinline__ unsigned dropout_keep8(const DropoutCoords& d, long long r, int c) {
    const long long tok = r / d.b_loc;
    const uint32_t t = (uint32_t)(d.seq_base + tok), smp = (uint32_t)(d.sample_base + (r - tok * d.b_loc));
    const uint2 key = make_uint2(d.seed, d.site);
    const uint4 a = philox4x32_10(make_uint4(2u * c, t, smp, d.iteration), key);
    const uint4 b = philox4x32_10(make_uint4(2u * c + 1u, t, smp, d.iteration), key);
    const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    unsigned bits = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) bits |= (w[i] >= d.threshold ? 1u : 0u) << i;
    return bits;
}

// the same bits with row r's sample read from the map: sample_ids[r % b_loc].  (A shared helper taking (t, sample) would be one
// definition, but it changes the register allocation of every kernel that inlines dropout_keep8; the Philox counter, key and
// threshold here are dropout_keep8's, term for term.)
__device__ __forceinline__ unsigned dropout_keep8_ids(const DropoutCoords& d, long long r, int c) {
    const long long tok = r / d.b_loc;
    const uint32_t t = (uint32_t)(d.seq_base + tok), smp = __ldg(d.sample_ids + (r - tok * d.b_loc));
    const uint2 key = make_uint2(d.seed, d.site);
    const uint4 a = philox4x32_10(make_uint4(2u * c, t, smp, d.iteration), key);
    const uint4 b = philox4x32_10(make_uint4(2u * c + 1u, t, smp, d.iteration), key);
    const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    unsigned bits = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) bits |= (w[i] >= d.threshold ? 1u : 0u) << i;
    return bits;
}

// Per-sample drop path of Swin's attention branch (stochastic depth) uses the same kernels with a per-sample mask: row r of a
// [rows, h] SBH block is sample sample_base + r % b_loc, and the sample is kept iff word 0 of Philox4x32-10(ctr = (0, 0xffffffff,
// sample, iteration), key = (seed, site)) >= threshold (token 0xffffffff: a counter no dropout element uses).
__device__ __forceinline__ bool drop_path_keep(const DropoutCoords& d, long long r) {
    const uint32_t smp = (uint32_t)(d.sample_base + r % d.b_loc);
    return philox4x32_10(make_uint4(0u, 0xffffffffu, smp, d.iteration), make_uint2(d.seed, d.site)).x >= d.threshold;
}

// The mask policies: keep8 = the keep bits of the 8 columns starting at column 8 * c of row r.  The kernels below draw a sample
// mask (kPerSample) before they read the row, so that a dropped sample's row is not read and a kept one keeps all 8 columns; they
// draw an element mask after the row's loads are issued, so that the loads are in flight while Philox runs.
struct ElementMask {
    static constexpr bool kPerSample = false;
    __device__ static __forceinline__ unsigned keep8(const DropoutCoords& d, long long r, int c) { return dropout_keep8(d, r, c); }
};
struct SampleMask {
    static constexpr bool kPerSample = true;
    __device__ static __forceinline__ unsigned keep8(const DropoutCoords& d, long long r, int) { return drop_path_keep(d, r) ? 0xffu : 0u; }
};
// the element mask at an explicit sample map: row r is sample sample_ids[r % b_loc] (the samples a layer holds after a relocation
// re-split the batch are not one run of consecutive indices); counter, key, threshold and scale as ElementMask
struct IdMask {
    static constexpr bool kPerSample = false;
    __device__ static __forceinline__ unsigned keep8(const DropoutCoords& d, long long r, int c) { return dropout_keep8_ids(d, r, c); }
};

// grid = (column blocks, row groups), a thread owns one 8-column vector of every row of its group.  fp32 math in the order
// (x + bias) * scale, then masked, then + residual, each step rounded once (__fadd_rn / __fmul_rn: no FMA contraction).
template <class Mask, bool kBiasF32>
__global__ void __launch_bounds__(kThreads) bias_dropout_add_kernel(const uint4* __restrict__ x, const void* __restrict__ bias,
                                                                    const uint4* __restrict__ residual, uint4* __restrict__ y,
                                                                    long long rows, int nvec, DropoutCoords d) {
    const int c = blockIdx.x * kThreads + threadIdx.x;
    if (c >= nvec) return;
    float bv[8];
    load_bias8<kBiasF32>(bias, c, bv);
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {
        const size_t i = (size_t)r * nvec + c;
        float f[8], o[8];
        unpack8(residual != nullptr ? ld16_stream(residual + i) : make_uint4(0u, 0u, 0u, 0u), o);
        if (!Mask::kPerSample || Mask::keep8(d, r, c)) {
            unpack8(ld16_stream(x + i), f);
#pragma unroll
            for (int k = 0; k < 8; ++k) f[k] = __fadd_rn(f[k], bv[k]);
            apply_keep8(f, Mask::kPerSample ? 0xffu : Mask::keep8(d, r, c), d.scale);
#pragma unroll
            for (int k = 0; k < 8; ++k) o[k] = __fadd_rn(o[k], f[k]);
        } else {    // a dropped sample adds 0, as a dropped element does (so a -0 residual becomes +0)
#pragma unroll
            for (int k = 0; k < 8; ++k) o[k] = __fadd_rn(o[k], 0.f);
        }
        st16(y + i, pack8(o));
    }
}

// dx = keep * scale * dy (bf16);  dbias_partial[blockIdx.y] = the fp32 column sums of keep * scale * dy over the CTA's rows
template <class Mask>
__global__ void __launch_bounds__(kThreads) dropout_bwd_kernel(const uint4* __restrict__ dy, uint4* __restrict__ dx,
                                                               float* __restrict__ dbias_partial, long long rows, int nvec,
                                                               DropoutCoords d) {
    const int c = blockIdx.x * kThreads + threadIdx.x;
    if (c >= nvec) return;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (long long r = blockIdx.y; r < rows; r += gridDim.y) {
        const size_t i = (size_t)r * nvec + c;
        float g[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (!Mask::kPerSample || Mask::keep8(d, r, c)) {
            unpack8(ld16_stream(dy + i), g);
            apply_keep8(g, Mask::kPerSample ? 0xffu : Mask::keep8(d, r, c), d.scale);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = __fadd_rn(acc[k], g[k]);
        st16(dx + i, pack8(g));
    }
    if (dbias_partial != nullptr) store_partial8(dbias_partial, blockIdx.y, nvec, c, acc);
}

// ---------------------------------------------------------------------------------------------
// swiglu: gate_up = [rows, 2*ffn] (gate = first half, up = second; transformer.py:122-124)
// ---------------------------------------------------------------------------------------------
// grid = (column blocks of a row, row groups): no index division; two rows per iteration = four 16-B loads in flight per thread
__global__ void __launch_bounds__(kThreads) swiglu_fwd_kernel(const uint4* __restrict__ gu, uint4* __restrict__ y,
                                                              long long rows, int fvec) {
    const int c = blockIdx.x * kThreads + threadIdx.x;
    if (c >= fvec) return;
    const long long step = gridDim.y;
    for (long long r = blockIdx.y; r < rows; r += 2 * step) {
        const long long r2 = r + step;
        const bool two = r2 < rows;
        const uint4 g0 = ld16_stream(gu + r * 2 * fvec + c), u0 = ld16_stream(gu + r * 2 * fvec + fvec + c);
        uint4 g1 = g0, u1 = u0;
        if (two) { g1 = ld16_stream(gu + r2 * 2 * fvec + c); u1 = ld16_stream(gu + r2 * 2 * fvec + fvec + c); }
        float g[8], u[8];
        unpack8(g0, g); unpack8(u0, u);
#pragma unroll
        for (int k = 0; k < 8; ++k) g[k] = g[k] / (1.f + __expf(-g[k])) * u[k];
        st16(y + r * fvec + c, pack8(g));
        if (two) {
            unpack8(g1, g); unpack8(u1, u);
#pragma unroll
            for (int k = 0; k < 8; ++k) g[k] = g[k] / (1.f + __expf(-g[k])) * u[k];
            st16(y + r2 * fvec + c, pack8(g));
        }
    }
}

__global__ void __launch_bounds__(kThreads) swiglu_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ gu,
                                                              uint4* __restrict__ dgu, long long rows, int fvec) {
    const int c = blockIdx.x * kThreads + threadIdx.x;
    if (c >= fvec) return;
    const long long step = gridDim.y;
    for (long long r = blockIdx.y; r < rows; r += 2 * step) {
        const long long r2 = r + step;
        const bool two = r2 < rows;
        const uint4 g0 = ld16_stream(gu + r * 2 * fvec + c), u0 = ld16_stream(gu + r * 2 * fvec + fvec + c), d0 = ld16_stream(dy + r * fvec + c);
        uint4 g1 = g0, u1 = u0, d1 = d0;
        if (two) {
            g1 = ld16_stream(gu + r2 * 2 * fvec + c); u1 = ld16_stream(gu + r2 * 2 * fvec + fvec + c); d1 = ld16_stream(dy + r2 * fvec + c);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (h == 1 && !two) break;
            const long long rr = h ? r2 : r;
            float g[8], u[8], d[8], dg[8], du[8];
            unpack8(h ? g1 : g0, g); unpack8(h ? u1 : u0, u); unpack8(h ? d1 : d0, d);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float sg = 1.f / (1.f + __expf(-g[k]));
                du[k] = d[k] * g[k] * sg;
                dg[k] = d[k] * u[k] * sg * (1.f + g[k] * (1.f - sg));
            }
            st16(dgu + rr * 2 * fvec + c, pack8(dg));
            st16(dgu + rr * 2 * fvec + fvec + c, pack8(du));
        }
    }
}

// ---------------------------------------------------------------------------------------------
// fused QKV split + RoPE + [s,b,..] -> [b,s,heads,hn] relayout (and its exact transpose for backward).
// mixed: [s, b, ng, (r+2)*hn]  (per-group interleaved fused-QKV layout, transformer.py:733-756)
// q: [b, s, ng*r, hn]   k, v: [b, s, ng, hn]   cos/sin: [s, hn/2] fp32 (already offset for this rank)
// forward: q,k rotated by (+theta); backward: reads dq,dk,dv and writes dmixed rotated by (-theta).
// ---------------------------------------------------------------------------------------------
// One CTA walks tokens (s, b); a thread owns the same (group, head, half-head vector) of every token it visits, so the index
// decomposition is done once, outside the token loop, and all loads of a token are issued before the first use.
constexpr int kRopePairs = 2;   // (lo, hi) vector pairs per thread and token: covers ng * (r + 2) * hn / 16 <= 512 pairs (8192 columns)
__global__ void __launch_bounds__(kThreads) qkv_rope_kernel(uint4* __restrict__ mixed, uint4* __restrict__ q,
                                                            uint4* __restrict__ k, uint4* __restrict__ v,
                                                            const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                                            long long s, long long b, int ng, int r, int hn, int backward) {
    const int half_vec = hn / 16;              // 16-B vectors in half a head
    const int heads = r + 2;
    const int pairs = ng * heads * half_vec;   // per token
    int pc[kRopePairs], pj[kRopePairs];
    size_t pm[kRopePairs], po[kRopePairs];     // offsets inside a token of the mixed row / of the destination row
    for (int e = 0; e < kRopePairs; ++e) {
        const int p = threadIdx.x + e * kThreads;
        const int c = p % half_vec, j = (p / half_vec) % heads, g = p / (half_vec * heads);
        pc[e] = c; pj[e] = p < pairs ? j : -1;
        pm[e] = ((size_t)g * heads + j) * (2 * half_vec) + c;
        po[e] = (j < r) ? ((size_t)g * r + j) * (2 * half_vec) + c : (size_t)g * (2 * half_vec) + c;
    }
    const size_t mixed_tok = (size_t)pairs * 2, q_tok = (size_t)ng * r * 2 * half_vec, kv_tok = (size_t)ng * 2 * half_vec;
    const long long tokens = s * b;
    for (int base = 0; base < pairs; base += kRopePairs * kThreads) {   // rows wider than kRopePairs * kThreads pairs: extra passes
        for (long long t = blockIdx.x; t < tokens; t += gridDim.x) {
            const long long si = t / b, bi = t - si * b;
            const size_t tok_out = (size_t)bi * s + si;                // q/k/v are [b, s, ...]
            uint4 lo4[kRopePairs], hi4[kRopePairs];
            uint4* dst[kRopePairs];
#pragma unroll
            for (int e = 0; e < kRopePairs; ++e) {
                if (pj[e] < 0) continue;
                uint4* m = mixed + (size_t)t * mixed_tok + pm[e];
                uint4* o = (pj[e] < r) ? q + tok_out * q_tok + po[e] : ((pj[e] == r) ? k : v) + tok_out * kv_tok + po[e];
                uint4* src = backward ? o : m;
                dst[e] = backward ? m : o;
                lo4[e] = ld16_stream(src);
                hi4[e] = ld16_stream(src + half_vec);
            }
#pragma unroll
            for (int e = 0; e < kRopePairs; ++e) {
                if (pj[e] < 0) continue;
                float lo[8], hi[8];
                unpack8(lo4[e], lo);
                unpack8(hi4[e], hi);
                if (pj[e] <= r) {  // q and k heads are rotated, v is copied
                    const float4* cp = reinterpret_cast<const float4*>(cos_t + si * (hn / 2) + pc[e] * 8);
                    const float4* sp = reinterpret_cast<const float4*>(sin_t + si * (hn / 2) + pc[e] * 8);
                    float4 c0 = __ldg(cp), c1 = __ldg(cp + 1), s0 = __ldg(sp), s1 = __ldg(sp + 1);
                    const float cs[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
                    const float sn[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const float sg = backward ? -sn[i] : sn[i];
                        const float a = lo[i], bb = hi[i];
                        lo[i] = a * cs[i] - bb * sg;   // t*cos + rotate_half(t)*sin, rotate_half = (-x2, x1)
                        hi[i] = bb * cs[i] + a * sg;
                    }
                }
                st16(dst[e], pack8(lo));
                st16(dst[e] + half_vec, pack8(hi));
            }
        }
        if (base + kRopePairs * kThreads < pairs) {   // next pass: shift this thread's pairs
            for (int e = 0; e < kRopePairs; ++e) {
                const int p = threadIdx.x + e * kThreads + base + kRopePairs * kThreads;
                const int c = p % half_vec, j = (p / half_vec) % heads, g = p / (half_vec * heads);
                pc[e] = c; pj[e] = p < pairs ? j : -1;
                pm[e] = ((size_t)g * heads + j) * (2 * half_vec) + c;
                po[e] = (j < r) ? ((size_t)g * r + j) * (2 * half_vec) + c : (size_t)g * (2 * half_vec) + c;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// vocab-parallel cross-entropy (cross_entropy.py:14-152): three row kernels around two tiny all-reduces
// ---------------------------------------------------------------------------------------------
constexpr int kCeThreads = 512;

template <bool kBf16>
__device__ __forceinline__ int ce_load(const void* row, size_t v, float* f) {
    if (kBf16) { unpack8(ld16_stream(reinterpret_cast<const uint4*>(row) + v), f); return 8; }
    uint4 a = ld16_stream(reinterpret_cast<const uint4*>(row) + v);
    f[0] = __uint_as_float(a.x); f[1] = __uint_as_float(a.y); f[2] = __uint_as_float(a.z); f[3] = __uint_as_float(a.w);
    return 4;
}

template <bool kBf16>
__global__ void __launch_bounds__(kCeThreads) ce_rowmax_kernel(const void* __restrict__ logits, float* __restrict__ rowmax,
                                                               long long rows, long long vocab) {
    __shared__ float smem[32];
    constexpr int E = kBf16 ? 8 : 4;
    const size_t nvec = vocab / E;
    for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
        const char* row = reinterpret_cast<const char*>(logits) + (size_t)r * vocab * (kBf16 ? 2 : 4);
        float m = -INFINITY;
        for (size_t v = threadIdx.x; v < nvec; v += blockDim.x) {
            float f[8];
            ce_load<kBf16>(row, v, f);
#pragma unroll
            for (int i = 0; i < E; ++i) m = fmaxf(m, f[i]);
        }
        m = block_reduce<true>(m, smem);
        if (threadIdx.x == 0) rowmax[r] = m;
    }
}

// out2[r] = (sum_j exp(x_j - max_r), x_target - max_r if the target falls in [vocab_start, vocab_start+vocab) else 0)
template <bool kBf16>
__global__ void __launch_bounds__(kCeThreads) ce_sumexp_kernel(const void* __restrict__ logits, const long long* __restrict__ target,
                                                               const float* __restrict__ rowmax, float* __restrict__ out2,
                                                               long long rows, long long vocab, long long vocab_start) {
    __shared__ float smem[32];
    constexpr int E = kBf16 ? 8 : 4;
    const size_t nvec = vocab / E;
    for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
        const char* row = reinterpret_cast<const char*>(logits) + (size_t)r * vocab * (kBf16 ? 2 : 4);
        const float m = rowmax[r];
        float sum = 0.f;
        for (size_t v = threadIdx.x; v < nvec; v += blockDim.x) {
            float f[8];
            ce_load<kBf16>(row, v, f);
#pragma unroll
            for (int i = 0; i < E; ++i) sum += __expf(f[i] - m);
        }
        sum = block_reduce<false>(sum, smem);
        if (threadIdx.x == 0) {
            const long long t = target[r] - vocab_start;
            float pred = 0.f;
            if (t >= 0 && t < vocab)
                pred = (kBf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(row)[t]) : reinterpret_cast<const float*>(row)[t]) - m;
            out2[2 * r] = sum;
            out2[2 * r + 1] = pred;
        }
    }
}

// in place: logits <- (softmax - onehot(target)) * grad_loss[r]
template <bool kBf16>
__global__ void __launch_bounds__(kCeThreads) ce_bwd_kernel(void* __restrict__ logits, const long long* __restrict__ target,
                                                            const float* __restrict__ rowmax, const float* __restrict__ sum2,
                                                            const float* __restrict__ grad_loss, long long rows, long long vocab,
                                                            long long vocab_start) {
    constexpr int E = kBf16 ? 8 : 4;
    const size_t nvec = vocab / E;
    for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
        char* row = reinterpret_cast<char*>(logits) + (size_t)r * vocab * (kBf16 ? 2 : 4);
        const float m = rowmax[r], inv = 1.f / sum2[2 * r], g = grad_loss[r];
        const long long t = target[r] - vocab_start;
        for (size_t v = threadIdx.x; v < nvec; v += blockDim.x) {
            float f[8];
            ce_load<kBf16>(row, v, f);
#pragma unroll
            for (int i = 0; i < E; ++i) {
                float p = __expf(f[i] - m) * inv;
                if ((long long)(v * E + i) == t) p -= 1.f;
                f[i] = p * g;
            }
            if (kBf16) st16(reinterpret_cast<uint4*>(row) + v, pack8(f));
            else reinterpret_cast<float4*>(row)[v] = make_float4(f[0], f[1], f[2], f[3]);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// ring context parallelism: log-sum-exp merge of one block's attention result (transformer.py:2209-2250)
// ---------------------------------------------------------------------------------------------
// One thread per 8 head-dim elements of one (sample, query row, head); the d / 8 threads of a row sit in one warp.  Every thread
// of a row reads the two LSEs, the warp synchronises, then the row's first thread writes the merged LSE.
__global__ void __launch_bounds__(kThreads) lse_merge_kernel(const uint4* __restrict__ blk_out, const float* __restrict__ blk_lse,
                                                             float* __restrict__ acc_out, float* __restrict__ acc_lse,
                                                             uint4* __restrict__ final_out, long long s, long long sq_blk, long long n,
                                                             int vpr, long long row_off, long long rows_total, int init) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool ok = idx < rows_total * vpr;
    const long long row = ok ? idx / vpr : 0, part = idx - row * vpr;      // row = (bi * s + q) * n + h
    const long long h = row % n, q = (row / n) % s, bi = row / (n * s);
    const bool in_blk = ok && q >= row_off && q < row_off + sq_blk;
    const long long qb = q - row_off;
    float la = -INFINITY, lb = -INFINITY;
    if (in_blk) {
        lb = blk_lse[(bi * n + h) * sq_blk + qb];
        if (!init) la = acc_lse[(bi * n + h) * s + q];
    }
    __syncwarp();
    if (!ok) return;
    float4* ao = reinterpret_cast<float4*>(acc_out) + idx * 2;
    float f[8];
    if (in_blk) {
        float b8[8];
        unpack8(ld16_stream(blk_out + ((bi * sq_blk + qb) * n + h) * vpr + part), b8);
        float wa = 0.f, wb = 1.f, lse = lb;
        if (!init) {
            const float m = fmaxf(la, lb);
            if (m == -INFINITY) {
                wb = 0.f;
            } else {
                lse = m + logf(expf(la - m) + expf(lb - m));
                wa = expf(la - lse);
                wb = expf(lb - lse);
            }
        }
        if (init) {
#pragma unroll
            for (int i = 0; i < 8; ++i) f[i] = b8[i];
        } else {
            const float4 x = ao[0], y = ao[1];
            f[0] = x.x * wa + b8[0] * wb; f[1] = x.y * wa + b8[1] * wb; f[2] = x.z * wa + b8[2] * wb; f[3] = x.w * wa + b8[3] * wb;
            f[4] = y.x * wa + b8[4] * wb; f[5] = y.y * wa + b8[5] * wb; f[6] = y.z * wa + b8[6] * wb; f[7] = y.w * wa + b8[7] * wb;
        }
        ao[0] = make_float4(f[0], f[1], f[2], f[3]);
        ao[1] = make_float4(f[4], f[5], f[6], f[7]);
        if (part == 0) acc_lse[(bi * n + h) * s + q] = lse;
    } else if (final_out) {
        const float4 x = ao[0], y = ao[1];
        f[0] = x.x; f[1] = x.y; f[2] = x.z; f[3] = x.w; f[4] = y.x; f[5] = y.y; f[6] = y.z; f[7] = y.w;
    }
    if (final_out) st16(final_out + idx, pack8(f));
}

// ---------------------------------------------------------------------------------------------
// ViT front end (vit_hf/ViTModel_sequential.py ViTEmbeddings_): patchify relayout, then the SBH activation assembled from the
// patch GEMM's output, the patch bias, the CLS token and the learned position table, with the embedding dropout fused in.
// ---------------------------------------------------------------------------------------------
// pixels [B, C, H, W] -> patch rows [rows_pad, p*p*C] in einops' "b c (h p1) (w p2) -> b (h w) (p1 p2 c)" order, bf16 (one RNE
// rounding for fp32 pixels); rows B*P .. rows_pad - 1 are zeros.  A thread writes one 16-B vector of 8 consecutive columns.
template <bool kF32>
__global__ void __launch_bounds__(kThreads) vit_patchify_kernel(const void* __restrict__ pix, uint4* __restrict__ out,
                                                                long long rows_real, long long rows_pad, int kvec, int C, int H,
                                                                int W, int p, int P) {
    const size_t total = (size_t)rows_pad * kvec, stride = (size_t)gridDim.x * blockDim.x;
    const int gw = W / p;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const long long r = (long long)(i / kvec);
        const int cv = (int)(i - (size_t)r * kvec);
        float f[8];
        if (r < rows_real) {
            const long long b = r / P;
            const int patch = (int)(r - b * P), hi = patch / gw, wi = patch - (patch / gw) * gw;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int col = cv * 8 + k, c = col % C, q = col / C, p2 = q % p, p1 = q / p;
                const size_t idx = ((size_t)(b * C + c) * H + (size_t)(hi * p + p1)) * W + (size_t)(wi * p + p2);
                f[k] = kF32 ? __ldg(reinterpret_cast<const float*>(pix) + idx)
                            : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(pix)[idx]);
            }
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) f[k] = 0.f;
        }
        st16(out + i, pack8(f));
    }
}

// y [s_run, b, h]: row 0 = cls + pos[0]; row s in 1..P = patch[bi * P + s - 1] + (bias + pos[s]); rows > P zero.  fp32 math, one
// rounding to bf16; with kDrop the dropout of bg_dropout_add_fwd at (token s, sample sample_base + bi) is applied before it.
// grid = (column blocks, row groups over s); a thread owns one 8-column vector of every sample of its rows.
template <bool kDrop>
__global__ void __launch_bounds__(kThreads) vit_embed_fwd_kernel(const uint4* __restrict__ patch, const uint4* __restrict__ bias,
                                                                 const uint4* __restrict__ cls, const uint4* __restrict__ pos,
                                                                 uint4* __restrict__ y, long long b, long long P, long long s_run,
                                                                 int nvec, DropoutCoords d) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nvec) return;
    float bv[8], cv[8];
    unpack8(__ldg(bias + c), bv);
    unpack8(__ldg(cls + c), cv);
    for (long long s = blockIdx.y; s < s_run; s += gridDim.y) {
        if (s > P) {
            for (long long bi = 0; bi < b; ++bi) st16(y + (size_t)(s * b + bi) * nvec + c, make_uint4(0u, 0u, 0u, 0u));
            continue;
        }
        float base[8];
        unpack8(__ldg(pos + (size_t)s * nvec + c), base);
#pragma unroll
        for (int k = 0; k < 8; ++k) base[k] = __fadd_rn(base[k], s == 0 ? cv[k] : bv[k]);
#pragma unroll 4
        for (long long bi = 0; bi < b; ++bi) {
            const long long r = s * b + bi;
            float f[8];
            if (s == 0) {
#pragma unroll
                for (int k = 0; k < 8; ++k) f[k] = base[k];
            } else {
                unpack8(ld16_stream(patch + (size_t)(bi * P + s - 1) * nvec + c), f);
#pragma unroll
                for (int k = 0; k < 8; ++k) f[k] = __fadd_rn(f[k], base[k]);
            }
            if (kDrop) apply_keep8(f, dropout_keep8(d, r, c), d.scale);
            st16(y + (size_t)r * nvec + c, pack8(f));
        }
    }
}

// backward of the above: g = (keep * scale *) dy.  dpatch[bi * P + s - 1] = bf16(g[s, bi]) for s in 1..P, rows b*P .. rows_pad - 1
// zero; dpos[s] = fp32 sum over the samples in order of g[s, bi] for s < P + 1 (dpos[0] is also dcls); dbias_partial[blockIdx.y] =
// the CTA's fp32 sum of dpos rows 1..P in row order.  Rows > P of dy belong to padding tokens and are not read.
template <bool kDrop>
__global__ void __launch_bounds__(kThreads) vit_embed_bwd_kernel(const uint4* __restrict__ dy, uint4* __restrict__ dpatch,
                                                                 float* __restrict__ dpos, float* __restrict__ dbias_partial,
                                                                 long long b, long long P, long long rows_pad, int nvec,
                                                                 DropoutCoords d) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nvec) return;
    float accb[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) accb[k] = 0.f;
    for (long long s = blockIdx.y; s <= P; s += gridDim.y) {
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
#pragma unroll 4
        for (long long bi = 0; bi < b; ++bi) {
            const long long r = s * b + bi;
            float g[8];
            unpack8(ld16_stream(dy + (size_t)r * nvec + c), g);
            if (kDrop) apply_keep8(g, dropout_keep8(d, r, c), d.scale);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] = __fadd_rn(acc[k], g[k]);
            if (s > 0) st16(dpatch + (size_t)(bi * P + s - 1) * nvec + c, pack8(g));
        }
        store_partial8(dpos, s, nvec, c, acc);
        if (s > 0) {
#pragma unroll
            for (int k = 0; k < 8; ++k) accb[k] = __fadd_rn(accb[k], acc[k]);
        }
    }
    if (blockIdx.y == 0)
        for (long long r = b * P; r < rows_pad; ++r) st16(dpatch + (size_t)r * nvec + c, make_uint4(0u, 0u, 0u, 0u));
    store_partial8(dbias_partial, blockIdx.y, nvec, c, accb);
}

// ---------------------------------------------------------------------------------------------
// Swin (swin/SwinModel_tensor_parallel.py): the window relayouts around attention, patch merging + LayerNorm and the token
// mean-pool (its per-sample drop path is the dropout kernels' SampleMask).  Activations are SBH rows (row = token * mb + sample)
// of tokens_run tokens per sample, the real tokens first; a shifted window partition is one int32 token map per layer shape:
// map[w * L + i] = the token at position i of window w (L = window * window tokens), and inv[t] = w * L + i its inverse.  Window
// rows are [mb * nW, L, ...], window b * nW + w of sample b.
// ---------------------------------------------------------------------------------------------
// mixed [tokens_run * mb, heads * 3 * hn] (per head q | k | v, the fused QKV GEMM's layout) + bias -> q, k, v [mb * nW, L, heads, hn]
// (one rounding).  A thread writes one 16-B vector; consecutive threads read consecutive vectors of one mixed row.
__global__ void __launch_bounds__(kThreads) swin_window_qkv_fwd_kernel(const uint4* __restrict__ mixed, const uint4* __restrict__ bias,
                                                                       const int* __restrict__ map, uint4* __restrict__ q,
                                                                       uint4* __restrict__ k, uint4* __restrict__ v, long long mb,
                                                                       long long nW, int L, int heads, int hv) {
    const int ncol = heads * 3 * hv;
    const size_t total = (size_t)mb * nW * L * ncol, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const long long wrow = (long long)(i / ncol);
        const int col = (int)(i - (size_t)wrow * ncol);
        const long long wi = wrow / L, b = wi / nW;
        const int pos = (int)(wrow - wi * L), w = (int)(wi - b * nW);
        const long long src = (long long)__ldg(map + (size_t)w * L + pos) * mb + b;
        const int h = col / (3 * hv), part = (col / hv) % 3, c = col % hv;
        float f[8], bv[8];
        unpack8(ld16_stream(mixed + (size_t)src * ncol + col), f);
        unpack8(__ldg(bias + col), bv);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = __fadd_rn(f[e], bv[e]);
        uint4* dst = part == 0 ? q : (part == 1 ? k : v);
        st16(dst + ((size_t)wrow * heads + h) * hv + c, pack8(f));
    }
}

// its backward: dmixed rows gathered from dq, dk, dv through inv (padding-token rows zero); dbias_partial[blockIdx.y] = the CTA's
// fp32 column sums in row order.  grid = (column blocks, row groups); a thread owns one column vector of every row it visits.
__global__ void __launch_bounds__(kThreads) swin_window_qkv_bwd_kernel(const uint4* __restrict__ dq, const uint4* __restrict__ dk,
                                                                       const uint4* __restrict__ dv, uint4* __restrict__ dmixed,
                                                                       float* __restrict__ dbias_partial, const int* __restrict__ inv,
                                                                       long long mb, long long T, long long T_run, long long nW, int L,
                                                                       int heads, int hv) {
    const int ncol = heads * 3 * hv;
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= ncol) return;
    const int h = col / (3 * hv), part = (col / hv) % 3, c = col % hv;
    const uint4* src = part == 0 ? dq : (part == 1 ? dk : dv);
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    for (long long r = blockIdx.y; r < T_run * mb; r += gridDim.y) {
        const long long t = r / mb, b = r - t * mb;
        uint4 g = make_uint4(0u, 0u, 0u, 0u);
        if (t < T) {
            const int p = __ldg(inv + t), w = p / L, pos = p - w * L;
            const long long wrow = (b * nW + w) * L + pos;
            g = ld16_stream(src + ((size_t)wrow * heads + h) * hv + c);
            float f[8];
            unpack8(g, f);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = __fadd_rn(acc[e], f[e]);
        }
        st16(dmixed + (size_t)r * ncol + col, g);
    }
    store_partial8(dbias_partial, blockIdx.y, ncol, col, acc);
}

// window rows [mb * nW, L, cvec vectors] <-> SBH rows [T_run * mb, cvec vectors], a pure copy.  Forward (window rows -> SBH):
// SBH row t * mb + b reads window row (b * nW + w) * L + i with w * L + i = inv[t]; padding-token rows are zero.  Backward (SBH ->
// window rows): window row (b * nW + w) * L + i reads SBH row map[w * L + i] * mb + b.  A thread writes one 16-B vector.
template <bool kBackward>
__global__ void __launch_bounds__(kThreads) swin_window_merge_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst,
                                                                     const int* __restrict__ map, const int* __restrict__ inv,
                                                                     long long mb, long long T, long long T_run, long long nW, int L,
                                                                     int cvec) {
    const size_t rows = kBackward ? (size_t)mb * nW * L : (size_t)T_run * mb;
    const size_t total = rows * cvec, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const long long r = (long long)(i / cvec);
        const int c = (int)(i - (size_t)r * cvec);
        long long s = -1;
        if (kBackward) {
            const long long wi = r / L, b = wi / nW;
            const int pos = (int)(r - wi * L), w = (int)(wi - b * nW);
            s = (long long)__ldg(map + (size_t)w * L + pos) * mb + b;
        } else {
            const long long t = r / mb, b = r - t * mb;
            if (t < T) {
                const int p = __ldg(inv + t), w = p / L;
                s = (b * nW + w) * L + (p - w * L);
            }
        }
        st16(dst + i, s < 0 ? make_uint4(0u, 0u, 0u, 0u) : ld16_stream(src + (size_t)s * cvec + c));
    }
}

// Patch merging (r = 2) or the embedding's bias + norm (r = 1), then LayerNorm over the gathered row of r * r * C columns.  Output
// row t' * mb + b (t' = (i', j') on the (H / r) x (W / r) grid) is the concatenation over q = 0..r*r-1 of input token
// (r i' + (q & 1), r j' + (q >> 1)) of sample b -- HF's x0, x1, x2, x3 order -- plus add_bias when given, then
// (v - mean) * rstd * w + b exactly as layernorm_fwd_kernel computes it (the same per-thread vectors, so the same rounding).
// Input rows are SBH (token * mb + b) or, with in_bsh, (b * T_in + token) as the patch GEMM writes them.  Output rows of padding
// tokens (t' >= T_out) are zero, with mean = rstd = 0.
constexpr int kMergeVpt = 5;    // rows up to 256 * 8 * 5 = 10240 columns (Swin-H's widest merged row is 4 x 1280)
struct MergeGeom {
    long long mb, T_in, T_out, T_out_run;
    int Wi, Wo, r, cvec_in, in_bsh;
};
__device__ __forceinline__ long long merge_src_row(const MergeGeom& g, long long to, long long b, int q) {
    const long long io = to / g.Wo, jo = to - io * g.Wo;
    const long long ts = (g.r * io + (q & 1)) * g.Wi + g.r * jo + (q >> 1);
    return g.in_bsh ? b * g.T_in + ts : ts * g.mb + b;
}

template <bool kBias>
__global__ void __launch_bounds__(kThreads) swin_merge_ln_fwd_kernel(const uint4* __restrict__ x, const uint4* __restrict__ add_bias,
                                                                     const uint4* __restrict__ w, const uint4* __restrict__ bb,
                                                                     uint4* __restrict__ y, float* __restrict__ mean_out,
                                                                     float* __restrict__ rstd_out, MergeGeom g, float eps) {
    __shared__ float smem[32];
    const int nvec = g.r * g.r * g.cvec_in;
    const float inv_n = 1.f / (float)(nvec * 8);
    for (long long ro = blockIdx.x; ro < g.T_out_run * g.mb; ro += gridDim.x) {
        const long long to = ro / g.mb, b = ro - to * g.mb;
        if (to >= g.T_out) {
            for (int v = threadIdx.x; v < nvec; v += kThreads) st16(y + ro * nvec + v, make_uint4(0u, 0u, 0u, 0u));
            if (threadIdx.x == 0) { mean_out[ro] = 0.f; rstd_out[ro] = 0.f; }
            continue;
        }
        float xf[kMergeVpt][8];
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < kMergeVpt; ++j) {
            const int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
                const int q = v / g.cvec_in, c = v - q * g.cvec_in;
                unpack8(ld16_stream(x + (size_t)merge_src_row(g, to, b, q) * g.cvec_in + c), xf[j]);
                if (kBias) {
                    float bv[8];
                    unpack8(__ldg(add_bias + v), bv);
#pragma unroll
                    for (int i = 0; i < 8; ++i) xf[j][i] = __fadd_rn(xf[j][i], bv[i]);
                }
#pragma unroll
                for (int i = 0; i < 8; ++i) s += xf[j][i];
            }
        }
        const float mean = block_reduce<false>(s, smem) * inv_n;
        float ss = 0.f;
#pragma unroll
        for (int j = 0; j < kMergeVpt; ++j) {
            const int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
#pragma unroll
                for (int i = 0; i < 8; ++i) ss += (xf[j][i] - mean) * (xf[j][i] - mean);
            }
        }
        const float rstd = rsqrtf(block_reduce<false>(ss, smem) * inv_n + eps);
        if (threadIdx.x == 0) { mean_out[ro] = mean; rstd_out[ro] = rstd; }
#pragma unroll
        for (int j = 0; j < kMergeVpt; ++j) {
            const int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
                float f[8], gw[8], c[8];
                unpack8(__ldg(w + v), gw);
                unpack8(__ldg(bb + v), c);
#pragma unroll
                for (int i = 0; i < 8; ++i) f[i] = (xf[j][i] - mean) * rstd * gw[i] + c[i];
                st16(y + ro * nvec + v, pack8(f));
            }
        }
    }
}

// its backward, layernorm_bwd_kernel's math on the gathered row: dv = rstd * (g - mean(g) - vhat * mean(g * vhat)), g = dy * w,
// scattered back to the r * r source rows (each input token feeds exactly one output token, so no two CTAs write one row).  The
// output rows of padding tokens are not read; input rows mb * T_in .. rows_in - 1 get zeros.  Per-CTA fp32 partials: dw = sum
// dy * vhat, db = sum dy, and with kBias dbias = sum dv (the column sums of the input gradient, before its rounding).
template <int VPT, bool kBias>
__global__ void __launch_bounds__(kThreads) swin_merge_ln_bwd_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ x,
                                                                     const uint4* __restrict__ add_bias, const uint4* __restrict__ w,
                                                                     const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                                                                     uint4* __restrict__ dx, float* __restrict__ dw_partial,
                                                                     float* __restrict__ db_partial, float* __restrict__ dbias_partial,
                                                                     MergeGeom g, long long rows_in) {
    __shared__ float smem[32];
    const int nvec = g.r * g.r * g.cvec_in;
    float dw[VPT][8], db[VPT][8], dbi[kBias ? VPT : 1][8];
#pragma unroll
    for (int j = 0; j < VPT; ++j)
#pragma unroll
        for (int i = 0; i < 8; ++i) { dw[j][i] = 0.f; db[j][i] = 0.f; if (kBias) dbi[j][i] = 0.f; }
    const float inv_n = 1.f / (float)(nvec * 8);
    for (long long ro = blockIdx.x; ro < g.T_out * g.mb; ro += gridDim.x) {
        const long long to = ro / g.mb, b = ro - to * g.mb;
        const float mean = mean_in[ro], rstd = rstd_in[ro];
        float xh[VPT][8], gv[VPT][8];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < VPT; ++j) {
            const int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
                const int q = v / g.cvec_in, c = v - q * g.cvec_in;
                float wv[8];
                unpack8(ld16_stream(x + (size_t)merge_src_row(g, to, b, q) * g.cvec_in + c), xh[j]);
                unpack8(ld16_stream(dy + ro * nvec + v), gv[j]);
                unpack8(__ldg(w + v), wv);
                if (kBias) {
                    float bv[8];
                    unpack8(__ldg(add_bias + v), bv);
#pragma unroll
                    for (int i = 0; i < 8; ++i) xh[j][i] = __fadd_rn(xh[j][i], bv[i]);
                }
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    xh[j][i] = (xh[j][i] - mean) * rstd;
                    dw[j][i] += gv[j][i] * xh[j][i];
                    db[j][i] += gv[j][i];
                    gv[j][i] *= wv[i];
                    s1 += gv[j][i];
                    s2 += gv[j][i] * xh[j][i];
                }
            }
        }
        s1 = block_reduce<false>(s1, smem) * inv_n;
        s2 = block_reduce<false>(s2, smem) * inv_n;
#pragma unroll
        for (int j = 0; j < VPT; ++j) {
            const int v = threadIdx.x + j * kThreads;
            if (v < nvec) {
                const int q = v / g.cvec_in, c = v - q * g.cvec_in;
                float o[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    o[i] = rstd * (gv[j][i] - s1 - xh[j][i] * s2);
                    if (kBias) dbi[j][i] += o[i];
                }
                st16(dx + (size_t)merge_src_row(g, to, b, q) * g.cvec_in + c, pack8(o));
            }
        }
    }
    for (long long r = g.mb * g.T_in + blockIdx.x; r < rows_in; r += gridDim.x)
        for (int c = threadIdx.x; c < g.cvec_in; c += kThreads) st16(dx + (size_t)r * g.cvec_in + c, make_uint4(0u, 0u, 0u, 0u));
#pragma unroll
    for (int j = 0; j < VPT; ++j) {
        const int v = threadIdx.x + j * kThreads;
        if (v < nvec) {
            store_partial8(dw_partial, blockIdx.x, nvec, v, dw[j]);
            store_partial8(db_partial, blockIdx.x, nvec, v, db[j]);
            if (kBias) store_partial8(dbias_partial, blockIdx.x, nvec, v, dbi[j]);
        }
    }
}

// Swin's pooler: y[b] = (sum over the first T tokens of x[t, b], fp32 in token order) / T for b < mb, zero rows up to rows_out.
// Backward: dx[t, b] = dy[b] / T for t < T, zero for the padding tokens.  A thread owns one 16-B vector of output.
template <bool kBackward>
__global__ void __launch_bounds__(kThreads) swin_mean_pool_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, long long T,
                                                                  long long T_run, long long mb, long long rows_out, int cvec) {
    const size_t rows = kBackward ? (size_t)T_run * mb : (size_t)rows_out;
    const size_t total = rows * cvec, stride = (size_t)gridDim.x * blockDim.x;
    const float tf = (float)T;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const long long r = (long long)(i / cvec);
        const int c = (int)(i - (size_t)r * cvec);
        float f[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = 0.f;
        if (kBackward) {
            const long long t = r / mb;
            if (t < T) {
                unpack8(__ldg(in + (size_t)(r - t * mb) * cvec + c), f);
#pragma unroll
                for (int e = 0; e < 8; ++e) f[e] = __fdiv_rn(f[e], tf);
            }
        } else if (r < mb) {
            for (long long t = 0; t < T; ++t) {
                float a[8];
                unpack8(ld16_stream(in + ((size_t)t * mb + r) * cvec + c), a);
#pragma unroll
                for (int e = 0; e < 8; ++e) f[e] = __fadd_rn(f[e], a[e]);
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) f[e] = __fdiv_rn(f[e], tf);
        }
        st16(out + i, pack8(f));
    }
}

// ---------------------------------------------------------------------------------------------
// T5 cross-attention (t5/T5Model_tensor_parallel.py): the query and key_value projections are two GEMMs over different sequences,
// so the fused qkv_rope relayout does not apply.  q_mixed [s_q * b, np * hn] (row = token * b + sample) + q_bias and kv_mixed
// [s_k * b, np * 2 * hn] (per head k | v) + kv_bias -> q [b, s_q, np, hn] and k, v [b, s_k, np, hn], the bias added in fp32 and rounded
// once (a null bias adds nothing).  One launch for both inputs: a thread writes one 16-B vector; the first s_q * b * np * hv vectors
// are the query's, consecutive threads read consecutive vectors of one input row.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) cross_attn_qkv_fwd_kernel(const uint4* __restrict__ qm, const uint4* __restrict__ qb,
                                                                      const uint4* __restrict__ kvm, const uint4* __restrict__ kvb,
                                                                      uint4* __restrict__ q, uint4* __restrict__ k,
                                                                      uint4* __restrict__ v, long long s_q, long long s_k, long long batch,
                                                                      int heads, int hv) {
    const int qcol = heads * hv, kvcol = 2 * qcol;
    const size_t nq = (size_t)s_q * batch * qcol, total = nq + (size_t)s_k * batch * kvcol, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const bool is_q = i < nq;
        const size_t j = is_q ? i : i - nq;
        const int ncol = is_q ? qcol : kvcol;
        const long long r = (long long)(j / ncol);
        const int col = (int)(j - (size_t)r * ncol);
        const long long t = r / batch, bi = r - t * batch;
        const uint4* bias = is_q ? qb : kvb;
        float f[8];
        unpack8(ld16_stream((is_q ? qm : kvm) + j), f);
        if (bias != nullptr) {
            float bv[8];
            unpack8(__ldg(bias + col), bv);
#pragma unroll
            for (int e = 0; e < 8; ++e) f[e] = __fadd_rn(f[e], bv[e]);
        }
        if (is_q) {
            st16(q + ((size_t)bi * s_q + t) * qcol + col, pack8(f));
        } else {
            const int h = col / (2 * hv), part = (col / hv) & 1, e = col - (2 * h + part) * hv;
            st16((part ? v : k) + (((size_t)bi * s_k + t) * heads + h) * hv + e, pack8(f));
        }
    }
}

// its backward: dq_mixed [s_q * b, np * hn] and dkv_mixed [s_k * b, np * 2 * hn] gathered from dq, dk, dv; dbias_partial[blockIdx.y]
// [np * 3 * hn] = the CTA's fp32 column sums in row order, the query's np * hn columns first.  grid = (column blocks over both
// outputs' columns, row groups); a thread owns one column vector of every row it visits.
__global__ void __launch_bounds__(kThreads) cross_attn_qkv_bwd_kernel(const uint4* __restrict__ dq, const uint4* __restrict__ dk,
                                                                      const uint4* __restrict__ dv, uint4* __restrict__ dqm,
                                                                      uint4* __restrict__ dkvm, float* __restrict__ dbias_partial,
                                                                      long long s_q, long long s_k, long long batch, int heads, int hv) {
    const int qcol = heads * hv, ncol = 3 * qcol;
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= ncol) return;
    const bool is_q = col < qcol;
    const int c = is_q ? col : col - qcol;
    const long long s = is_q ? s_q : s_k;
    const uint4* src = dq;
    int off = c;
    if (!is_q) {
        const int h = c / (2 * hv), part = (c / hv) & 1;
        src = part ? dv : dk;
        off = h * hv + (c - (2 * h + part) * hv);
    }
    uint4* dst = is_q ? dqm : dkvm;
    const int width = is_q ? qcol : 2 * qcol;
    float acc[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    for (long long r = blockIdx.y; r < s * batch; r += gridDim.y) {
        const long long t = r / batch, bi = r - t * batch;
        const uint4 g = ld16_stream(src + ((size_t)bi * s + t) * qcol + off);
        float f[8];
        unpack8(g, f);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = __fadd_rn(acc[e], f[e]);
        st16(dst + (size_t)r * width + c, g);
    }
    store_partial8(dbias_partial, blockIdx.y, ncol, col, acc);
}

}  // namespace

#define BG_ALIGNED16(p) (((uintptr_t)(p) % 16) == 0)

extern "C" int bg_lse_merge(const void* blk_out, const float* blk_lse, float* acc_out, float* acc_lse, void* final_out, long long b,
                            long long s, long long sq_blk, long long n, long long d, long long row_off, int init, void* stream) {
    if (b < 1 || s < 1 || n < 1 || d < 8 || d % 8 || d > 256 || 32 % (d / 8) || sq_blk < 1 || row_off < 0 || row_off + sq_blk > s)
        return fail(BG_EINVAL, "bg_lse_merge: bad shape b %lld s %lld sq_blk %lld n %lld d %lld row_off %lld", b, s, sq_blk, n, d, row_off);
    if (init && (row_off != 0 || sq_blk != s)) return fail(BG_EINVAL, "bg_lse_merge: init needs a block of every row");
    if (!BG_ALIGNED16(blk_out) || !BG_ALIGNED16(acc_out) || !BG_ALIGNED16(final_out))
        return fail(BG_EINVAL, "bg_lse_merge: pointers must be 16-B aligned");
    const int vpr = (int)(d / 8);
    const long long rows = b * s * n, threads = rows * vpr;
    const int grid = (int)((threads + kThreads - 1) / kThreads);
    lse_merge_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>((const uint4*)blk_out, blk_lse, acc_out, acc_lse, (uint4*)final_out, s,
                                                                 sq_blk, n, vpr, row_off, rows, init);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_cast(const void* src, int src_dtype, void* dst, int dst_dtype, size_t elems, float scale, int accumulate,
                       void* stream) {
    if (elems % 8) return fail(BG_EINVAL, "bg_cast: elems %zu must be a multiple of 8", elems);
    if (!BG_ALIGNED16(src) || !BG_ALIGNED16(dst)) return fail(BG_EINVAL, "bg_cast: pointers must be 16-B aligned");
    if (elems == 0) return BG_OK;
    const size_t nvec = elems / 8;
    int grid = local_grid(nvec, kThreads);
    cudaStream_t st = (cudaStream_t)stream;
    const bool sb = src_dtype == BG_BF16, db = dst_dtype == BG_BF16;
    if (sb && db) cast_kernel<true, true><<<grid, kThreads, 0, st>>>(src, dst, nvec, scale, accumulate);
    else if (sb && !db) cast_kernel<true, false><<<grid, kThreads, 0, st>>>(src, dst, nvec, scale, accumulate);
    else if (!sb && db) cast_kernel<false, true><<<grid, kThreads, 0, st>>>(src, dst, nvec, scale, accumulate);
    else cast_kernel<false, false><<<grid, kThreads, 0, st>>>(src, dst, nvec, scale, accumulate);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

static int norm_args(long long rows, long long cols, const char* who) {
    if (rows < 0) return fail(BG_EINVAL, "%s: rows %lld must be >= 0", who, rows);
    if (cols <= 0 || cols % 8) return fail(BG_EINVAL, "%s: cols %lld must be a positive multiple of 8", who, cols);
    if (cols / 8 > (long long)kMaxVpt * kThreads) return fail(BG_EUNSUPPORTED, "%s: cols %lld > %d", who, cols, kMaxVpt * kThreads * 8);
    return BG_OK;
}

extern "C" int bg_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, long long rows, long long cols, float eps,
                              void* stream) {
    int rc = norm_args(rows, cols, "bg_rmsnorm_fwd");
    if (rc) return rc;
    if (!BG_ALIGNED16(x) || !BG_ALIGNED16(w) || !BG_ALIGNED16(y)) return fail(BG_EINVAL, "bg_rmsnorm_fwd: 16-B alignment");
    if (rows == 0) return BG_OK;
    int grid = (int)(rows < g_tun.local_ctas ? rows : g_tun.local_ctas);
    const int nvec = (int)(cols / 8), vpt = (nvec + kThreads - 1) / kThreads;
#define BG_RMS_FWD(V) rmsnorm_fwd_kernel<V><<<grid, kThreads, 0, (cudaStream_t)stream>>>((const uint4*)x, (const uint4*)w, (uint4*)y, rstd, rows, nvec, eps)
    if (vpt <= 1) BG_RMS_FWD(1); else if (vpt == 2) BG_RMS_FWD(2); else BG_RMS_FWD(4);
#undef BG_RMS_FWD
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, void* dx, float* dw_partial,
                              long long rows, long long cols, int n_partial, void* stream) {
    int rc = norm_args(rows, cols, "bg_rmsnorm_bwd");
    if (rc) return rc;
    if (n_partial < 1) return fail(BG_EINVAL, "bg_rmsnorm_bwd: n_partial must be >= 1");
    if (!BG_ALIGNED16(dy) || !BG_ALIGNED16(x) || !BG_ALIGNED16(w) || !BG_ALIGNED16(dx) || !BG_ALIGNED16(dw_partial))
        return fail(BG_EINVAL, "bg_rmsnorm_bwd: 16-B alignment");
    const int nvec = (int)(cols / 8), vpt = (nvec + kThreads - 1) / kThreads;
#define BG_RMS_BWD(V) rmsnorm_bwd_kernel<V><<<n_partial, kThreads, 0, (cudaStream_t)stream>>>((const uint4*)dy, (const uint4*)x, (const uint4*)w, rstd, (uint4*)dx, dw_partial, rows, nvec)
    if (vpt <= 1) BG_RMS_BWD(1); else if (vpt == 2) BG_RMS_BWD(2); else BG_RMS_BWD(4);
#undef BG_RMS_BWD
    BG_CHECK_LAUNCH();
    return BG_OK;
}

// (column blocks, row groups): about local_ctas CTAs in total, every CTA visiting >= 2 rows when there are enough of them
static dim3 swiglu_grid(long long rows, long long fvec) {
    const long long cb = (fvec + kThreads - 1) / kThreads;
    long long gy = g_tun.local_ctas / cb;
    if (gy < 1) gy = 1;
    if (gy > (rows + 1) / 2) gy = (rows + 1) / 2;
    if (gy > 65535) gy = 65535;
    return dim3((unsigned)cb, (unsigned)gy, 1);
}

extern "C" int bg_swiglu_fwd(const void* gate_up, void* y, long long rows, long long ffn, void* stream) {
    if (ffn <= 0 || ffn % 8) return fail(BG_EINVAL, "bg_swiglu_fwd: ffn %lld must be a multiple of 8", ffn);
    if (!BG_ALIGNED16(gate_up) || !BG_ALIGNED16(y)) return fail(BG_EINVAL, "bg_swiglu_fwd: 16-B alignment");
    if (rows == 0) return BG_OK;
    swiglu_fwd_kernel<<<swiglu_grid(rows, ffn / 8), kThreads, 0, (cudaStream_t)stream>>>((const uint4*)gate_up, (uint4*)y, rows, (int)(ffn / 8));
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_swiglu_bwd(const void* dy, const void* gate_up, void* dgate_up, long long rows, long long ffn, void* stream) {
    if (ffn <= 0 || ffn % 8) return fail(BG_EINVAL, "bg_swiglu_bwd: ffn %lld must be a multiple of 8", ffn);
    if (!BG_ALIGNED16(dy) || !BG_ALIGNED16(gate_up) || !BG_ALIGNED16(dgate_up)) return fail(BG_EINVAL, "bg_swiglu_bwd: 16-B alignment");
    if (rows == 0) return BG_OK;
    swiglu_bwd_kernel<<<swiglu_grid(rows, ffn / 8), kThreads, 0, (cudaStream_t)stream>>>((const uint4*)dy, (const uint4*)gate_up, (uint4*)dgate_up, rows,
                                                                                       (int)(ffn / 8));
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_qkv_rope(void* mixed, void* q, void* k, void* v, const float* cos_t, const float* sin_t, long long s,
                           long long b, long long ng, long long r, long long hn, int backward, void* stream) {
    if (hn <= 0 || hn % 16) return fail(BG_EINVAL, "bg_qkv_rope: head dim %lld must be a multiple of 16", hn);
    if (ng < 1 || r < 1) return fail(BG_EINVAL, "bg_qkv_rope: bad head counts");
    if (!BG_ALIGNED16(mixed) || !BG_ALIGNED16(q) || !BG_ALIGNED16(k) || !BG_ALIGNED16(v) || !BG_ALIGNED16(cos_t) || !BG_ALIGNED16(sin_t))
        return fail(BG_EINVAL, "bg_qkv_rope: 16-B alignment");
    const size_t total = (size_t)s * b * ng * (r + 2) * (hn / 16);
    if (total == 0) return BG_OK;
    const long long tokens = s * b;
    qkv_rope_kernel<<<(int)(tokens < g_tun.local_ctas ? tokens : g_tun.local_ctas), kThreads, 0, (cudaStream_t)stream>>>(
        (uint4*)mixed, (uint4*)q, (uint4*)k, (uint4*)v, cos_t, sin_t, s, b, (int)ng, (int)r, (int)hn, backward);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

static int ce_args(int dtype, long long vocab, const void* logits, const char* who) {
    if (dtype != BG_BF16 && dtype != BG_F32) return fail(BG_EUNSUPPORTED, "%s: dtype %d", who, dtype);
    if (vocab <= 0 || vocab % 8) return fail(BG_EINVAL, "%s: local vocab %lld must be a multiple of 8", who, vocab);
    if (!BG_ALIGNED16(logits)) return fail(BG_EINVAL, "%s: 16-B alignment", who);
    return BG_OK;
}

extern "C" int bg_ce_rowmax(const void* logits, int dtype, float* rowmax, long long rows, long long vocab, void* stream) {
    int rc = ce_args(dtype, vocab, logits, "bg_ce_rowmax");
    if (rc) return rc;
    if (rows == 0) return BG_OK;
    int grid = (int)(rows < g_tun.local_ctas ? rows : g_tun.local_ctas);
    if (dtype == BG_BF16) ce_rowmax_kernel<true><<<grid, kCeThreads, 0, (cudaStream_t)stream>>>(logits, rowmax, rows, vocab);
    else ce_rowmax_kernel<false><<<grid, kCeThreads, 0, (cudaStream_t)stream>>>(logits, rowmax, rows, vocab);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_ce_sumexp(const void* logits, int dtype, const long long* target, const float* rowmax, float* out2,
                            long long rows, long long vocab, long long vocab_start, void* stream) {
    int rc = ce_args(dtype, vocab, logits, "bg_ce_sumexp");
    if (rc) return rc;
    if (rows == 0) return BG_OK;
    int grid = (int)(rows < g_tun.local_ctas ? rows : g_tun.local_ctas);
    if (dtype == BG_BF16) ce_sumexp_kernel<true><<<grid, kCeThreads, 0, (cudaStream_t)stream>>>(logits, target, rowmax, out2, rows, vocab, vocab_start);
    else ce_sumexp_kernel<false><<<grid, kCeThreads, 0, (cudaStream_t)stream>>>(logits, target, rowmax, out2, rows, vocab, vocab_start);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_ce_bwd(void* logits, int dtype, const long long* target, const float* rowmax, const float* sum2,
                         const float* grad_loss, long long rows, long long vocab, long long vocab_start, void* stream) {
    int rc = ce_args(dtype, vocab, logits, "bg_ce_bwd");
    if (rc) return rc;
    if (rows == 0) return BG_OK;
    int grid = (int)(rows < g_tun.local_ctas ? rows : g_tun.local_ctas);
    if (dtype == BG_BF16) ce_bwd_kernel<true><<<grid, kCeThreads, 0, (cudaStream_t)stream>>>(logits, target, rowmax, sum2, grad_loss, rows, vocab, vocab_start);
    else ce_bwd_kernel<false><<<grid, kCeThreads, 0, (cudaStream_t)stream>>>(logits, target, rowmax, sum2, grad_loss, rows, vocab, vocab_start);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_layernorm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, long long rows,
                                long long cols, float eps, void* stream) {
    int rc = norm_args(rows, cols, "bg_layernorm_fwd");
    if (rc) return rc;
    if (!BG_ALIGNED16(x) || !BG_ALIGNED16(w) || !BG_ALIGNED16(b) || !BG_ALIGNED16(y)) return fail(BG_EINVAL, "bg_layernorm_fwd: 16-B alignment");
    if (rows == 0) return BG_OK;
    const int grid = (int)(rows < g_tun.local_ctas ? rows : g_tun.local_ctas);
    layernorm_fwd_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>((const uint4*)x, (const uint4*)w, (const uint4*)b, (uint4*)y, mean, rstd,
                                                                      rows, (int)(cols / 8), eps);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_layernorm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx,
                                float* dw_partial, float* db_partial, long long rows, long long cols, int n_partial, void* stream) {
    int rc = norm_args(rows, cols, "bg_layernorm_bwd");
    if (rc) return rc;
    if (n_partial < 1) return fail(BG_EINVAL, "bg_layernorm_bwd: n_partial must be >= 1");
    if (!BG_ALIGNED16(dy) || !BG_ALIGNED16(x) || !BG_ALIGNED16(w) || !BG_ALIGNED16(dx) || !BG_ALIGNED16(dw_partial) || !BG_ALIGNED16(db_partial))
        return fail(BG_EINVAL, "bg_layernorm_bwd: 16-B alignment");
    // (rows == 0 still launches: every one of the n_partial CTAs writes its partial rows, zeros if it visits no row)
    layernorm_bwd_kernel<<<n_partial, kThreads, 0, (cudaStream_t)stream>>>((const uint4*)dy, (const uint4*)x, (const uint4*)w, mean, rstd, (uint4*)dx,
                                                                           dw_partial, db_partial, rows, (int)(cols / 8));
    BG_CHECK_LAUNCH();
    return BG_OK;
}

// out = act(x + bias) when dy is null, else dy * act'(x + bias)
template <class Act>
static int bias_act(const char* who, const void* x, const void* bias, const void* dy, void* out, long long rows, long long cols,
                    void* stream) {
    if (cols <= 0 || cols % 8) return fail(BG_EINVAL, "%s: cols %lld must be a positive multiple of 8", who, cols);
    if (rows < 0) return fail(BG_EINVAL, "%s: rows %lld must be >= 0", who, rows);
    if (!BG_ALIGNED16(x) || !BG_ALIGNED16(bias) || !BG_ALIGNED16(dy) || !BG_ALIGNED16(out)) return fail(BG_EINVAL, "%s: 16-B alignment", who);
    if (rows == 0) return BG_OK;
    const int grid = local_grid((size_t)rows * cols / 8, kThreads);
    cudaStream_t st = (cudaStream_t)stream;
    const uint4 *xv = (const uint4*)x, *bv = (const uint4*)bias, *dv = (const uint4*)dy;
    if (dy == nullptr) bias_act_kernel<Act, false><<<grid, kThreads, 0, st>>>(xv, bv, dv, (uint4*)out, rows, (int)(cols / 8));
    else bias_act_kernel<Act, true><<<grid, kThreads, 0, st>>>(xv, bv, dv, (uint4*)out, rows, (int)(cols / 8));
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_bias_gelu(const void* x, const void* bias, const void* dy, void* out, long long rows, long long cols, int tanh_form,
                            void* stream) {
    if (tanh_form) return bias_act<GeluTanh>("bg_bias_gelu", x, bias, dy, out, rows, cols, stream);
    return bias_act<GeluErf>("bg_bias_gelu", x, bias, dy, out, rows, cols, stream);
}

extern "C" void bg_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
    const uint4 o = philox4x32_10(make_uint4(ctr[0], ctr[1], ctr[2], ctr[3]), make_uint2(key[0], key[1]));
    out[0] = o.x; out[1] = o.y; out[2] = o.z; out[3] = o.w;
}

static int dropout_args(long long rows, long long h, long long b_loc, long long seq_base, long long sample_base, double p,
                        unsigned seed, unsigned iteration, unsigned site, DropoutCoords* d, const char* who) {
    if (h <= 0 || h % 8) return fail(BG_EINVAL, "%s: hidden %lld must be a positive multiple of 8", who, h);
    if (h / 8 > (long long)kThreads * 65535) return fail(BG_EUNSUPPORTED, "%s: hidden %lld too wide", who, h);
    if (rows < 0 || b_loc < 1 || rows % b_loc) return fail(BG_EINVAL, "%s: rows %lld must be a multiple of b_loc %lld", who, rows, b_loc);
    if (seq_base < 0 || sample_base < 0 || seq_base + rows / b_loc > 0xffffffffLL || sample_base + b_loc > 0xffffffffLL)
        return fail(BG_EINVAL, "%s: token / sample coordinates must fit 32 bits", who);
    if (!(p >= 0.0 && p < 1.0)) return fail(BG_EINVAL, "%s: dropout probability %g must be in [0, 1)", who, p);
    d->b_loc = b_loc; d->seq_base = seq_base; d->sample_base = sample_base;
    d->threshold = (uint32_t)floor(p * 4294967296.0);
    d->scale = (float)(1.0 / (1.0 - p));
    d->seed = seed; d->iteration = iteration; d->site = site;
    return BG_OK;
}

// (column blocks, row groups) with about local_ctas CTAs in total
static dim3 dropout_grid(long long rows, long long nvec, long long want_rows) {
    const long long cb = (nvec + kThreads - 1) / kThreads;
    long long gy = want_rows > 0 ? want_rows : g_tun.local_ctas / cb;
    if (gy < 1) gy = 1;
    if (want_rows <= 0 && gy > rows) gy = rows > 0 ? rows : 1;
    if (gy > 65535) gy = 65535;
    return dim3((unsigned)cb, (unsigned)gy, 1);
}

// the sample map of an IdMask launch: BG_EINVAL for a null or not 4-B aligned one (its entries are read as 32-bit words)
template <class Mask>
static int sample_ids_arg(const uint32_t* sample_ids, DropoutCoords* d, const char* who) {
    if (!std::is_same<Mask, IdMask>::value) return BG_OK;
    if (sample_ids == nullptr || reinterpret_cast<uintptr_t>(sample_ids) % 4)
        return fail(BG_EINVAL, "%s: sample_ids must be non-null and 4-B aligned", who);
    d->sample_ids = sample_ids;
    return BG_OK;
}

// y = residual + keep * scale * (x + bias) under the element (dropout), element-at-a-sample-map or sample (drop path) mask
template <class Mask>
static int bias_dropout_add(const char* who, const void* x, const void* bias, int bias_dtype, const void* residual, void* y,
                            long long rows, long long h, long long b_loc, long long seq_base, long long sample_base, double p,
                            unsigned seed, unsigned iteration, unsigned site, void* stream, const uint32_t* sample_ids = nullptr) {
    DropoutCoords d;
    int rc = dropout_args(rows, h, b_loc, seq_base, sample_base, p, seed, iteration, site, &d, who);
    if (!rc) rc = sample_ids_arg<Mask>(sample_ids, &d, who);
    if (rc) return rc;
    if (bias != nullptr && bias_dtype != BG_BF16 && bias_dtype != BG_F32) return fail(BG_EUNSUPPORTED, "%s: bias dtype %d", who, bias_dtype);
    if (x == nullptr || y == nullptr || !BG_ALIGNED16(x) || !BG_ALIGNED16(bias) || !BG_ALIGNED16(residual) || !BG_ALIGNED16(y))
        return fail(BG_EINVAL, "%s: x and y must be non-null; 16-B alignment", who);
    if (rows == 0) return BG_OK;
    const dim3 grid = dropout_grid(rows, h / 8, 0);
    cudaStream_t st = (cudaStream_t)stream;
    if (bias != nullptr && bias_dtype == BG_F32)
        bias_dropout_add_kernel<Mask, true><<<grid, kThreads, 0, st>>>((const uint4*)x, bias, (const uint4*)residual, (uint4*)y, rows, (int)(h / 8), d);
    else
        bias_dropout_add_kernel<Mask, false><<<grid, kThreads, 0, st>>>((const uint4*)x, bias, (const uint4*)residual, (uint4*)y, rows, (int)(h / 8), d);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

// dx = keep * scale * dy and the dbias partials, the mask regenerated from the forward's arguments
template <class Mask>
static int dropout_bwd(const char* who, const void* dy, void* dx, float* dbias_partial, int n_partial, long long rows, long long h,
                       long long b_loc, long long seq_base, long long sample_base, double p, unsigned seed, unsigned iteration,
                       unsigned site, void* stream, const uint32_t* sample_ids = nullptr) {
    DropoutCoords d;
    int rc = dropout_args(rows, h, b_loc, seq_base, sample_base, p, seed, iteration, site, &d, who);
    if (!rc) rc = sample_ids_arg<Mask>(sample_ids, &d, who);
    if (rc) return rc;
    if (n_partial < 1 || n_partial > 65535) return fail(BG_EINVAL, "%s: n_partial %d must be in [1, 65535]", who, n_partial);
    if (dy == nullptr || dx == nullptr || !BG_ALIGNED16(dy) || !BG_ALIGNED16(dx) || !BG_ALIGNED16(dbias_partial))
        return fail(BG_EINVAL, "%s: dy and dx must be non-null; 16-B alignment", who);
    // (rows == 0 still launches: every one of the n_partial CTAs writes its partial row, zeros if it visits no row)
    dropout_bwd_kernel<Mask><<<dropout_grid(rows, h / 8, n_partial), kThreads, 0, (cudaStream_t)stream>>>((const uint4*)dy, (uint4*)dx,
                                                                                                         dbias_partial, rows, (int)(h / 8), d);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_dropout_add_fwd(const void* x, const void* bias, int bias_dtype, const void* residual, void* y, long long rows,
                                  long long h, long long b_loc, long long seq_base, long long sample_base, double p, unsigned seed,
                                  unsigned iteration, unsigned site, void* stream) {
    return bias_dropout_add<ElementMask>("bg_dropout_add_fwd", x, bias, bias_dtype, residual, y, rows, h, b_loc, seq_base, sample_base, p,
                                         seed, iteration, site, stream);
}

extern "C" int bg_dropout_bwd(const void* dy, void* dx, float* dbias_partial, int n_partial, long long rows, long long h, long long b_loc,
                              long long seq_base, long long sample_base, double p, unsigned seed, unsigned iteration, unsigned site,
                              void* stream) {
    return dropout_bwd<ElementMask>("bg_dropout_bwd", dy, dx, dbias_partial, n_partial, rows, h, b_loc, seq_base, sample_base, p, seed,
                                    iteration, site, stream);
}

extern "C" int bg_dropout_add_fwd_ids(const void* x, const void* bias, int bias_dtype, const void* residual, void* y, long long rows,
                                      long long h, long long b_loc, long long seq_base, const uint32_t* sample_ids, double p, unsigned seed,
                                      unsigned iteration, unsigned site, void* stream) {
    return bias_dropout_add<IdMask>("bg_dropout_add_fwd_ids", x, bias, bias_dtype, residual, y, rows, h, b_loc, seq_base, 0, p, seed,
                                    iteration, site, stream, sample_ids);
}

extern "C" int bg_dropout_bwd_ids(const void* dy, void* dx, float* dbias_partial, int n_partial, long long rows, long long h,
                                  long long b_loc, long long seq_base, const uint32_t* sample_ids, double p, unsigned seed,
                                  unsigned iteration, unsigned site, void* stream) {
    return dropout_bwd<IdMask>("bg_dropout_bwd_ids", dy, dx, dbias_partial, n_partial, rows, h, b_loc, seq_base, 0, p, seed, iteration,
                               site, stream, sample_ids);
}

extern "C" int bg_vit_patchify(const void* pixels, int pixel_dtype, void* out, long long batch, long long channels, long long height,
                               long long width, long long patch, long long rows_pad, void* stream) {
    const char* who = "bg_vit_patchify";
    if (pixel_dtype != BG_BF16 && pixel_dtype != BG_F32) return fail(BG_EUNSUPPORTED, "%s: pixel dtype %d", who, pixel_dtype);
    if (batch < 1 || channels < 1 || patch < 1 || height < patch || width < patch || height % patch || width % patch)
        return fail(BG_EINVAL, "%s: image %lldx%lldx%lld x %lld does not split into %lldx%lld patches", who, batch, channels, height, width,
                    patch, patch);
    const long long k = patch * patch * channels, P = (height / patch) * (width / patch);
    if (k % 8) return fail(BG_EINVAL, "%s: patch row p*p*C = %lld must be a multiple of 8", who, k);
    if (rows_pad < batch * P || rows_pad % 8) return fail(BG_EINVAL, "%s: rows_pad %lld must be a multiple of 8 >= B*P = %lld", who, rows_pad, batch * P);
    if (batch * channels * height * width > (1LL << 40) || k > (1LL << 24)) return fail(BG_EUNSUPPORTED, "%s: image too large", who);
    const size_t esz = pixel_dtype == BG_F32 ? 4 : 2;
    if ((uintptr_t)pixels % esz || !BG_ALIGNED16(out)) return fail(BG_EINVAL, "%s: alignment", who);
    const int grid = local_grid((size_t)rows_pad * (k / 8), kThreads);
    cudaStream_t st = (cudaStream_t)stream;
    if (pixel_dtype == BG_F32)
        vit_patchify_kernel<true><<<grid, kThreads, 0, st>>>(pixels, (uint4*)out, batch * P, rows_pad, (int)(k / 8), (int)channels,
                                                             (int)height, (int)width, (int)patch, (int)P);
    else
        vit_patchify_kernel<false><<<grid, kThreads, 0, st>>>(pixels, (uint4*)out, batch * P, rows_pad, (int)(k / 8), (int)channels,
                                                              (int)height, (int)width, (int)patch, (int)P);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

// shared checks of the two embedding entries: shapes (the dropout arguments as bg_dropout_add_fwd's, over s_run x batch rows)
static int vit_embed_args(long long batch, long long n_patches, long long s_run, long long h, long long sample_base, double p,
                          unsigned seed, unsigned iteration, unsigned site, DropoutCoords* d, const char* who) {
    if (batch < 1 || n_patches < 1 || s_run < n_patches + 1)
        return fail(BG_EINVAL, "%s: batch %lld, patches %lld and s_run %lld must satisfy batch >= 1, s_run > patches >= 1", who, batch,
                    n_patches, s_run);
    return dropout_args(s_run * batch, h, batch, 0, sample_base, p, seed, iteration, site, d, who);
}

// threads of a (column blocks, row groups) launch: one thread per 8-column vector, at most kThreads per CTA
static dim3 vit_block(long long nvec) {
    const long long t = (nvec + 31) / 32 * 32;
    return dim3((unsigned)(t < kThreads ? t : kThreads), 1, 1);
}

extern "C" int bg_vit_embed_fwd(const void* patch_out, const void* bias, const void* cls, const void* pos, void* y, long long batch,
                                long long n_patches, long long s_run, long long h, long long sample_base, double p, unsigned seed,
                                unsigned iteration, unsigned site, void* stream) {
    DropoutCoords d;
    int rc = vit_embed_args(batch, n_patches, s_run, h, sample_base, p, seed, iteration, site, &d, "bg_vit_embed_fwd");
    if (rc) return rc;
    if (patch_out == nullptr || bias == nullptr || cls == nullptr || pos == nullptr || y == nullptr || !BG_ALIGNED16(patch_out) ||
        !BG_ALIGNED16(bias) || !BG_ALIGNED16(cls) || !BG_ALIGNED16(pos) || !BG_ALIGNED16(y))
        return fail(BG_EINVAL, "bg_vit_embed_fwd: pointers must be non-null and 16-B aligned");
    const long long nvec = h / 8;
    const dim3 block = vit_block(nvec);
    long long gy = g_tun.local_ctas / ((nvec + block.x - 1) / block.x);
    gy = gy < 1 ? 1 : (gy > s_run ? s_run : gy);
    const dim3 grid((unsigned)((nvec + block.x - 1) / block.x), (unsigned)(gy > 65535 ? 65535 : gy), 1);
    cudaStream_t st = (cudaStream_t)stream;
    const uint4 *pv = (const uint4*)patch_out, *bv = (const uint4*)bias, *cv = (const uint4*)cls, *qv = (const uint4*)pos;
    if (p > 0.0) vit_embed_fwd_kernel<true><<<grid, block, 0, st>>>(pv, bv, cv, qv, (uint4*)y, batch, n_patches, s_run, (int)nvec, d);
    else vit_embed_fwd_kernel<false><<<grid, block, 0, st>>>(pv, bv, cv, qv, (uint4*)y, batch, n_patches, s_run, (int)nvec, d);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_vit_embed_bwd(const void* dy, void* dpatch, float* dpos, float* dbias_partial, int n_partial, long long batch,
                                long long n_patches, long long s_run, long long rows_pad, long long h, long long sample_base, double p,
                                unsigned seed, unsigned iteration, unsigned site, void* stream) {
    DropoutCoords d;
    int rc = vit_embed_args(batch, n_patches, s_run, h, sample_base, p, seed, iteration, site, &d, "bg_vit_embed_bwd");
    if (rc) return rc;
    if (rows_pad < batch * n_patches || rows_pad % 8)
        return fail(BG_EINVAL, "bg_vit_embed_bwd: rows_pad %lld must be a multiple of 8 >= batch x patches = %lld", rows_pad, batch * n_patches);
    if (n_partial < 1 || n_partial > 65535) return fail(BG_EINVAL, "bg_vit_embed_bwd: n_partial %d must be in [1, 65535]", n_partial);
    if (dy == nullptr || dpatch == nullptr || dpos == nullptr || dbias_partial == nullptr || !BG_ALIGNED16(dy) || !BG_ALIGNED16(dpatch) ||
        !BG_ALIGNED16(dpos) || !BG_ALIGNED16(dbias_partial))
        return fail(BG_EINVAL, "bg_vit_embed_bwd: pointers must be non-null and 16-B aligned");
    const long long nvec = h / 8;
    const dim3 block = vit_block(nvec);
    const dim3 grid((unsigned)((nvec + block.x - 1) / block.x), (unsigned)n_partial, 1);
    cudaStream_t st = (cudaStream_t)stream;
    // (every one of the n_partial row groups writes its dbias partial, zeros if it visits no row)
    if (p > 0.0)
        vit_embed_bwd_kernel<true><<<grid, block, 0, st>>>((const uint4*)dy, (uint4*)dpatch, dpos, dbias_partial, batch, n_patches, rows_pad,
                                                           (int)nvec, d);
    else
        vit_embed_bwd_kernel<false><<<grid, block, 0, st>>>((const uint4*)dy, (uint4*)dpatch, dpos, dbias_partial, batch, n_patches,
                                                            rows_pad, (int)nvec, d);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_bias_tanh(const void* x, const void* bias, const void* dy, void* out, long long rows, long long cols, void* stream) {
    return bias_act<Tanh>("bg_bias_tanh", x, bias, dy, out, rows, cols, stream);
}

// ---- Swin ---------------------------------------------------------------------------------------------------------------------
static int swin_window_args(long long mb, long long T, long long T_run, long long nW, long long L, const char* who) {
    if (mb < 1 || nW < 1 || L < 1 || T != nW * L || T_run < T)
        return fail(BG_EINVAL, "%s: mb %lld, windows %lld x %lld tokens and tokens %lld / %lld (run) must satisfy mb >= 1, tokens = windows "
                    "x window tokens <= tokens_run", who, mb, nW, L, T, T_run);
    if (T_run * mb > (1LL << 31) || L > (1 << 20)) return fail(BG_EUNSUPPORTED, "%s: too many rows", who);
    return BG_OK;
}

extern "C" int bg_swin_window_qkv_fwd(const void* mixed, const void* bias, const int* map, void* q, void* k, void* v, long long mb,
                                      long long tokens, long long tokens_run, long long n_windows, long long window_tokens, long long heads,
                                      long long head_dim, void* stream) {
    const char* who = "bg_swin_window_qkv_fwd";
    int rc = swin_window_args(mb, tokens, tokens_run, n_windows, window_tokens, who);
    if (rc) return rc;
    if (heads < 1 || head_dim < 8 || head_dim % 8 || heads * head_dim * 3 / 8 > (1 << 24))
        return fail(BG_EINVAL, "%s: heads %lld x head_dim %lld (a multiple of 8)", who, heads, head_dim);
    if (mixed == nullptr || bias == nullptr || map == nullptr || q == nullptr || k == nullptr || v == nullptr || !BG_ALIGNED16(mixed) ||
        !BG_ALIGNED16(bias) || !BG_ALIGNED16(q) || !BG_ALIGNED16(k) || !BG_ALIGNED16(v) || (uintptr_t)map % 4)
        return fail(BG_EINVAL, "%s: pointers must be non-null and aligned", who);
    const int hv = (int)(head_dim / 8);
    const int grid = local_grid((size_t)mb * tokens * heads * 3 * hv, kThreads);
    swin_window_qkv_fwd_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>((const uint4*)mixed, (const uint4*)bias, map, (uint4*)q,
                                                                           (uint4*)k, (uint4*)v, mb, n_windows, (int)window_tokens,
                                                                           (int)heads, hv);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_swin_window_qkv_bwd(const void* dq, const void* dk, const void* dv, void* dmixed, float* dbias_partial, int n_partial,
                                      const int* inv, long long mb, long long tokens, long long tokens_run, long long n_windows,
                                      long long window_tokens, long long heads, long long head_dim, void* stream) {
    const char* who = "bg_swin_window_qkv_bwd";
    int rc = swin_window_args(mb, tokens, tokens_run, n_windows, window_tokens, who);
    if (rc) return rc;
    if (heads < 1 || head_dim < 8 || head_dim % 8 || heads * head_dim * 3 / 8 > (long long)kThreads * 65535)
        return fail(BG_EINVAL, "%s: heads %lld x head_dim %lld (a multiple of 8)", who, heads, head_dim);
    if (n_partial < 1 || n_partial > 65535) return fail(BG_EINVAL, "%s: n_partial %d must be in [1, 65535]", who, n_partial);
    if (dq == nullptr || dk == nullptr || dv == nullptr || dmixed == nullptr || dbias_partial == nullptr || inv == nullptr ||
        !BG_ALIGNED16(dq) || !BG_ALIGNED16(dk) || !BG_ALIGNED16(dv) || !BG_ALIGNED16(dmixed) || !BG_ALIGNED16(dbias_partial) ||
        (uintptr_t)inv % 4)
        return fail(BG_EINVAL, "%s: pointers must be non-null and aligned", who);
    const long long ncol = heads * 3 * (head_dim / 8);
    const dim3 block = vit_block(ncol);
    const dim3 grid((unsigned)((ncol + block.x - 1) / block.x), (unsigned)n_partial, 1);
    swin_window_qkv_bwd_kernel<<<grid, block, 0, (cudaStream_t)stream>>>((const uint4*)dq, (const uint4*)dk, (const uint4*)dv,
                                                                         (uint4*)dmixed, dbias_partial, inv, mb, tokens, tokens_run,
                                                                         n_windows, (int)window_tokens, (int)heads, (int)(head_dim / 8));
    BG_CHECK_LAUNCH();
    return BG_OK;
}

static int swin_window_merge(const void* src, void* dst, const int* map, const int* inv, long long mb, long long tokens,
                             long long tokens_run, long long n_windows, long long window_tokens, long long cols, bool backward,
                             void* stream, const char* who) {
    int rc = swin_window_args(mb, tokens, tokens_run, n_windows, window_tokens, who);
    if (rc) return rc;
    if (cols <= 0 || cols % 8 || cols / 8 > (1 << 24)) return fail(BG_EINVAL, "%s: cols %lld must be a positive multiple of 8", who, cols);
    if (src == nullptr || dst == nullptr || map == nullptr || inv == nullptr || !BG_ALIGNED16(src) || !BG_ALIGNED16(dst) ||
        (uintptr_t)map % 4 || (uintptr_t)inv % 4)
        return fail(BG_EINVAL, "%s: pointers must be non-null and aligned", who);
    const size_t rows = backward ? (size_t)mb * tokens : (size_t)mb * tokens_run;
    const int grid = local_grid(rows * (cols / 8), kThreads);
    cudaStream_t st = (cudaStream_t)stream;
    if (backward)
        swin_window_merge_kernel<true><<<grid, kThreads, 0, st>>>((const uint4*)src, (uint4*)dst, map, inv, mb, tokens, tokens_run,
                                                                  n_windows, (int)window_tokens, (int)(cols / 8));
    else
        swin_window_merge_kernel<false><<<grid, kThreads, 0, st>>>((const uint4*)src, (uint4*)dst, map, inv, mb, tokens, tokens_run,
                                                                   n_windows, (int)window_tokens, (int)(cols / 8));
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_swin_window_merge_fwd(const void* windows, void* rows, const int* map, const int* inv, long long mb, long long tokens,
                                        long long tokens_run, long long n_windows, long long window_tokens, long long cols, void* stream) {
    return swin_window_merge(windows, rows, map, inv, mb, tokens, tokens_run, n_windows, window_tokens, cols, false, stream,
                             "bg_swin_window_merge_fwd");
}

extern "C" int bg_swin_window_merge_bwd(const void* drows, void* dwindows, const int* map, const int* inv, long long mb, long long tokens,
                                        long long tokens_run, long long n_windows, long long window_tokens, long long cols, void* stream) {
    return swin_window_merge(drows, dwindows, map, inv, mb, tokens, tokens_run, n_windows, window_tokens, cols, true, stream,
                             "bg_swin_window_merge_bwd");
}

static int merge_ln_args(long long mb, long long height, long long width, long long r, int in_bsh, long long rows_in, long long cols_in,
                         long long tokens_out_run, MergeGeom* g, const char* who) {
    if (r != 1 && r != 2) return fail(BG_EINVAL, "%s: merge factor %lld must be 1 or 2", who, r);
    if (mb < 1 || height < r || width < r || height % r || width % r)
        return fail(BG_EINVAL, "%s: a %lldx%lld token grid does not merge in %lldx%lld blocks (mb %lld)", who, height, width, r, r, mb);
    if (cols_in <= 0 || cols_in % 8) return fail(BG_EINVAL, "%s: cols %lld must be a positive multiple of 8", who, cols_in);
    if (r * r * cols_in / 8 > (long long)kMergeVpt * kThreads)
        return fail(BG_EUNSUPPORTED, "%s: merged row of %lld columns > %d", who, r * r * cols_in, kMergeVpt * kThreads * 8);
    const long long T_in = height * width, T_out = T_in / (r * r);
    if (rows_in < mb * T_in) return fail(BG_EINVAL, "%s: rows_in %lld < mb x tokens = %lld", who, rows_in, mb * T_in);
    if (tokens_out_run < T_out) return fail(BG_EINVAL, "%s: tokens_out_run %lld < merged tokens %lld", who, tokens_out_run, T_out);
    if (rows_in > (1LL << 31) || tokens_out_run * mb > (1LL << 31)) return fail(BG_EUNSUPPORTED, "%s: too many rows", who);
    g->mb = mb; g->T_in = T_in; g->T_out = T_out; g->T_out_run = tokens_out_run;
    g->Wi = (int)width; g->Wo = (int)(width / r); g->r = (int)r; g->cvec_in = (int)(cols_in / 8); g->in_bsh = in_bsh ? 1 : 0;
    return BG_OK;
}

extern "C" int bg_swin_merge_ln_fwd(const void* x, const void* add_bias, const void* w, const void* b, void* y, float* mean, float* rstd,
                                    long long mb, long long height, long long width, long long r, int in_bsh, long long rows_in,
                                    long long cols_in, long long tokens_out_run, float eps, void* stream) {
    const char* who = "bg_swin_merge_ln_fwd";
    MergeGeom g;
    int rc = merge_ln_args(mb, height, width, r, in_bsh, rows_in, cols_in, tokens_out_run, &g, who);
    if (rc) return rc;
    if (x == nullptr || w == nullptr || b == nullptr || y == nullptr || mean == nullptr || rstd == nullptr || !BG_ALIGNED16(x) ||
        !BG_ALIGNED16(add_bias) || !BG_ALIGNED16(w) || !BG_ALIGNED16(b) || !BG_ALIGNED16(y) || (uintptr_t)mean % 4 || (uintptr_t)rstd % 4)
        return fail(BG_EINVAL, "%s: pointers must be non-null (add_bias may be) and aligned", who);
    const int grid = local_grid((size_t)tokens_out_run * mb, 1);
    cudaStream_t st = (cudaStream_t)stream;
    if (add_bias != nullptr)
        swin_merge_ln_fwd_kernel<true><<<grid, kThreads, 0, st>>>((const uint4*)x, (const uint4*)add_bias, (const uint4*)w, (const uint4*)b,
                                                                  (uint4*)y, mean, rstd, g, eps);
    else
        swin_merge_ln_fwd_kernel<false><<<grid, kThreads, 0, st>>>((const uint4*)x, nullptr, (const uint4*)w, (const uint4*)b, (uint4*)y,
                                                                   mean, rstd, g, eps);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_swin_merge_ln_bwd(const void* dy, const void* x, const void* add_bias, const void* w, const float* mean, const float* rstd,
                                    void* dx, float* dw_partial, float* db_partial, float* dbias_partial, int n_partial, long long mb,
                                    long long height, long long width, long long r, int in_bsh, long long rows_in, long long cols_in,
                                    void* stream) {
    const char* who = "bg_swin_merge_ln_bwd";
    MergeGeom g;
    int rc = merge_ln_args(mb, height, width, r, in_bsh, rows_in, cols_in, (height / (r < 1 ? 1 : r)) * (width / (r < 1 ? 1 : r)), &g, who);
    if (rc) return rc;
    if (n_partial < 1 || n_partial > 65535) return fail(BG_EINVAL, "%s: n_partial %d must be in [1, 65535]", who, n_partial);
    if ((add_bias == nullptr) != (dbias_partial == nullptr)) return fail(BG_EINVAL, "%s: add_bias and dbias_partial go together", who);
    if (dy == nullptr || x == nullptr || w == nullptr || mean == nullptr || rstd == nullptr || dx == nullptr || dw_partial == nullptr ||
        db_partial == nullptr || !BG_ALIGNED16(dy) || !BG_ALIGNED16(x) || !BG_ALIGNED16(add_bias) || !BG_ALIGNED16(w) ||
        !BG_ALIGNED16(dx) || !BG_ALIGNED16(dw_partial) || !BG_ALIGNED16(db_partial) || !BG_ALIGNED16(dbias_partial) ||
        (uintptr_t)mean % 4 || (uintptr_t)rstd % 4)
        return fail(BG_EINVAL, "%s: pointers must be non-null (add_bias / dbias_partial may be) and aligned", who);
    const int nvec = (int)(r * r * cols_in / 8);
    cudaStream_t st = (cudaStream_t)stream;
    const uint4 *dyv = (const uint4*)dy, *xv = (const uint4*)x, *bv = (const uint4*)add_bias, *wv = (const uint4*)w;
#define BG_MERGE_BWD(V, B) swin_merge_ln_bwd_kernel<V, B><<<n_partial, kThreads, 0, st>>>(dyv, xv, bv, wv, mean, rstd, (uint4*)dx, dw_partial, db_partial, dbias_partial, g, rows_in)
    const bool bias = add_bias != nullptr;
    if (nvec <= kThreads) { if (bias) BG_MERGE_BWD(1, true); else BG_MERGE_BWD(1, false); }
    else if (nvec <= 2 * kThreads) { if (bias) BG_MERGE_BWD(2, true); else BG_MERGE_BWD(2, false); }
    else { if (bias) BG_MERGE_BWD(kMergeVpt, true); else BG_MERGE_BWD(kMergeVpt, false); }
#undef BG_MERGE_BWD
    BG_CHECK_LAUNCH();
    return BG_OK;
}

static int mean_pool_args(long long tokens, long long tokens_run, long long mb, long long cols, const char* who) {
    if (tokens < 1 || tokens_run < tokens || mb < 1) return fail(BG_EINVAL, "%s: tokens %lld / %lld (run), mb %lld", who, tokens, tokens_run, mb);
    if (cols <= 0 || cols % 8) return fail(BG_EINVAL, "%s: cols %lld must be a positive multiple of 8", who, cols);
    if (tokens_run * mb * (cols / 8) > (1LL << 40)) return fail(BG_EUNSUPPORTED, "%s: too large", who);
    return BG_OK;
}

extern "C" int bg_swin_mean_pool_fwd(const void* x, void* y, long long tokens, long long tokens_run, long long mb, long long rows_out,
                                     long long cols, void* stream) {
    const char* who = "bg_swin_mean_pool_fwd";
    int rc = mean_pool_args(tokens, tokens_run, mb, cols, who);
    if (rc) return rc;
    if (rows_out < mb) return fail(BG_EINVAL, "%s: rows_out %lld < mb %lld", who, rows_out, mb);
    if (x == nullptr || y == nullptr || !BG_ALIGNED16(x) || !BG_ALIGNED16(y)) return fail(BG_EINVAL, "%s: pointers must be non-null and 16-B aligned", who);
    const int grid = local_grid((size_t)rows_out * (cols / 8), kThreads);
    swin_mean_pool_kernel<false><<<grid, kThreads, 0, (cudaStream_t)stream>>>((const uint4*)x, (uint4*)y, tokens, tokens_run, mb, rows_out,
                                                                             (int)(cols / 8));
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_swin_mean_pool_bwd(const void* dy, void* dx, long long tokens, long long tokens_run, long long mb, long long cols,
                                     void* stream) {
    const char* who = "bg_swin_mean_pool_bwd";
    int rc = mean_pool_args(tokens, tokens_run, mb, cols, who);
    if (rc) return rc;
    if (dy == nullptr || dx == nullptr || !BG_ALIGNED16(dy) || !BG_ALIGNED16(dx)) return fail(BG_EINVAL, "%s: pointers must be non-null and 16-B aligned", who);
    const int grid = local_grid((size_t)tokens_run * mb * (cols / 8), kThreads);
    swin_mean_pool_kernel<true><<<grid, kThreads, 0, (cudaStream_t)stream>>>((const uint4*)dy, (uint4*)dx, tokens, tokens_run, mb, 0,
                                                                            (int)(cols / 8));
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_drop_path_add_fwd(const void* x, const void* bias, int bias_dtype, const void* residual, void* y, long long rows,
                                    long long h, long long b_loc, long long sample_base, double p, unsigned seed, unsigned iteration,
                                    unsigned site, void* stream) {
    return bias_dropout_add<SampleMask>("bg_drop_path_add_fwd", x, bias, bias_dtype, residual, y, rows, h, b_loc, 0, sample_base, p, seed,
                                        iteration, site, stream);
}

extern "C" int bg_drop_path_add_bwd(const void* dy, void* dx, float* dbias_partial, int n_partial, long long rows, long long h,
                                    long long b_loc, long long sample_base, double p, unsigned seed, unsigned iteration, unsigned site,
                                    void* stream) {
    return dropout_bwd<SampleMask>("bg_drop_path_add_bwd", dy, dx, dbias_partial, n_partial, rows, h, b_loc, 0, sample_base, p, seed,
                                   iteration, site, stream);
}

// ---- Swin relative-position bias (HF SwinSelfAttention.relative_position_bias_table) ------------------------------------------
// The additive attention mask of one block, [mb * nW][heads][L][ld] bf16 (ld >= L, a multiple of 8; columns L .. ld - 1 zero):
// element (n, h, i, j) = table[index[i * L + j]][h] rounded to bf16, or -inf where the shift mask of window n % nW separates i and j.
// A thread forms one 16-B vector (8 columns of row i of window w, head h) and stores it for every sample b (window b * nW + w),
// so the index, table and mask reads are shared by the mb copies.
template <typename T>
__global__ void __launch_bounds__(kThreads) swin_rel_bias_fwd_kernel(const T* __restrict__ table, const int* __restrict__ index,
                                                                     const unsigned char* __restrict__ mask, uint4* __restrict__ out,
                                                                     long long mb, long long nW, int heads, int L, int lv) {
    const size_t tile = (size_t)nW * heads * L * lv, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < tile; v += stride) {
        const size_t row = v / lv;
        const int jv = (int)(v - row * lv);
        const size_t wh = row / L;
        const int i = (int)(row - wh * L);
        const long long w = (long long)(wh / heads);
        const int h = (int)(wh - (size_t)w * heads);
        const unsigned char* mrow = mask != nullptr ? mask + ((size_t)w * L + i) * L : nullptr;
        float f[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int j = jv * 8 + e;
            f[e] = 0.f;
            if (j < L) {
                f[e] = (float)__ldg(table + (size_t)__ldg(index + i * L + j) * heads + h);
                if (mrow != nullptr && __ldg(mrow + j)) f[e] = -INFINITY;
            }
        }
        const uint4 packed = pack8(f);
        for (long long b = 0; b < mb; ++b) st16(out + (size_t)b * tile + v, packed);
    }
}

// Its backward: dtable_partial[p][t][h] = the sum, over the cells c = i * L + j listed for entry t (cells[offsets[t]] ..
// cells[offsets[t + 1] - 1], in that order), of the fp32 sum over windows n = p, p + n_partial, ... (ascending) of dbias[n][h][i][j].
// grid = (heads, n_partial); a thread owns whole 8-column vectors of the L x ld tile, so every sum has one fixed order.  The
// per-cell sums wait in shared memory [L * L] fp32 for the gather by table entry.
__global__ void __launch_bounds__(kThreads) swin_rel_bias_bwd_kernel(const uint4* __restrict__ dbias, const int* __restrict__ cells,
                                                                     const int* __restrict__ offsets, float* __restrict__ partial,
                                                                     long long N, int L, int lv, int n_table) {
    extern __shared__ float cell_sum[];
    const int h = blockIdx.x, heads = gridDim.x, p = blockIdx.y, np = gridDim.y;
    const int nvec = L * lv;
    const size_t step = (size_t)np * heads * nvec;
    for (int u = threadIdx.x; u < nvec; u += blockDim.x) {
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
        const uint4* src = dbias + ((size_t)p * heads + h) * nvec + u;
        long long n = p;
        for (; n + 3LL * np < N; n += 4LL * np, src += 4 * step) {
            uint4 g[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) g[k] = ld16_stream(src + k * step);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float f[8];
                unpack8(g[k], f);
#pragma unroll
                for (int e = 0; e < 8; ++e) acc[e] = __fadd_rn(acc[e], f[e]);
            }
        }
        for (; n < N; n += np, src += step) {
            float f[8];
            unpack8(ld16_stream(src), f);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = __fadd_rn(acc[e], f[e]);
        }
        const int i = u / lv, j0 = (u - i * lv) * 8;
#pragma unroll
        for (int e = 0; e < 8; ++e)
            if (j0 + e < L) cell_sum[i * L + j0 + e] = acc[e];
    }
    __syncthreads();
    for (int t = threadIdx.x; t < n_table; t += blockDim.x) {
        float s = 0.f;
        for (int k = __ldg(offsets + t), end = __ldg(offsets + t + 1); k < end; ++k) s = __fadd_rn(s, cell_sum[__ldg(cells + k)]);
        partial[((size_t)p * n_table + t) * heads + h] = s;
    }
}

static const size_t kRelBiasMaxSmem = 200 * 1024;

static int rel_bias_args(long long mb, long long n_windows, long long heads, long long window, long long window_tokens, long long ld,
                         const char* who) {
    if (mb < 1 || n_windows < 1 || heads < 1 || window < 1)
        return fail(BG_EINVAL, "%s: mb %lld, windows %lld, heads %lld and window %lld must be >= 1", who, mb, n_windows, heads, window);
    if (window_tokens != window * window)
        return fail(BG_EINVAL, "%s: window_tokens %lld is not window %lld squared", who, window_tokens, window);
    if (ld < window_tokens || ld % 8)
        return fail(BG_EINVAL, "%s: row stride %lld must be a multiple of 8 >= window_tokens %lld", who, ld, window_tokens);
    if (heads > 65535 || (size_t)window_tokens * window_tokens * sizeof(float) > kRelBiasMaxSmem ||
        mb * n_windows * heads * window_tokens * ld > (1LL << 40))
        return fail(BG_EUNSUPPORTED, "%s: %lld heads, a %lld-token window or %lld windows is too large", who, heads, window_tokens,
                    mb * n_windows);
    return BG_OK;
}

extern "C" int bg_swin_rel_bias_fwd(const void* table, int table_dtype, const int* index, const unsigned char* shift_mask, void* bias,
                                    long long mb, long long n_windows, long long heads, long long window, long long window_tokens,
                                    long long ld, void* stream) {
    const char* who = "bg_swin_rel_bias_fwd";
    int rc = rel_bias_args(mb, n_windows, heads, window, window_tokens, ld, who);
    if (rc) return rc;
    if (table_dtype != BG_BF16 && table_dtype != BG_F32) return fail(BG_EUNSUPPORTED, "%s: table dtype %d", who, table_dtype);
    if (table == nullptr || index == nullptr || bias == nullptr || (uintptr_t)table % (table_dtype == BG_F32 ? 4 : 2) ||
        (uintptr_t)index % 4 || !BG_ALIGNED16(bias))
        return fail(BG_EINVAL, "%s: pointers must be non-null (shift_mask may be) and aligned", who);
    const int L = (int)window_tokens, lv = (int)(ld / 8);
    const int grid = local_grid((size_t)n_windows * heads * L * lv, kThreads);
    cudaStream_t st = (cudaStream_t)stream;
    if (table_dtype == BG_F32)
        swin_rel_bias_fwd_kernel<float><<<grid, kThreads, 0, st>>>((const float*)table, index, shift_mask, (uint4*)bias, mb, n_windows,
                                                                   (int)heads, L, lv);
    else
        swin_rel_bias_fwd_kernel<__nv_bfloat16><<<grid, kThreads, 0, st>>>((const __nv_bfloat16*)table, index, shift_mask, (uint4*)bias,
                                                                           mb, n_windows, (int)heads, L, lv);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_swin_rel_bias_bwd(const void* dbias, const int* cells, const int* offsets, float* dtable_partial, int n_partial,
                                    long long mb, long long n_windows, long long heads, long long window, long long window_tokens,
                                    long long ld, void* stream) {
    const char* who = "bg_swin_rel_bias_bwd";
    int rc = rel_bias_args(mb, n_windows, heads, window, window_tokens, ld, who);
    if (rc) return rc;
    if (n_partial < 1 || n_partial > 65535) return fail(BG_EINVAL, "%s: n_partial %d must be in [1, 65535]", who, n_partial);
    if (dbias == nullptr || cells == nullptr || offsets == nullptr || dtable_partial == nullptr || !BG_ALIGNED16(dbias) ||
        (uintptr_t)cells % 4 || (uintptr_t)offsets % 4 || (uintptr_t)dtable_partial % 4)
        return fail(BG_EINVAL, "%s: pointers must be non-null and aligned", who);
    const int L = (int)window_tokens;
    const size_t smem = (size_t)L * L * sizeof(float);
    if (smem > 48 * 1024)          // above the default dynamic shared memory (w = 12: 81 KiB)
        BG_CUDA(cudaFuncSetAttribute(swin_rel_bias_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRelBiasMaxSmem));
    const dim3 grid((unsigned)heads, (unsigned)n_partial, 1);
    swin_rel_bias_bwd_kernel<<<grid, kThreads, smem, (cudaStream_t)stream>>>((const uint4*)dbias, cells, offsets, dtable_partial,
                                                                              mb * n_windows, L, (int)(ld / 8),
                                                                              (int)((2 * window - 1) * (2 * window - 1)));
    BG_CHECK_LAUNCH();
    return BG_OK;
}

// ---- T5 cross-attention ---------------------------------------------------------------------------------------------------------
static int cross_attn_args(long long s_q, long long s_k, long long batch, long long heads, long long head_dim, const char* who) {
    if (s_q < 1 || s_k < 1 || batch < 1 || heads < 1 || head_dim < 8 || head_dim % 8)
        return fail(BG_EINVAL, "%s: s_q %lld, s_k %lld, batch %lld, heads %lld must be >= 1 and head_dim %lld a positive multiple of 8", who,
                    s_q, s_k, batch, heads, head_dim);
    if (heads * 3 * (head_dim / 8) > (long long)kThreads * 65535 || (s_q > s_k ? s_q : s_k) * batch > (1LL << 40))
        return fail(BG_EUNSUPPORTED, "%s: too many rows or columns", who);
    return BG_OK;
}

extern "C" int bg_cross_attn_qkv_fwd(const void* q_mixed, const void* q_bias, const void* kv_mixed, const void* kv_bias, void* q, void* k,
                                     void* v, long long s_q, long long s_k, long long batch, long long heads, long long head_dim,
                                     void* stream) {
    const char* who = "bg_cross_attn_qkv_fwd";
    int rc = cross_attn_args(s_q, s_k, batch, heads, head_dim, who);
    if (rc) return rc;
    if (q_mixed == nullptr || kv_mixed == nullptr || q == nullptr || k == nullptr || v == nullptr || !BG_ALIGNED16(q_mixed) ||
        !BG_ALIGNED16(q_bias) || !BG_ALIGNED16(kv_mixed) || !BG_ALIGNED16(kv_bias) || !BG_ALIGNED16(q) || !BG_ALIGNED16(k) ||
        !BG_ALIGNED16(v))
        return fail(BG_EINVAL, "%s: pointers must be non-null (the biases may be null) and 16-B aligned", who);
    const int hv = (int)(head_dim / 8);
    const int grid = local_grid((size_t)(s_q + 2 * s_k) * batch * heads * hv, kThreads);
    cross_attn_qkv_fwd_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>((const uint4*)q_mixed, (const uint4*)q_bias,
                                                                          (const uint4*)kv_mixed, (const uint4*)kv_bias, (uint4*)q,
                                                                          (uint4*)k, (uint4*)v, s_q, s_k, batch, (int)heads, hv);
    BG_CHECK_LAUNCH();
    return BG_OK;
}

extern "C" int bg_cross_attn_qkv_bwd(const void* dq, const void* dk, const void* dv, void* dq_mixed, void* dkv_mixed, float* dbias_partial,
                                     int n_partial, long long s_q, long long s_k, long long batch, long long heads, long long head_dim,
                                     void* stream) {
    const char* who = "bg_cross_attn_qkv_bwd";
    int rc = cross_attn_args(s_q, s_k, batch, heads, head_dim, who);
    if (rc) return rc;
    if (n_partial < 1 || n_partial > 65535) return fail(BG_EINVAL, "%s: n_partial %d must be in [1, 65535]", who, n_partial);
    if (dq == nullptr || dk == nullptr || dv == nullptr || dq_mixed == nullptr || dkv_mixed == nullptr || dbias_partial == nullptr ||
        !BG_ALIGNED16(dq) || !BG_ALIGNED16(dk) || !BG_ALIGNED16(dv) || !BG_ALIGNED16(dq_mixed) || !BG_ALIGNED16(dkv_mixed) ||
        !BG_ALIGNED16(dbias_partial))
        return fail(BG_EINVAL, "%s: pointers must be non-null and 16-B aligned", who);
    const long long ncol = heads * 3 * (head_dim / 8);
    const dim3 block = vit_block(ncol);
    const dim3 grid((unsigned)((ncol + block.x - 1) / block.x), (unsigned)n_partial, 1);
    cross_attn_qkv_bwd_kernel<<<grid, block, 0, (cudaStream_t)stream>>>((const uint4*)dq, (const uint4*)dk, (const uint4*)dv,
                                                                        (uint4*)dq_mixed, (uint4*)dkv_mixed, dbias_partial, s_q, s_k, batch,
                                                                        (int)heads, (int)(head_dim / 8));
    BG_CHECK_LAUNCH();
    return BG_OK;
}

// loads every kernel of this file up front (see bg_preload_coll in bg_coll.cu)
int bg_preload_ops() {
#define K(f) reinterpret_cast<const void*>(&f)
    const void* kernels[] = {K((cast_kernel<true, true>)), K((cast_kernel<true, false>)), K((cast_kernel<false, true>)), K((cast_kernel<false, false>)),
                             K(rmsnorm_fwd_kernel<1>), K(rmsnorm_fwd_kernel<2>), K(rmsnorm_fwd_kernel<4>), K(rmsnorm_bwd_kernel<1>), K(rmsnorm_bwd_kernel<2>), K(rmsnorm_bwd_kernel<4>), K(layernorm_fwd_kernel), K(layernorm_bwd_kernel),
                             K((bias_act_kernel<GeluTanh, false>)), K((bias_act_kernel<GeluErf, false>)), K((bias_act_kernel<Tanh, false>)),
                             K((bias_act_kernel<GeluTanh, true>)), K((bias_act_kernel<GeluErf, true>)), K((bias_act_kernel<Tanh, true>)),
                             K(swiglu_fwd_kernel), K(swiglu_bwd_kernel), K(qkv_rope_kernel),
                             K(ce_rowmax_kernel<true>), K(ce_rowmax_kernel<false>), K(ce_sumexp_kernel<true>), K(ce_sumexp_kernel<false>),
                             K(ce_bwd_kernel<true>), K(ce_bwd_kernel<false>),
                             K((bias_dropout_add_kernel<ElementMask, true>)), K((bias_dropout_add_kernel<ElementMask, false>)),
                             K((bias_dropout_add_kernel<SampleMask, true>)), K((bias_dropout_add_kernel<SampleMask, false>)),
                             K(dropout_bwd_kernel<ElementMask>), K(dropout_bwd_kernel<SampleMask>),
                             K((bias_dropout_add_kernel<IdMask, true>)), K((bias_dropout_add_kernel<IdMask, false>)),
                             K(dropout_bwd_kernel<IdMask>), K(vit_patchify_kernel<true>),
                             K(vit_patchify_kernel<false>), K(vit_embed_fwd_kernel<true>), K(vit_embed_fwd_kernel<false>),
                             K(vit_embed_bwd_kernel<true>), K(vit_embed_bwd_kernel<false>),
                             K(swin_window_qkv_fwd_kernel), K(swin_window_qkv_bwd_kernel),
                             K(swin_window_merge_kernel<true>), K(swin_window_merge_kernel<false>), K(swin_merge_ln_fwd_kernel<true>),
                             K(swin_merge_ln_fwd_kernel<false>), K((swin_merge_ln_bwd_kernel<1, true>)),
                             K((swin_merge_ln_bwd_kernel<1, false>)), K((swin_merge_ln_bwd_kernel<2, true>)),
                             K((swin_merge_ln_bwd_kernel<2, false>)), K((swin_merge_ln_bwd_kernel<kMergeVpt, true>)),
                             K((swin_merge_ln_bwd_kernel<kMergeVpt, false>)), K(swin_mean_pool_kernel<true>),
                             K(swin_mean_pool_kernel<false>), K(cross_attn_qkv_fwd_kernel), K(cross_attn_qkv_bwd_kernel),
                             K(swin_rel_bias_fwd_kernel<float>), K(swin_rel_bias_fwd_kernel<__nv_bfloat16>), K(swin_rel_bias_bwd_kernel)};
#undef K
    for (const void* k : kernels) {
        cudaFuncAttributes attr;
        BG_CUDA(cudaFuncGetAttributes(&attr, k));
    }
    return BG_OK;
}

// channelnorm.cu -- per-pixel L2 norm over channels, forward and backward (HBM-streaming).
//
// Replaces kernel_channelnorm_update_output / kernel_channelnorm_backward_input1
// (reference channelnorm_package/channelnorm_kernel.cu:18-60, :63-96).
//
// Design: pure streaming, 0.2-0.5 FLOP/B -> HBM-bound.  One thread owns 4 consecutive pixels:
// C independent 128-bit read-once loads (L1 no-allocate) are issued back to back before any use,
// so each SM keeps >= 2048 thr x C x 16 B in flight (enough for ~6.6 TB/s at ~600 ns latency),
// then one 128-bit store.  No shared memory, no pre-zeroed outputs (the reference zero-fills
// them first, channelnorm.py:11,23: 2x the write traffic).
#include "common.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace fn2 {

template <int CT>  // CT > 0: compile-time channel count; CT == 0: runtime loop
__global__ void __launch_bounds__(256)
channelnorm_fwd_v4(const float *__restrict__ in, float *__restrict__ out, int C, int hw4, long n4) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n4) return;
    int b = (int)(idx / hw4);
    int p = (int)(idx - (long)b * hw4);
    const int Cn = CT > 0 ? CT : C;
    const float *src = in + ((long)b * Cn * hw4 + p) * 4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (CT > 0) {
        float4 v[CT > 0 ? CT : 1];
#pragma unroll
        for (int c = 0; c < CT; ++c) v[c] = ldg_stream4(src + (long)c * hw4 * 4);
#pragma unroll
        for (int c = 0; c < CT; ++c) {  // channel order = the reference's accumulation order
            acc.x += v[c].x * v[c].x; acc.y += v[c].y * v[c].y;
            acc.z += v[c].z * v[c].z; acc.w += v[c].w * v[c].w;
        }
    } else {
        for (int c = 0; c < Cn; ++c) {
            float4 v = ldg_stream4(src + (long)c * hw4 * 4);
            acc.x += v.x * v.x; acc.y += v.y * v.y; acc.z += v.z * v.z; acc.w += v.w * v.w;
        }
    }
    float4 r = make_float4(sqrtf(acc.x), sqrtf(acc.y), sqrtf(acc.z), sqrtf(acc.w));
    stg_stream4(out + idx * 4, r);
}

__global__ void __launch_bounds__(256)
channelnorm_fwd_scalar(const float *__restrict__ in, float *__restrict__ out, int C, int hw, long n) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    int b = (int)(idx / hw);
    int p = (int)(idx - (long)b * hw);
    const float *src = in + (long)b * C * hw + p;
    float acc = 0.f;
    for (int c = 0; c < C; ++c) {
        float v = __ldg(src + (long)c * hw);
        acc += v * v;
    }
    out[idx] = sqrtf(acc);
}

// gI = gO * in / (out + 1e-9).  The reference's divide is promoted to double by the 1e-9 literal
// (channelnorm_kernel.cu:92-94); fp32 here differs by <= 1 ulp-level relative error (~1e-7),
// far inside the 1e-4 contract, and out == 0 still yields gO*0/1e-9 = 0.
__device__ __forceinline__ float cn_bwd(float g, float x, float o) { return g * x / (o + 1e-9f); }

template <int CT>
__global__ void __launch_bounds__(256)
channelnorm_bwd_v4(const float *__restrict__ in, const float *__restrict__ out,
                   const float *__restrict__ gout, float *__restrict__ gin, int C, int hw4, long n4) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n4) return;
    int b = (int)(idx / hw4);
    int p = (int)(idx - (long)b * hw4);
    const int Cn = CT > 0 ? CT : C;
    const long base = ((long)b * Cn * hw4 + p) * 4;
    float4 o = ldg_stream4(out + idx * 4);
    float4 g = ldg_stream4(gout + idx * 4);
    if (CT > 0) {
        float4 v[CT > 0 ? CT : 1];
#pragma unroll
        for (int c = 0; c < CT; ++c) v[c] = ldg_stream4(in + base + (long)c * hw4 * 4);
#pragma unroll
        for (int c = 0; c < CT; ++c) {
            float4 r = make_float4(cn_bwd(g.x, v[c].x, o.x), cn_bwd(g.y, v[c].y, o.y),
                                   cn_bwd(g.z, v[c].z, o.z), cn_bwd(g.w, v[c].w, o.w));
            stg_stream4(gin + base + (long)c * hw4 * 4, r);
        }
    } else {
        for (int c = 0; c < Cn; ++c) {
            float4 v = ldg_stream4(in + base + (long)c * hw4 * 4);
            float4 r = make_float4(cn_bwd(g.x, v.x, o.x), cn_bwd(g.y, v.y, o.y),
                                   cn_bwd(g.z, v.z, o.z), cn_bwd(g.w, v.w, o.w));
            stg_stream4(gin + base + (long)c * hw4 * 4, r);
        }
    }
}

__global__ void __launch_bounds__(256)
channelnorm_bwd_scalar(const float *__restrict__ in, const float *__restrict__ out,
                       const float *__restrict__ gout, float *__restrict__ gin, int C, int hw, long n) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    int b = (int)(idx / hw);
    int p = (int)(idx - (long)b * hw);
    float o = __ldg(out + idx), g = __ldg(gout + idx);
    for (int c = 0; c < C; ++c) {
        long i = ((long)b * C + c) * hw + p;
        gin[i] = cn_bwd(g, __ldg(in + i), o);
    }
}

// ---- 16-bit storage variants (the reference dispatches K8/K9 on half too, channelnorm_kernel.cu:111,152:
// ChannelNorm is the one custom layer that sees fp16 tensors in --fp16 mode, models.py:39).  Same
// arithmetic as the reference: `val * val` is a product of two scalar_t, i.e. ROUNDED to the storage type before
// it is widened and accumulated in fp32 (channelnorm_kernel.cu:55-56); the backward divides in fp32 and rounds once.
template <typename T> __device__ __forceinline__ float h2f(T v);
template <> __device__ __forceinline__ float h2f<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float h2f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T f2h(float v);
template <> __device__ __forceinline__ __half f2h<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 f2h<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// one thread = 8 consecutive pixels (one 128-bit load per channel)
template <typename T>
__global__ void __launch_bounds__(256)
channelnorm_fwd_h8(const T *__restrict__ in, T *__restrict__ out, int C, int hw8, long n8) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n8) return;
    int b = (int)(idx / hw8);
    int p = (int)(idx - (long)b * hw8);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int c = 0; c < C; ++c) {
        uint4 raw = *reinterpret_cast<const uint4 *>(in + (((long)b * C + c) * hw8 + p) * 8);
        const T *v = reinterpret_cast<const T *>(&raw);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float x = h2f<T>(v[i]);
            acc[i] += h2f<T>(f2h<T>(x * x));
        }
    }
    uint4 o;
    T *ov = reinterpret_cast<T *>(&o);
#pragma unroll
    for (int i = 0; i < 8; ++i) ov[i] = f2h<T>(sqrtf(acc[i]));
    *reinterpret_cast<uint4 *>(out + idx * 8) = o;
}
template <typename T>
__global__ void __launch_bounds__(256)
channelnorm_fwd_h1(const T *__restrict__ in, T *__restrict__ out, int C, int hw, long n) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    int b = (int)(idx / hw);
    int p = (int)(idx - (long)b * hw);
    float acc = 0.f;
    for (int c = 0; c < C; ++c) {
        float x = h2f<T>(in[((long)b * C + c) * hw + p]);
        acc += h2f<T>(f2h<T>(x * x));
    }
    out[idx] = f2h<T>(sqrtf(acc));
}
template <typename T>
__global__ void __launch_bounds__(256)
channelnorm_bwd_h1(const T *__restrict__ in, const T *__restrict__ out, const T *__restrict__ gout,
                   T *__restrict__ gin, int C, int hw, long n) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    int b = (int)(idx / hw);
    int p = (int)(idx - (long)b * hw);
    float o = h2f<T>(out[idx]), g = h2f<T>(gout[idx]);
    for (int c = 0; c < C; ++c) {
        long i = ((long)b * C + c) * hw + p;
        gin[i] = f2h<T>(cn_bwd(g, h2f<T>(in[i]), o));
    }
}

// one thread = 8 consecutive pixels: norm and gradOutput once (128-bit loads), then one 128-bit load + store per channel
template <typename T>
__global__ void __launch_bounds__(256)
channelnorm_bwd_h8(const T *__restrict__ in, const T *__restrict__ out, const T *__restrict__ gout,
                   T *__restrict__ gin, int C, int hw8, long n8) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n8) return;
    int b = (int)(idx / hw8);
    int p = (int)(idx - (long)b * hw8);
    const uint4 oraw = *reinterpret_cast<const uint4 *>(out + idx * 8);
    const uint4 graw = *reinterpret_cast<const uint4 *>(gout + idx * 8);
    const T *ov = reinterpret_cast<const T *>(&oraw), *gv = reinterpret_cast<const T *>(&graw);
    float o[8], g[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        o[i] = h2f<T>(ov[i]);
        g[i] = h2f<T>(gv[i]);
    }
    for (int c = 0; c < C; ++c) {
        const long off = (((long)b * C + c) * hw8 + p) * 8;
        const uint4 raw = *reinterpret_cast<const uint4 *>(in + off);
        const T *v = reinterpret_cast<const T *>(&raw);
        uint4 res;
        T *rv = reinterpret_cast<T *>(&res);
#pragma unroll
        for (int i = 0; i < 8; ++i) rv[i] = f2h<T>(cn_bwd(g[i], h2f<T>(v[i]), o[i]));
        *reinterpret_cast<uint4 *>(gin + off) = res;
    }
}

template <typename T>
static int channelnorm_forward_16(const void *in, void *out, int B, int C, int H, int W, cudaStream_t st) {
    const int hw = H * W, Tn = 256;
    if (hw % 8 == 0 && ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0) {
        long n8 = (long)B * (hw / 8);
        channelnorm_fwd_h8<T><<<(unsigned)((n8 + Tn - 1) / Tn), Tn, 0, st>>>((const T *)in, (T *)out, C, hw / 8, n8);
    } else {
        long n = (long)B * hw;
        channelnorm_fwd_h1<T><<<(unsigned)((n + Tn - 1) / Tn), Tn, 0, st>>>((const T *)in, (T *)out, C, hw, n);
    }
    count_launch();
    return check_launch("channelnorm_forward(16-bit)");
}
template <typename T>
static int channelnorm_backward_16(const void *in, const void *out, const void *gout, void *gin, int B, int C,
                                   int H, int W, cudaStream_t st) {
    const int hw = H * W, Tn = 256;
    const uintptr_t al = reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out) |
                         reinterpret_cast<uintptr_t>(gout) | reinterpret_cast<uintptr_t>(gin);
    if (hw % 8 == 0 && (al & 15) == 0) {
        long n8 = (long)B * (hw / 8);
        channelnorm_bwd_h8<T><<<(unsigned)((n8 + Tn - 1) / Tn), Tn, 0, st>>>((const T *)in, (const T *)out, (const T *)gout,
                                                                             (T *)gin, C, hw / 8, n8);
    } else {
        long n = (long)B * hw;
        channelnorm_bwd_h1<T><<<(unsigned)((n + Tn - 1) / Tn), Tn, 0, st>>>((const T *)in, (const T *)out, (const T *)gout,
                                                                            (T *)gin, C, hw, n);
    }
    count_launch();
    return check_launch("channelnorm_backward(16-bit)");
}
// dtype: 1 = fp16, 2 = bf16
int channelnorm_forward_half(const void *in, void *out, int B, int C, int H, int W, int dtype, cudaStream_t st) {
    return dtype == 1 ? channelnorm_forward_16<__half>(in, out, B, C, H, W, st)
                      : channelnorm_forward_16<__nv_bfloat16>(in, out, B, C, H, W, st);
}
int channelnorm_backward_half(const void *in, const void *out, const void *gout, void *gin, int B, int C, int H,
                              int W, int dtype, cudaStream_t st) {
    return dtype == 1 ? channelnorm_backward_16<__half>(in, out, gout, gin, B, C, H, W, st)
                      : channelnorm_backward_16<__nv_bfloat16>(in, out, gout, gin, B, C, H, W, st);
}

static inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int channelnorm_forward(const float *in, float *out, int B, int C, int H, int W, cudaStream_t st) {
    const int hw = H * W;
    const int T = 256;
    if (hw % 4 == 0 && aligned16(in) && aligned16(out)) {
        long n4 = (long)B * (hw / 4);
        unsigned grid = (unsigned)((n4 + T - 1) / T);
        switch (C) {
            case 1: channelnorm_fwd_v4<1><<<grid, T, 0, st>>>(in, out, C, hw / 4, n4); break;
            case 2: channelnorm_fwd_v4<2><<<grid, T, 0, st>>>(in, out, C, hw / 4, n4); break;
            case 3: channelnorm_fwd_v4<3><<<grid, T, 0, st>>>(in, out, C, hw / 4, n4); break;
            case 4: channelnorm_fwd_v4<4><<<grid, T, 0, st>>>(in, out, C, hw / 4, n4); break;
            default: channelnorm_fwd_v4<0><<<grid, T, 0, st>>>(in, out, C, hw / 4, n4); break;
        }
    } else {
        long n = (long)B * hw;
        channelnorm_fwd_scalar<<<(unsigned)((n + T - 1) / T), T, 0, st>>>(in, out, C, hw, n);
    }
    count_launch();
    return check_launch("channelnorm_forward");
}

int channelnorm_backward(const float *in, const float *out, const float *gout, float *gin, int B,
                         int C, int H, int W, cudaStream_t st) {
    const int hw = H * W;
    const int T = 256;
    if (hw % 4 == 0 && aligned16(in) && aligned16(out) && aligned16(gout) && aligned16(gin)) {
        long n4 = (long)B * (hw / 4);
        unsigned grid = (unsigned)((n4 + T - 1) / T);
        switch (C) {
            case 1: channelnorm_bwd_v4<1><<<grid, T, 0, st>>>(in, out, gout, gin, C, hw / 4, n4); break;
            case 2: channelnorm_bwd_v4<2><<<grid, T, 0, st>>>(in, out, gout, gin, C, hw / 4, n4); break;
            case 3: channelnorm_bwd_v4<3><<<grid, T, 0, st>>>(in, out, gout, gin, C, hw / 4, n4); break;
            case 4: channelnorm_bwd_v4<4><<<grid, T, 0, st>>>(in, out, gout, gin, C, hw / 4, n4); break;
            default: channelnorm_bwd_v4<0><<<grid, T, 0, st>>>(in, out, gout, gin, C, hw / 4, n4); break;
        }
    } else {
        long n = (long)B * hw;
        channelnorm_bwd_scalar<<<(unsigned)((n + T - 1) / T), T, 0, st>>>(in, out, gout, gin, C, hw, n);
    }
    count_launch();
    return check_launch("channelnorm_backward");
}

}  // namespace fn2

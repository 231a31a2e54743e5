// common.cuh -- shared host/device helpers for libfn2b200 (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/fn2b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ < 900)
#error "libfn2b200 is written for sm_90a (H100) only"
#endif

namespace fn2 {

// ---- error plumbing (thread-local, no global mutable state) -------------------------------
void set_error(const char *fmt, ...);
int fail(int code, const char *fmt, ...);
void count_launch(int n = 1);
uint64_t launches_so_far();
const char *last_error_text();
int check_launch(const char *what);
int bind_device_of(const void *ptr);  // make the device owning ptr current on this thread  // cudaGetLastError -> return code (+ message)

// ---- TMA descriptor creation (driver entry point resolved through the runtime; no -lcuda) --
// Encodes a tiled tensor map over an fp32 tensor of `rank` dims (dims[0] fastest).
// strides_bytes[i] is the byte stride of dim i+1 (rank-1 entries).  Returns 0 / error code.
int make_tensor_map_f32(CUtensorMap *map, const void *base, int rank, const uint64_t *dims,
                        const uint64_t *strides_bytes, const uint32_t *box);

// ---- device-side PTX wrappers ---------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// 3D / 4D tiled TMA loads global -> shared, completion on an mbarrier (transaction bytes).
__device__ __forceinline__ void tma_load_3d(void *dst, const CUtensorMap *map, uint64_t *bar,
                                            int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void *dst, const CUtensorMap *map, uint64_t *bar,
                                            int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "r"(c3)
        : "memory");
}
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap *map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// streaming (read-once) 128-bit / 32-bit global loads that do not allocate in L1
__device__ __forceinline__ float4 ldg_stream4(const float *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ float ldg_stream1(const float *p) {
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}
// write-once streaming stores (evict-first in L2 is left to hardware; bypass L1 allocation)
__device__ __forceinline__ void stg_stream4(float *p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x),
                 "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ void red_add_f32(float *p, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ void red_add_v2(float *p, float a, float b) {      // p 8-byte aligned
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void red_add_v4(float *p, float a, float b, float c, float d) {      // p 16-byte aligned
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
#endif  // __CUDACC__

// ---- kernel launchers (one per .cu) -----------------------------------------------------------
int channelnorm_forward(const float *in, float *out, int B, int C, int H, int W, cudaStream_t st);
int channelnorm_backward(const float *in, const float *out, const float *gout, float *gin, int B,
                         int C, int H, int W, cudaStream_t st);
int channelnorm_forward_half(const void *in, void *out, int B, int C, int H, int W, int dtype, cudaStream_t st);
int channelnorm_backward_half(const void *in, const void *out, const void *gout, void *gin, int B, int C, int H,
                              int W, int dtype, cudaStream_t st);

// Where a kernel gets its flow from.  mode 0: a full-resolution [B,2,H,W] tensor.  mode 1 / 2: a quarter-resolution
// [B,2,fh,fw] tensor (H = 4 fh, W = 4 fw) that is multiplied by `mul` and upsampled x4 on the fly --
// bilinear with align_corners = False (nn.Upsample(scale_factor=4, mode='bilinear'), models.py:42,56: source index
// 0.25 (i + 0.5) - 0.5 clamped at 0, second tap i0 + (i0 < n - 1)) or nearest (i >> 2; models.py:72-73) -- the
// composition models.py:130,142,154,167 spells out as `upsample(flow2 * div_flow)`.
struct FlowSrc {
    const float *p;
    int fh, fw;
    int mode;
    float mul;
};


// Where the tile forward kernel writes (resample2d_tile.cu).  `cat` is a [B, cat_channels, H, W] fp32 tensor; each
// ch_* is the first channel of that product inside it, or -1 to skip the product:
//   ch_x       n_x channels copied from x (img0's C channels, then img1's)        models.py:138 `x`
//   ch_warped  C channels  img1 warped by the flow                               models.py:133
//   ch_flow    2 channels  flow / flow_div                                       models.py:138 `flow / div_flow`
//   ch_fnorm   1 channel   sqrt(dx^2 + dy^2) of the (upsampled) flow             models.py:155,166
//   ch_dnorm   1 channel   sqrt(sum_c (img0 - warped)^2)                         models.py:134-135
// Plain Resample2d forward = {cat = output, cat_channels = C, ch_warped = 0, everything else -1}.
struct WarpOut {
    float *cat;
    int cat_channels;
    int ch_x, n_x, ch_warped, ch_flow, ch_fnorm, ch_dnorm;
    float flow_div;
};
// 2-D tile kernels (resample2d_tile.cu): any strides, any C.  The backward scatters the image gradient with vector
// reductions into the pixel-interleaved scratch (zero-filled inside the call, transposed afterwards) when C <= 3 and
// `workspace` is 16-byte aligned and holds resample2d_backward_workspace_bytes(); otherwise with planar scalar
// reductions into gimg.  zero_gimg == 0: the gradient is added to what gimg holds.
int resample2d_forward_tile(const float *img1, const int64_t *is1, const float *img0, const int64_t *is0,
                            const FlowSrc &fs, const WarpOut &o, int B, int C, int H, int W, int bilinear, cudaStream_t st);
int resample2d_backward_tile(const float *img, const int64_t *istride, const float *flow, const float *gout, float *gimg,
                             float *gflow, void *workspace, size_t workspace_bytes, int zero_gimg, int B, int C, int iH,
                             int iW, int H, int W, cudaStream_t st);
size_t resample2d_backward_workspace_bytes(int B, int iH, int iW);
int resample2d_backward_finish(const float *T, float *gimg, int accumulate, int B, int C, int iH, int iW, cudaStream_t st,
                               long gimg_bstride = 0);
// backward of the fused upsample -> warp -> diff -> channel-norm -> concat forward (C <= 3).  gx == NULL: no image
// gradient (no scatter); gflow == NULL: no flow gradient.  gflow is [B,2,fs.fh,fs.fw].  workspace: the scatter scratch
// above when gx is wanted, followed by the bilinear adjoint's per-tile partials (fs.mode == 1):
// warp_concat_backward_workspace_bytes() in all.
size_t warp_concat_backward_workspace_bytes(int B, int H, int W, int upsample_mode, bool need_x);
int warp_concat_backward_tile(const float *x, const int64_t *xstride, const FlowSrc &fs, const float *gcat, const WarpOut &o,
                              float *gx, float *gflow, void *workspace, int B, int C, int H, int W, cudaStream_t st);

struct CorrParams {
    int B, C, H, W;        // inputs [B,C,H,W]
    int pad, k, md, s1, s2;
    int kr, dr, ds, D;     // kernel radius, displacement radius / size / count
    int oH, oW;            // output spatial dims
    // forward output placement / epilogue (SURVEY 8f-2, FlowNetC.py:86-92): sample n's D planes start at
    // out + n * out_bstride (elements; D*oH*oW = a dense [B,D,oH,oW] tensor, larger = a channel range of a wider
    // concat buffer), and v < 0 is multiplied by `leaky` (1 = no activation, 0.1 = nn.LeakyReLU(0.1)).
    long out_bstride;
    float leaky;
    // backward input placement / activation (fn2b200_correlation_backward_cat): sample n's D gradOutput planes start at
    // gout + n * g_bstride (D*oH*oW = dense; larger = a channel range of a concat gradient).  act != NULL: the forward's
    // activated output, same layout as gout; every gradOutput value g becomes (act > 0 ? g : g * leaky) before use.
    long g_bstride;
    const float *act;
};
int corr_forward_generic(const float *in1, const float *in2, float *out, const CorrParams &p,
                         cudaStream_t st);
int corr_backward_generic(const float *in1, const float *in2, const float *gout, float *gin1,
                          float *gin2, const CorrParams &p, cudaStream_t st);
// TMA-tiled FMA kernels: kernel_size == 1, stride1 == 1, (s2, dr) in the instantiated set, W % 4 == 0; the caller also
// guarantees 16-byte aligned operands (capi.cu's corr_family chooses the family).
bool corr_tiled_supported(const CorrParams &p);
int corr_forward_tiled(const float *in1, const float *in2, float *out, const CorrParams &p,
                       cudaStream_t st);
int corr_backward_tiled(const float *in1, const float *in2, const float *gout, float *gin1,
                        float *gin2, const CorrParams &p, cudaStream_t st);

// Tensor-core (wgmma) forward and backward for FlowNetC's configuration; needs a caller-provided workspace.
bool corr_tc_supported(const CorrParams &p);
size_t corr_tc_workspace_bytes(const CorrParams &p);
int corr_backward_tc(const float *in1, const float *in2, const float *gout, float *gin1, float *gin2,
                     const CorrParams &p, void *workspace, size_t workspace_bytes, int have_split, cudaStream_t st);
int corr_forward_tc(const float *in1, const float *in2, float *out, const CorrParams &p, void *workspace,
                    size_t workspace_bytes, cudaStream_t st);

}  // namespace fn2

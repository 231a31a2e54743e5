// resample_common.cuh -- tap arithmetic and flow sources of the Resample2d kernels (resample2d_tile.cu: 2-D tile
// kernels, optionally fused with the flow upsample and the concat epilogue).
#pragma once
#include "common.cuh"

namespace fn2 {

struct Taps {
    int xL, xR, yT, yB;
};

__device__ __forceinline__ Taps clamp_taps(float fx, float fy, int W, int H) {
    // fx = floor(xf), fy = floor(yf).  int(floor(xf)+1): the +1 is done in float like the
    // reference (resample2d_kernel.cu:49-52); cvt.rzi saturates for huge |xf|.
    Taps t;
    t.xL = max(min((int)fx, W - 1), 0);
    t.xR = max(min((int)(fx + 1.0f), W - 1), 0);
    t.yT = max(min((int)fy, H - 1), 0);
    t.yB = max(min((int)(fy + 1.0f), H - 1), 0);
    return t;
}

__device__ __forceinline__ float2 load_flow(const FlowSrc &f, int b, int y, int x, int H, int W) {
    if (f.mode == 0) {
        const float *q = f.p + ((long)b * 2 * H + y) * W + x;
        return make_float2(ldg_stream1(q), ldg_stream1(q + (long)H * W));
    }
    const long plane = (long)f.fh * f.fw;
    const float *q = f.p + (long)b * 2 * plane;
    if (f.mode == 2) {
        const long o = (long)(y >> 2) * f.fw + (x >> 2);
        return make_float2(__ldg(q + o) * f.mul, __ldg(q + plane + o) * f.mul);
    }
    float hs = fmaxf(0.25f * ((float)y + 0.5f) - 0.5f, 0.f), ws = fmaxf(0.25f * ((float)x + 0.5f) - 0.5f, 0.f);
    int h1 = (int)hs, w1 = (int)ws;
    int hp = h1 < f.fh - 1 ? f.fw : 0, wp = w1 < f.fw - 1 ? 1 : 0;
    float l1h = hs - (float)h1, l0h = 1.f - l1h, l1w = ws - (float)w1, l0w = 1.f - l1w;
    const float *r = q + (long)h1 * f.fw + w1;
    float2 out;
    // torch's upsample_bilinear2d: h0 * (w0 * v00 + w1 * v01) + h1 * (w0 * v10 + w1 * v11).  Explicit mul / fma (the
    // contraction the compiler chose for the plain expression) so that every kernel variant computes the same flow
    // bits: a 1-ulp change of the flow can move a tap's floor.
    const auto lerp = [&](const float *p) {
        const float row0 = __fmaf_rn(l0w, __fmul_rn(__ldg(p), f.mul), __fmul_rn(l1w, __fmul_rn(__ldg(p + wp), f.mul)));
        const float row1 = __fmaf_rn(l0w, __fmul_rn(__ldg(p + hp), f.mul), __fmul_rn(l1w, __fmul_rn(__ldg(p + hp + wp), f.mul)));
        return __fmaf_rn(l0h, row0, __fmul_rn(l1h, row1));
    };
    out.x = lerp(r);
    out.y = lerp(r + plane);
    return out;
}

}  // namespace fn2

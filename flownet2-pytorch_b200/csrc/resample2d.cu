// resample2d.cu -- backward bilinear (or nearest) warp of an image by a flow field, fwd + bwd.
//
// Replaces kernel_resample2d_update_output / _backward_input1 / _backward_input2
// (reference resample2d_package/resample2d_kernel.cu:15-72, :75-125, :127-198).
//
// Design (HBM/L2-bound gather): ONE thread per output PIXEL (the reference uses one per
// pixel x channel and re-reads the flow and recomputes taps per channel): the two flow values are
// read once, tap indices / weights computed once, then the C channels are gathered with 4*C
// independent loads in flight.  The image is addressed through explicit element strides so the
// non-contiguous channel slice FlowNet2 passes (models.py:133) needs no .contiguous() copy
// (resample2d.py:48 copies 44 MB per call).  The gathers hit L2 (a 448x1024x3x8 image is 44 MB
// << 126 MB).  Outputs are written once, without the reference's zero-fill pass.
// Backward: a single fused kernel computes both flow-gradient channels per thread (the reference
// runs 2 threads that each redo the 4*C gathers) and scatters the image gradient with
// red.global.add.f32 (no return value -> no round trip).
//
// Round 2: these row kernels (one CTA = 256 consecutive pixels of one row) are kept as the comparison point
// (FN2B200_RESAMPLE=row); the shipped kernels are the 2-D tile kernels of resample2d_tile.cu.
#include "resample_common.cuh"

namespace fn2 {

template <int CT>
__global__ void __launch_bounds__(256)
resample2d_fwd(const float *__restrict__ img, long sb, long sc, long sh, long sw,
               const float *__restrict__ flow, float *__restrict__ out, int C, int H, int W,
               long npix, int bilinear) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= npix) return;
    const int hw = H * W;
    int b = (int)(idx / hw);
    int p = (int)(idx - (long)b * hw);
    int y = p / W, x = p - y * W;
    const float *fl = flow + (long)b * 2 * hw + p;
    float dx = ldg_stream1(fl), dy = ldg_stream1(fl + hw);
    float xf = (float)x + dx, yf = (float)y + dy;
    const int Cn = CT > 0 ? CT : C;
    const float *ib = img + (long)b * sb;
    float *ob = out + (long)b * Cn * hw + p;
    if (bilinear) {
        float fx = floorf(xf), fy = floorf(yf);
        float a = xf - fx, be = yf - fy;
        Taps t = clamp_taps(fx, fy, W, H);  // clamps use the OUTPUT dims (:28-31)
        float w00 = (1.f - a) * (1.f - be), w01 = a * (1.f - be);
        float w10 = (1.f - a) * be, w11 = a * be;
        long oTL = t.yT * sh + t.xL * sw, oTR = t.yT * sh + t.xR * sw;
        long oBL = t.yB * sh + t.xL * sw, oBR = t.yB * sh + t.xR * sw;
#pragma unroll
        for (int c = 0; c < (CT > 0 ? CT : 1); ++c) {
            if (CT > 0) {
                const float *ic = ib + c * sc;
                float v = __fmul_rn(w00, __ldg(ic + oTL));  // same term order as the reference (:56-59)
                v = __fmaf_rn(w01, __ldg(ic + oTR), v);
                v = __fmaf_rn(w10, __ldg(ic + oBL), v);
                v = __fmaf_rn(w11, __ldg(ic + oBR), v);
                __stcs(ob + (long)c * hw, v);
            }
        }
        if (CT == 0) {
            for (int c = 0; c < Cn; ++c) {
                const float *ic = ib + c * sc;
                float v = __fmul_rn(w00, __ldg(ic + oTL));
                v = __fmaf_rn(w01, __ldg(ic + oTR), v);
                v = __fmaf_rn(w10, __ldg(ic + oBL), v);
                v = __fmaf_rn(w11, __ldg(ic + oBR), v);
                __stcs(ob + (long)c * hw, v);
            }
        }
    } else {
        // floor(xf + 0.5) is evaluated in double by the reference (0.5 literal, :66-67)
        int xN = max(min((int)floor((double)xf + 0.5), W - 1), 0);
        int yN = max(min((int)floor((double)yf + 0.5), H - 1), 0);
        long o = yN * sh + xN * sw;
        for (int c = 0; c < Cn; ++c) __stcs(ob + (long)c * hw, __ldg(ib + c * sc + o));
    }
}

template <int CT>
__global__ void __launch_bounds__(256)
resample2d_bwd(const float *__restrict__ img, long sb, long sc, long sh, long sw,
               const float *__restrict__ flow, const float *__restrict__ gout,
               float *__restrict__ gimg, float *__restrict__ gflow, int C, int iH, int iW, int H,
               int W, long npix) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= npix) return;
    const int hw = H * W;
    int b = (int)(idx / hw);
    int p = (int)(idx - (long)b * hw);
    int y = p / W, x = p - y * W;
    const float *fl = flow + (long)b * 2 * hw + p;
    float dx = ldg_stream1(fl), dy = ldg_stream1(fl + hw);
    float xf = (float)x + dx, yf = (float)y + dy;
    float fx = floorf(xf), fy = floorf(yf);
    const int Cn = CT > 0 ? CT : C;

    // K7 (flow gradient): taps clamped with the FLOW dims, floor-based fractions (:145-166)
    Taps tf = clamp_taps(fx, fy, W, H);
    float a = xf - fx, be = yf - fy;
    long oTL = tf.yT * sh + tf.xL * sw, oTR = tf.yT * sh + tf.xR * sw;
    long oBL = tf.yB * sh + tf.xL * sw, oBR = tf.yB * sh + tf.xR * sw;
    // K6 (image gradient): taps clamped with the IMAGE dims, int()-truncation fractions (:105-114)
    Taps ti = clamp_taps(fx, fy, iW, iH);
    float at = xf - (float)(int)xf, bt = yf - (float)(int)yf;
    float s00 = (1.f - at) * (1.f - bt), s01 = at * (1.f - bt);
    float s10 = (1.f - at) * bt, s11 = at * bt;
    const long ihw = (long)iH * iW;
    long gTL = (long)ti.yT * iW + ti.xL, gTR = (long)ti.yT * iW + ti.xR;
    long gBL = (long)ti.yB * iW + ti.xL, gBR = (long)ti.yB * iW + ti.xR;

    const float *ib = img + (long)b * sb;
    const float *gb = gout + (long)b * Cn * hw + p;
    float *gi = gimg ? gimg + (long)b * Cn * ihw : nullptr;
    float gx = 0.f, gy = 0.f;
#pragma unroll
    for (int c0 = 0; c0 < (CT > 0 ? CT : 1); ++c0) {
        const int cend = CT > 0 ? c0 + 1 : Cn;
        for (int c = c0; c < cend; ++c) {
            float g = ldg_stream1(gb + (long)c * hw);
            if (gflow) {
                const float *ic = ib + c * sc;
                float iTL = __ldg(ic + oTL), iTR = __ldg(ic + oTR);
                float iBL = __ldg(ic + oBL), iBR = __ldg(ic + oBR);
                // d/dxf: gamma = 1 - beta (:181-192); d/dyf: gamma = 1 - alpha (:168-179)
                gx += g * ((1.f - be) * (iTR - iTL) + be * (iBR - iBL));
                gy += g * ((1.f - a) * (iBL - iTL) + a * (iBR - iTR));
            }
            if (gi) {
                float *gc = gi + (long)c * ihw;
                red_add_f32(gc + gTL, s00 * g);
                red_add_f32(gc + gTR, s01 * g);
                red_add_f32(gc + gBL, s10 * g);
                red_add_f32(gc + gBR, s11 * g);
            }
        }
    }
    if (gflow) {
        float *gf = gflow + (long)b * 2 * hw + p;
        __stcs(gf, gx);
        __stcs(gf + hw, gy);
    }
}

int resample2d_forward(const float *img, const int64_t *is, const float *flow, float *out, int B,
                       int C, int iH, int iW, int H, int W, int bilinear, cudaStream_t st) {
    (void)iH; (void)iW;
    long npix = (long)B * H * W;
    const int T = 256;
    unsigned grid = (unsigned)((npix + T - 1) / T);
    long sb = is[0], sc = is[1], sh = is[2], sw = is[3];
    switch (C) {
        case 1: resample2d_fwd<1><<<grid, T, 0, st>>>(img, sb, sc, sh, sw, flow, out, C, H, W, npix, bilinear); break;
        case 2: resample2d_fwd<2><<<grid, T, 0, st>>>(img, sb, sc, sh, sw, flow, out, C, H, W, npix, bilinear); break;
        case 3: resample2d_fwd<3><<<grid, T, 0, st>>>(img, sb, sc, sh, sw, flow, out, C, H, W, npix, bilinear); break;
        default: resample2d_fwd<0><<<grid, T, 0, st>>>(img, sb, sc, sh, sw, flow, out, C, H, W, npix, bilinear); break;
    }
    count_launch();
    return check_launch("resample2d_forward");
}

int resample2d_backward(const float *img, const int64_t *is, const float *flow, const float *gout,
                        float *gimg, float *gflow, int B, int C, int iH, int iW, int H, int W,
                        cudaStream_t st) {
    long npix = (long)B * H * W;
    const int T = 256;
    unsigned grid = (unsigned)((npix + T - 1) / T);
    long sb = is[0], sc = is[1], sh = is[2], sw = is[3];
    switch (C) {
        case 1: resample2d_bwd<1><<<grid, T, 0, st>>>(img, sb, sc, sh, sw, flow, gout, gimg, gflow, C, iH, iW, H, W, npix); break;
        case 2: resample2d_bwd<2><<<grid, T, 0, st>>>(img, sb, sc, sh, sw, flow, gout, gimg, gflow, C, iH, iW, H, W, npix); break;
        case 3: resample2d_bwd<3><<<grid, T, 0, st>>>(img, sb, sc, sh, sw, flow, gout, gimg, gflow, C, iH, iW, H, W, npix); break;
        default: resample2d_bwd<0><<<grid, T, 0, st>>>(img, sb, sc, sh, sw, flow, gout, gimg, gflow, C, iH, iW, H, W, npix); break;
    }
    count_launch();
    return check_launch("resample2d_backward");
}

}  // namespace fn2

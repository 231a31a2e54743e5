// resample2d_tile.cu -- Resample2d forward / backward on 2-D pixel tiles with L1-cached gathers, optionally fused with the
// flow upsample in front and the diff / channel-norm / concat epilogue behind (SURVEY 8f rows 1 and 3).
//
// Replaces kernel_resample2d_update_output / _backward_input1 / _backward_input2 (reference
// resample2d_package/resample2d_kernel.cu:15-72, :75-125, :127-198) and, with the fused outputs, the chain
// models.py:130-138 builds from nn.Upsample, Resample2d, a subtraction, ChannelNorm, a division and torch.cat.
//
// Why tiles: round 1's kernels mapped a CTA to 256 consecutive pixels of ONE row.  With a sigma = 4 px flow the taps
// of such a CTA spread over ~30 image rows, every 32-byte sector fetched for one tap is used once and the kernel ran
// at the L2->SM crossbar ceiling (0.51 GB moved for 0.117 GB of algorithmic traffic, 9.3 TB/s).  A CTA that owns a
// 32 x (8 PY) pixel tile touches (32 + 2h) x (8 PY + 2h) pixels of the image instead: the sectors it pulls are reused
// by its other threads out of L1 (the CTAs co-resident on an SM are x-neighbours and share their halos too).
// What bounds it is the L1 data pipe (a warp-wide tap load touches many lines).  A TMA-staged shared-memory box per
// CTA moves the same bytes, but flow read -> box placement -> TMA -> gather serialise inside a CTA and large boxes leave
// few CTAs per SM; it was dropped, as was,
// for the backward, accumulation in a shared-memory box (below).
//
// Thread (lx = tid & 31, ly = tid >> 5) owns pixels (tx0 + lx, ty0 + ly + 8 j), j < PY: flow reads and output stores
// are 128-byte coalesced rows, the PY pixels give 4 C PY independent gathers in flight per thread.
#include "resample_common.cuh"

namespace fn2 {

struct ImgView {        // a [*, C, H, W] fp32 view with element strides
    const float *p;
    long sb, sc, sh, sw;
};

template <int CT, int PY, bool FUSED>
__global__ void __launch_bounds__(256)
resample2d_fwd_tile(ImgView im1, ImgView im0, FlowSrc fs, WarpOut o, int C, int H, int W, int tiles_x, int tiles_y,
                    int bilinear) {
    const int tid = threadIdx.x, lx = tid & 31, ly = tid >> 5;
    int t = blockIdx.x;
    const int bx = t % tiles_x;
    t /= tiles_x;
    const int by = t % tiles_y, b = t / tiles_y;
    const int x = bx * 32 + lx, y0 = by * (8 * PY) + ly;
    if (x >= W) return;
    const int Cn = CT > 0 ? CT : C;
    const long hw = (long)H * W;
    const float *ib = im1.p + (long)b * im1.sb;
    float *ob = o.cat + (long)b * o.cat_channels * hw;

    float dx[PY], dy[PY];
#pragma unroll
    for (int j = 0; j < PY; ++j) {
        const int y = y0 + 8 * j;
        dx[j] = dy[j] = 0.f;
        if (y < H) {
            const float2 f = load_flow(fs, b, y, x, H, W);
            dx[j] = f.x;
            dy[j] = f.y;
        }
    }
#pragma unroll
    for (int j = 0; j < PY; ++j) {
        const int y = y0 + 8 * j;
        if (y >= H) continue;
        const float xf = (float)x + dx[j], yf = (float)y + dy[j];
        float *op = ob + (long)y * W + x;
        if (!bilinear) {
            // floor(xf + 0.5) is evaluated in double by the reference (0.5 literal, :66-67)
            const int xN = max(min((int)floor((double)xf + 0.5), W - 1), 0);
            const int yN = max(min((int)floor((double)yf + 0.5), H - 1), 0);
            const long off = yN * im1.sh + xN * im1.sw;
            for (int c = 0; c < Cn; ++c) __stcs(op + (long)(o.ch_warped + c) * hw, __ldg(ib + c * im1.sc + off));
            continue;
        }
        const float fx = floorf(xf), fy = floorf(yf);
        const float al = xf - fx, be = yf - fy;
        const Taps tp = clamp_taps(fx, fy, W, H);          // clamps use the OUTPUT dims (:28-31)
        const float w00 = (1.f - al) * (1.f - be), w01 = al * (1.f - be);
        const float w10 = (1.f - al) * be, w11 = al * be;
        const long oTL = tp.yT * im1.sh + tp.xL * im1.sw, oTR = tp.yT * im1.sh + tp.xR * im1.sw;
        const long oBL = tp.yB * im1.sh + tp.xL * im1.sw, oBR = tp.yB * im1.sh + tp.xR * im1.sw;
        float dacc = 0.f;
#pragma unroll
        for (int c = 0; c < (CT > 0 ? CT : 1); ++c) {
            const int cend = CT > 0 ? c + 1 : Cn;
            for (int cc = c; cc < cend; ++cc) {
                const float *ic = ib + cc * im1.sc;
                // same term order as the reference (:56-59); explicit mul / fma so that every kernel variant rounds alike
                float v = __fmul_rn(w00, __ldg(ic + oTL));
                v = __fmaf_rn(w01, __ldg(ic + oTR), v);
                v = __fmaf_rn(w10, __ldg(ic + oBL), v);
                v = __fmaf_rn(w11, __ldg(ic + oBR), v);
                if (o.ch_warped >= 0) __stcs(op + (long)(o.ch_warped + cc) * hw, v);
                if (FUSED) {
                    if (o.ch_dnorm >= 0 || (o.ch_x >= 0 && cc < o.n_x)) {
                        const float a0 = __ldg(im0.p + (long)b * im0.sb + cc * im0.sc + (long)y * im0.sh + x * im0.sw);
                        const float d = a0 - v;          // ChannelNorm of (img0 - warped): channel order, then sqrt
                        dacc = __fmaf_rn(d, d, dacc);
                        if (o.ch_x >= 0 && cc < o.n_x) __stcs(op + (long)(o.ch_x + cc) * hw, a0);
                    }
                    if (o.ch_x >= 0 && Cn + cc < o.n_x)
                        __stcs(op + (long)(o.ch_x + Cn + cc) * hw, __ldg(ib + cc * im1.sc + (long)y * im1.sh + x * im1.sw));
                }
            }
        }
        if (FUSED) {
            if (o.ch_dnorm >= 0) __stcs(op + (long)o.ch_dnorm * hw, sqrtf(dacc));
            if (o.ch_flow >= 0) {
                __stcs(op + (long)o.ch_flow * hw, __fdiv_rn(dx[j], o.flow_div));
                __stcs(op + (long)(o.ch_flow + 1) * hw, __fdiv_rn(dy[j], o.flow_div));
            }
            if (o.ch_fnorm >= 0) __stcs(op + (long)o.ch_fnorm * hw, sqrtf(__fmaf_rn(dy[j], dy[j], __fmul_rn(dx[j], dx[j]))));
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Backward.  One kernel: the flow gradient (K7, needs the image taps: gathered as in the forward) and the image
// gradient (K6, a bilinear scatter of gradOutput).  What bounds the scatter (csrc_test/atomics_bench.cu): an SM retires
// global reductions at a fixed cost per LANE whatever their width, and round 1 issued 4 taps x C of them per pixel.
// SC selects how the scatter is done:
//   1  one red.global.add.f32 per tap and channel into the planar gradient (round 1; any shape)
//   2  one red.global.add.v4.f32 per tap into a pixel-interleaved scratch T[b][y][x][4] (C <= 3), transposed into the
//      planar gradient by resample2d_bwd_finish: 4 lane-operations per pixel instead of 12
// Accumulating in a shared-memory box per CTA and flushing it with coalesced vector reductions was built and measured
// too: red.shared.add.f32 compiled to a compare-and-swap loop that retries whenever neighbouring pixels hit the same
// word, which made it slower than the global reductions: dropped.
// ---------------------------------------------------------------------------------------------------------------
template <int CT, int PY, int SC>
__global__ void __launch_bounds__(256)
resample2d_bwd_tile(ImgView im, FlowSrc fs, const float *__restrict__ gout, float *__restrict__ gimg,
                    float *__restrict__ T, float *__restrict__ gflow, int C, int iH, int iW, int H, int W, int tiles_x,
                    int tiles_y) {
    const int tid = threadIdx.x, lx = tid & 31, ly = tid >> 5;
    int t = blockIdx.x;
    const int bxi = t % tiles_x;
    t /= tiles_x;
    const int byi = t % tiles_y, b = t / tiles_y;
    const int x = bxi * 32 + lx, y0 = byi * (8 * PY) + ly;
    const int Cn = CT > 0 ? CT : C;
    const long hw = (long)H * W, ihw = (long)iH * iW;
    const bool xok = x < W;

    float dx[PY], dy[PY];
#pragma unroll
    for (int j = 0; j < PY; ++j) {
        const int y = y0 + 8 * j;
        dx[j] = dy[j] = 0.f;
        if (xok && y < H) {
            const float2 f = load_flow(fs, b, y, x, H, W);
            dx[j] = f.x;
            dy[j] = f.y;
        }
    }

    const float *ib = im.p + (long)b * im.sb;
    const float *gb = gout + (long)b * Cn * hw;
    float *gi = (SC == 1 && gimg) ? gimg + (long)b * Cn * ihw : nullptr;
    float *Tb = (SC == 2 && T) ? T + (long)b * ihw * 4 : nullptr;
#pragma unroll
    for (int j = 0; j < PY; ++j) {
        const int y = y0 + 8 * j;
        if (!(xok && y < H)) continue;
        const float xf = (float)x + dx[j], yf = (float)y + dy[j];
        const float fx = floorf(xf), fy = floorf(yf);
        // K7 (flow gradient): taps clamped with the FLOW dims, floor-based fractions (:145-166)
        const Taps tf = clamp_taps(fx, fy, W, H);
        const float al = xf - fx, be = yf - fy;
        const long oTL = tf.yT * im.sh + tf.xL * im.sw, oTR = tf.yT * im.sh + tf.xR * im.sw;
        const long oBL = tf.yB * im.sh + tf.xL * im.sw, oBR = tf.yB * im.sh + tf.xR * im.sw;
        // K6 (image gradient): taps clamped with the IMAGE dims, int()-truncation fractions (:105-114)
        const Taps ti = clamp_taps(fx, fy, iW, iH);
        const float at = xf - (float)(int)xf, bt = yf - (float)(int)yf;
        const float s00 = (1.f - at) * (1.f - bt), s01 = at * (1.f - bt), s10 = (1.f - at) * bt, s11 = at * bt;
        const long gTL = (long)ti.yT * iW + ti.xL, gTR = (long)ti.yT * iW + ti.xR;
        const long gBL = (long)ti.yB * iW + ti.xL, gBR = (long)ti.yB * iW + ti.xR;
        float gx = 0.f, gy = 0.f;
        float gv[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int c = 0; c < (CT > 0 ? CT : 1); ++c) {
            const int cend = CT > 0 ? c + 1 : Cn;
            for (int cc = c; cc < cend; ++cc) {
                const float g = ldg_stream1(gb + (long)cc * hw + (long)y * W + x);
                if (gflow) {
                    const float *ic = ib + cc * im.sc;
                    const float iTL = __ldg(ic + oTL), iTR = __ldg(ic + oTR), iBL = __ldg(ic + oBL), iBR = __ldg(ic + oBR);
                    // d/dxf: gamma = 1 - beta (:181-192); d/dyf: gamma = 1 - alpha (:168-179)
                    gx += g * ((1.f - be) * (iTR - iTL) + be * (iBR - iBL));
                    gy += g * ((1.f - al) * (iBL - iTL) + al * (iBR - iTR));
                }
                if (SC == 1 && gi) {
                    float *gc = gi + (long)cc * ihw;
                    red_add_f32(gc + gTL, s00 * g); red_add_f32(gc + gTR, s01 * g);
                    red_add_f32(gc + gBL, s10 * g); red_add_f32(gc + gBR, s11 * g);
                }
                if (SC == 2 && CT > 0) gv[cc < 3 ? cc : 0] = g;
            }
        }
        if (SC == 2 && Tb) {
            float *pTL = Tb + gTL * 4, *pTR = Tb + gTR * 4, *pBL = Tb + gBL * 4, *pBR = Tb + gBR * 4;
            if (CT == 1) {
                red_add_f32(pTL, s00 * gv[0]); red_add_f32(pTR, s01 * gv[0]);
                red_add_f32(pBL, s10 * gv[0]); red_add_f32(pBR, s11 * gv[0]);
            } else if (CT == 2) {
                red_add_v2(pTL, s00 * gv[0], s00 * gv[1]); red_add_v2(pTR, s01 * gv[0], s01 * gv[1]);
                red_add_v2(pBL, s10 * gv[0], s10 * gv[1]); red_add_v2(pBR, s11 * gv[0], s11 * gv[1]);
            } else {
                red_add_v4(pTL, s00 * gv[0], s00 * gv[1], s00 * gv[2], 0.f);
                red_add_v4(pTR, s01 * gv[0], s01 * gv[1], s01 * gv[2], 0.f);
                red_add_v4(pBL, s10 * gv[0], s10 * gv[1], s10 * gv[2], 0.f);
                red_add_v4(pBR, s11 * gv[0], s11 * gv[1], s11 * gv[2], 0.f);
            }
        }
        if (gflow) {
            float *gf = gflow + (long)b * 2 * hw + (long)y * W + x;
            __stcs(gf, gx);
            __stcs(gf + hw, gy);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Backward of the fused upsample -> warp -> diff -> channel-norm -> concat forward.  Per pixel, with flow = the
// full-resolution flow (recomputed by load_flow exactly as the forward does), v = the warped img1 (recomputed from the
// taps the flow gradient needs anyway), d = img0 - v, n = |d|, f = |flow|:
//   g_d[c]   = gcat[ch_dnorm] * d[c] / (n + 1e-9)                      ChannelNorm backward, channelnorm_kernel.cu:92
//   g_v[c]   = gcat[ch_warped + c] - g_d[c]                            the subtraction (models.py:134)
//   gx[c]    = gcat[ch_x + c] + g_d[c]          (img0 half),   gx[C + c] = gcat[ch_x + C + c] + scatter of g_v (K6)
//   g_up     = K7(g_v) + gcat[ch_flow ..] / flow_div + gcat[ch_fnorm] * flow / (f + 1e-9)
// The scatter goes through the interleaved scratch T exactly as in resample2d_bwd_tile<.., 2>; the finishing kernel adds
// T to the direct term this kernel stores into gx[:, C:2C].
// UP selects where the flow comes from and where g_up goes (FlowSrc mode):
//   0  full-resolution flow: g_up is the flow gradient, stored to gflow [B,2,H,W]
//   2  nearest x4: g_up is staged in shared memory; the 32 x 8 PY tile is aligned to 4, so each 4 x 4 block of it is one
//      quarter-resolution cell, summed in a fixed order, times mul, and stored to gflow [B,2,fh,fw]
//   1  bilinear x4: a cell receives from full-resolution rows / columns [4i - 2, 4i + 5], so the cells of a tile edge
//      are shared with the neighbouring tiles.  The tile's g_up is reduced in shared memory (rows of pixels onto cell
//      columns, then pixel rows onto cell rows, with load_flow's own lambdas; fixed order) into (8 PY / 4 + 2) x 10
//      per-tile partials per component, written to gflow = the partial scratch; warp_concat_up_finish adds the <= 2 x 2
//      partials of each cell in a fixed order.  Deterministic: no atomics touch the flow gradient.
// NX / NF: the image / flow gradient is wanted (gx / gflow are not touched otherwise): without NX there is no K6
// scatter, without NF no K7 and no flow reduction.
// ---------------------------------------------------------------------------------------------------------------
// weight of full-resolution pixel p in quarter-resolution cell `cell` of load_flow's bilinear x4 upsample (n cells)
__device__ __forceinline__ float up4_weight(int p, int cell, int n) {
    const float s = fmaxf(0.25f * ((float)p + 0.5f) - 0.5f, 0.f);
    const int i1 = (int)s, ip = i1 < n - 1 ? 1 : 0;
    const float l1 = s - (float)i1;
    return (i1 == cell ? 1.f - l1 : 0.f) + (i1 + ip == cell ? l1 : 0.f);
}

template <int CT, int PY, int UP, bool NX, bool NF>
__global__ void __launch_bounds__(256)
warp_concat_bwd_tile(ImgView xv, FlowSrc fs, const float *__restrict__ gcat, WarpOut o, float *__restrict__ gx,
                     float *__restrict__ T, float *__restrict__ gflow, int H, int W, int tiles_x, int tiles_y) {
    constexpr int TH = 8 * PY, NR = TH / 4 + 2, NC = 32 / 4 + 2;          // tile rows; bilinear partial cells
    constexpr bool STAGE = UP != 0 && NF;
    __shared__ float sg[STAGE ? 2 : 1][STAGE ? TH : 1][32];                 // g_up of the tile (0 outside the image)
    __shared__ float sr[UP == 1 && NF ? 2 : 1][UP == 1 && NF ? TH : 1][NC];  // bilinear: pixel rows x cell columns
    const int tid = threadIdx.x, lx = tid & 31, ly = tid >> 5;
    int t = blockIdx.x;
    const int bxi = t % tiles_x;
    t /= tiles_x;
    const int byi = t % tiles_y, b = t / tiles_y;
    const int x = bxi * 32 + lx, y0 = byi * (8 * PY) + ly;
    if (UP == 0 && x >= W) return;
    const long hw = (long)H * W;
    const float *i0 = xv.p + (long)b * xv.sb, *i1 = i0 + CT * xv.sc;
    const float *gc = gcat + (long)b * o.cat_channels * hw;
    float *gxb = NX ? gx + (long)b * 2 * CT * hw : nullptr;
    float *Tb = NX ? T + (long)b * hw * 4 : nullptr;
    if (STAGE) {
#pragma unroll
        for (int j = 0; j < PY; ++j) sg[0][ly + 8 * j][lx] = sg[1][ly + 8 * j][lx] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < PY; ++j) {
        const int y = y0 + 8 * j;
        if (y >= H || (UP != 0 && x >= W)) continue;
        const long pix = (long)y * W + x;
        const float2 fl = load_flow(fs, b, y, x, H, W);
        const float xf = (float)x + fl.x, yf = (float)y + fl.y;
        const float fx = floorf(xf), fy = floorf(yf);
        const float al = xf - fx, be = yf - fy;
        const Taps tp = clamp_taps(fx, fy, W, H);
        const float w00 = (1.f - al) * (1.f - be), w01 = al * (1.f - be), w10 = (1.f - al) * be, w11 = al * be;
        const long oTL = tp.yT * xv.sh + tp.xL * xv.sw, oTR = tp.yT * xv.sh + tp.xR * xv.sw;
        const long oBL = tp.yB * xv.sh + tp.xL * xv.sw, oBR = tp.yB * xv.sh + tp.xR * xv.sw;
        float iTL[CT], iTR[CT], iBL[CT], iBR[CT], d[CT];
        float nacc = 0.f;
#pragma unroll
        for (int c = 0; c < CT; ++c) {
            const float *ic = i1 + c * xv.sc;
            iTL[c] = __ldg(ic + oTL); iTR[c] = __ldg(ic + oTR); iBL[c] = __ldg(ic + oBL); iBR[c] = __ldg(ic + oBR);
            float v = __fmul_rn(w00, iTL[c]);
            v = __fmaf_rn(w01, iTR[c], v);
            v = __fmaf_rn(w10, iBL[c], v);
            v = __fmaf_rn(w11, iBR[c], v);
            d[c] = __ldg(i0 + c * xv.sc + (long)y * xv.sh + x * xv.sw) - v;
            nacc = __fmaf_rn(d[c], d[c], nacc);
        }
        const float nrm = sqrtf(nacc);
        const float gn = o.ch_dnorm >= 0 ? ldg_stream1(gc + (long)o.ch_dnorm * hw + pix) : 0.f;
        float gv[3] = {0.f, 0.f, 0.f};
        float gfx = 0.f, gfy = 0.f;
#pragma unroll
        for (int c = 0; c < CT; ++c) {
            const float gd = o.ch_dnorm >= 0 ? gn * d[c] / (nrm + 1e-9f) : 0.f;
            const float gw = o.ch_warped >= 0 ? ldg_stream1(gc + (long)(o.ch_warped + c) * hw + pix) : 0.f;
            gv[c] = gw - gd;
            if (NX) {
                const float gx0 = (o.ch_x >= 0 && c < o.n_x) ? ldg_stream1(gc + (long)(o.ch_x + c) * hw + pix) : 0.f;
                const float gx1 = (o.ch_x >= 0 && CT + c < o.n_x) ? ldg_stream1(gc + (long)(o.ch_x + CT + c) * hw + pix) : 0.f;
                __stcs(gxb + (long)c * hw + pix, gx0 + gd);
                __stcs(gxb + (long)(CT + c) * hw + pix, gx1);          // + the scattered part, added by the finishing kernel
            }
            if (NF) {
                // K7: d/dxf with gamma = 1 - beta (:181-192), d/dyf with gamma = 1 - alpha (:168-179)
                gfx += gv[c] * ((1.f - be) * (iTR[c] - iTL[c]) + be * (iBR[c] - iBL[c]));
                gfy += gv[c] * ((1.f - al) * (iBL[c] - iTL[c]) + al * (iBR[c] - iTR[c]));
            }
        }
        if (NX) {
            // K6: image-gradient scatter, int()-truncation fractions (:105-114); image dims == flow dims here
            const float at = xf - (float)(int)xf, bt = yf - (float)(int)yf;
            const float s00 = (1.f - at) * (1.f - bt), s01 = at * (1.f - bt), s10 = (1.f - at) * bt, s11 = at * bt;
            float *pTL = Tb + ((long)tp.yT * W + tp.xL) * 4, *pTR = Tb + ((long)tp.yT * W + tp.xR) * 4;
            float *pBL = Tb + ((long)tp.yB * W + tp.xL) * 4, *pBR = Tb + ((long)tp.yB * W + tp.xR) * 4;
            red_add_v4(pTL, s00 * gv[0], s00 * gv[1], s00 * gv[2], 0.f);
            red_add_v4(pTR, s01 * gv[0], s01 * gv[1], s01 * gv[2], 0.f);
            red_add_v4(pBL, s10 * gv[0], s10 * gv[1], s10 * gv[2], 0.f);
            red_add_v4(pBR, s11 * gv[0], s11 * gv[1], s11 * gv[2], 0.f);
        }
        if (!NF) continue;
        if (o.ch_flow >= 0) {
            gfx += ldg_stream1(gc + (long)o.ch_flow * hw + pix) / o.flow_div;
            gfy += ldg_stream1(gc + (long)(o.ch_flow + 1) * hw + pix) / o.flow_div;
        }
        if (o.ch_fnorm >= 0) {
            const float fnrm = sqrtf(__fmaf_rn(fl.y, fl.y, __fmul_rn(fl.x, fl.x)));
            const float gf = ldg_stream1(gc + (long)o.ch_fnorm * hw + pix);
            gfx += gf * fl.x / (fnrm + 1e-9f);
            gfy += gf * fl.y / (fnrm + 1e-9f);
        }
        if (STAGE) {
            sg[0][ly + 8 * j][lx] = gfx;
            sg[1][ly + 8 * j][lx] = gfy;
            continue;
        }
        float *gfp = gflow + (long)b * 2 * hw + pix;
        __stcs(gfp, gfx);
        __stcs(gfp + hw, gfy);
    }
    if (!STAGE) return;
    // ---- adjoint of the x4 upsample (no thread has left: the early return above is UP == 0 only) ----
    __syncthreads();
    if (UP == 2) {
        constexpr int NCELL = (TH / 4) * 8;
        if (tid < 2 * NCELL) {
            const int comp = tid / NCELL, r = (tid % NCELL) >> 3, q = tid & 7;
            const int ci = byi * (TH / 4) + r, cj = bxi * 8 + q;
            if (ci < fs.fh && cj < fs.fw) {
                float s = 0.f;
#pragma unroll
                for (int yy = 0; yy < 4; ++yy)
#pragma unroll
                    for (int xx = 0; xx < 4; ++xx) s += sg[comp][4 * r + yy][4 * q + xx];
                __stcs(gflow + ((long)b * 2 + comp) * fs.fh * fs.fw + (long)ci * fs.fw + cj, __fmul_rn(s, fs.mul));
            }
        }
        return;
    }
    // bilinear: tile-local cell (r, q) is cell (TH/4 byi - 1 + r, 8 bxi - 1 + q); its pixels are local rows / columns
    // [4r - 6, 4r + 1] / [4q - 6, 4q + 1] clipped to the tile
    for (int it = tid; it < 2 * TH * NC; it += 256) {
        const int comp = it / (TH * NC), yl = (it / NC) % TH, q = it % NC;
        const int cj = bxi * 8 - 1 + q, xhi = min(4 * q + 1, 31);
        float s = 0.f;
        for (int xl = max(4 * q - 6, 0); xl <= xhi; ++xl) s = __fmaf_rn(up4_weight(bxi * 32 + xl, cj, fs.fw), sg[comp][yl][xl], s);
        sr[comp][yl][q] = s;
    }
    __syncthreads();
    if (tid < 2 * NR * NC) {
        const int comp = tid / (NR * NC), r = (tid / NC) % NR, q = tid % NC;
        const int ci = byi * (TH / 4) - 1 + r, yhi = min(4 * r + 1, TH - 1);
        float s = 0.f;
        for (int yl = max(4 * r - 6, 0); yl <= yhi; ++yl) s = __fmaf_rn(up4_weight(byi * TH + yl, ci, fs.fh), sr[comp][yl][q], s);
        gflow[(long)blockIdx.x * (2 * NR * NC) + tid] = s;
    }
}

// Bilinear x4 flow gradient from the per-tile partials of warp_concat_bwd_tile<.., 1, .., true>: cell (i, j) of
// component c sums the partials of the tiles (ty, tx) whose (TR + 2) x (TC + 2) cell window holds it -- ty ascending,
// then tx -- and multiplies by mul.  TR x TC: the cells one tile covers (4 x 8 for a 16 x 32 pixel tile).
template <int TR, int TC>
__global__ void __launch_bounds__(256)
warp_concat_up_finish(const float *__restrict__ P, float *__restrict__ gflow, int fh, int fw, int tiles_x, int tiles_y,
                      float mul, long n) {
    constexpr int NR = TR + 2, NC = TC + 2;
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    const int j = (int)(idx % fw), i = (int)((idx / fw) % fh);
    const long bc = idx / ((long)fh * fw);
    const int comp = (int)(bc & 1), b = (int)(bc >> 1);
    const int ty0 = max((i + TR - 1) / TR - 1, 0), ty1 = min((i + 1) / TR, tiles_y - 1);
    const int tx0 = max((j + TC - 1) / TC - 1, 0), tx1 = min((j + 1) / TC, tiles_x - 1);
    float s = 0.f;
    for (int ty = ty0; ty <= ty1; ++ty)
        for (int tx = tx0; tx <= tx1; ++tx)
            s += __ldg(P + (((long)b * tiles_y + ty) * tiles_x + tx) * (2 * NR * NC) + (comp * NR + i - TR * ty + 1) * NC +
                       j - TC * tx + 1);
    __stcs(gflow + idx, __fmul_rn(s, mul));
}

// T[b][y][x][4] -> gimg[b][c][y][x] (accumulate != 0: added to what gimg holds -- the *_cuda shim's caller-zeroed buffer)
template <int CT>
__global__ void __launch_bounds__(256)
resample2d_bwd_finish(const float *__restrict__ T, float *__restrict__ gimg, long hw, long npix, long gimg_bstride,
                      int accumulate) {
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= npix) return;
    const long b = idx / hw, p = idx - b * hw;
    const float4 t = ldg_stream4(T + idx * 4);
    float *o = gimg + b * gimg_bstride + p;
    const float v[3] = {t.x, t.y, t.z};
#pragma unroll
    for (int c = 0; c < CT; ++c) {
        if (accumulate) o[c * hw] += v[c];
        else __stcs(o + c * hw, v[c]);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
static int env_int(const char *name, int dflt, int lo, int hi) {
    const char *e = getenv(name);
    if (!e || !*e) return dflt;
    int v = atoi(e);
    return v < lo ? lo : (v > hi ? hi : v);
}

static ImgView view_of(const float *p, const int64_t *s) {
    ImgView v = {p, 0, 0, 0, 0};
    if (s) { v.sb = s[0]; v.sc = s[1]; v.sh = s[2]; v.sw = s[3]; }
    return v;
}

int resample2d_forward_tile(const float *img1, const int64_t *is1, const float *img0, const int64_t *is0,
                            const FlowSrc &fs, const WarpOut &o, int B, int C, int H, int W, int bilinear,
                            cudaStream_t st) {
    const int py = env_int("FN2B200_RS_PY", 4, 1, 4);
    const int PYc = py >= 4 ? 4 : (py >= 2 ? 2 : 1);
    const int tiles_x = (W + 31) / 32, tiles_y = (H + 8 * PYc - 1) / (8 * PYc);
    const long ntiles = (long)tiles_x * tiles_y * B;
    if (ntiles >= (1L << 31)) return fail(FN2B200_EINVAL, "resample2d_forward: %ld tiles exceed the grid limit", ntiles);
    const bool fused = o.ch_dnorm >= 0 || o.ch_flow >= 0 || o.ch_fnorm >= 0 || o.ch_x >= 0;
    const ImgView v1 = view_of(img1, is1), v0 = view_of(img0, is0);
    const unsigned grid = (unsigned)ntiles;
#define FN2_L(CT, PY)                                                                                                    \
    do {                                                                                                               \
        if (fused) resample2d_fwd_tile<CT, PY, true><<<grid, 256, 0, st>>>(v1, v0, fs, o, C, H, W, tiles_x, tiles_y, bilinear); \
        else resample2d_fwd_tile<CT, PY, false><<<grid, 256, 0, st>>>(v1, v0, fs, o, C, H, W, tiles_x, tiles_y, bilinear);      \
    } while (0)
#define FN2_C(PY)                                                                                                        \
    switch (C) {                                                                                                       \
        case 1: FN2_L(1, PY); break;                                                                                   \
        case 2: FN2_L(2, PY); break;                                                                                   \
        case 3: FN2_L(3, PY); break;                                                                                   \
        default: FN2_L(0, PY); break;                                                                                  \
    }
    if (PYc == 4) { FN2_C(4) } else if (PYc == 2) { FN2_C(2) } else { FN2_C(1) }
#undef FN2_C
#undef FN2_L
    count_launch();
    return check_launch("resample2d_forward");
}

size_t resample2d_backward_workspace_bytes(int B, int iH, int iW) { return (size_t)B * iH * iW * 4 * sizeof(float); }

// scatter: 1 planar scalar reductions, 2 vector reductions into the interleaved scratch (needs workspace, C <= 3)
int resample2d_backward_tile(const float *img, const int64_t *is, const float *flow, const float *gout, float *gimg,
                             float *gflow, void *workspace, int scatter, int accumulate, int B, int C, int iH, int iW,
                             int H, int W, cudaStream_t st) {
    const int py = env_int("FN2B200_RS_PY", 4, 1, 4);
    const int PYc = py >= 4 ? 4 : (py >= 2 ? 2 : 1);
    const int tiles_x = (W + 31) / 32, tiles_y = (H + 8 * PYc - 1) / (8 * PYc);
    const long ntiles = (long)tiles_x * tiles_y * B;
    if (ntiles >= (1L << 31)) return fail(FN2B200_EINVAL, "resample2d_backward: %ld tiles exceed the grid limit", ntiles);
    const unsigned grid = (unsigned)ntiles;
    const ImgView v = view_of(img, is);
    const FlowSrc fs = {flow, H, W, 0, 1.f};
    if (!gimg) scatter = 0;
    if (scatter == 2 && (C > 3 || !workspace)) scatter = 1;
    float *T = nullptr;
    if (scatter == 2) {
        T = static_cast<float *>(workspace);
        cudaError_t e = cudaMemsetAsync(T, 0, resample2d_backward_workspace_bytes(B, iH, iW), st);
        if (e != cudaSuccess) return fail((int)e, "resample2d_backward: workspace memset failed (%s)", cudaGetErrorString(e));
    }
#define FN2_B(CT, PY, SC) resample2d_bwd_tile<CT, PY, SC><<<grid, 256, 0, st>>>(v, fs, gout, gimg, T, gflow, C, iH, iW, H, W, tiles_x, tiles_y)
#define FN2_BC(PY, SC)                                                                                                   \
    switch (C) {                                                                                                       \
        case 1: FN2_B(1, PY, SC); break;                                                                               \
        case 2: FN2_B(2, PY, SC); break;                                                                               \
        case 3: FN2_B(3, PY, SC); break;                                                                               \
        default: FN2_B(0, PY, SC); break;                                                                              \
    }
// scatter 2 has C <= 3 (see above): no runtime-C instantiation
#define FN2_BC2(PY)                                                                                                      \
    switch (C) {                                                                                                       \
        case 1: FN2_B(1, PY, 2); break;                                                                                \
        case 2: FN2_B(2, PY, 2); break;                                                                                \
        default: FN2_B(3, PY, 2); break;                                                                               \
    }
#define FN2_BS(PY)                                                                                                       \
    switch (scatter) {                                                                                                 \
        case 0: FN2_BC(PY, 0) break;                                                                                   \
        case 1: FN2_BC(PY, 1) break;                                                                                   \
        default: FN2_BC2(PY) break;                                                                                    \
    }
    if (PYc == 4) { FN2_BS(4) } else if (PYc == 2) { FN2_BS(2) } else { FN2_BS(1) }
#undef FN2_BS
#undef FN2_BC2
#undef FN2_BC
#undef FN2_B
    count_launch();
    int rc = check_launch("resample2d_backward");
    if (rc || scatter != 2) return rc;
    return resample2d_backward_finish(T, gimg, accumulate, B, C, iH, iW, st);
}

int resample2d_backward_finish(const float *T, float *gimg, int accumulate, int B, int C, int iH, int iW, cudaStream_t st,
                               long gimg_bstride) {
    const long ihw = (long)iH * iW, npix = (long)B * ihw;
    const long bs = gimg_bstride ? gimg_bstride : (long)C * ihw;
    const unsigned g2 = (unsigned)((npix + 255) / 256);
    switch (C) {
        case 1: resample2d_bwd_finish<1><<<g2, 256, 0, st>>>(T, gimg, ihw, npix, bs, accumulate); break;
        case 2: resample2d_bwd_finish<2><<<g2, 256, 0, st>>>(T, gimg, ihw, npix, bs, accumulate); break;
        default: resample2d_bwd_finish<3><<<g2, 256, 0, st>>>(T, gimg, ihw, npix, bs, accumulate); break;
    }
    count_launch();
    return check_launch("resample2d_backward (finish)");
}

// PY = 2: 16 live tap registers per channel set; a 32 x 16 pixel tile, 8 x 4 quarter-resolution cells
static long warp_concat_tiles(int B, int H, int W) { return (long)((W + 31) / 32) * ((H + 15) / 16) * B; }

size_t warp_concat_backward_workspace_bytes(int B, int H, int W, int upsample_mode, bool need_x) {
    return (need_x ? resample2d_backward_workspace_bytes(B, H, W) : 0) +
           (upsample_mode == 1 ? (size_t)warp_concat_tiles(B, H, W) * 2 * (4 + 2) * (8 + 2) * sizeof(float) : 0);
}

int warp_concat_backward_tile(const float *x, const int64_t *xs, const FlowSrc &fs, const float *gcat, const WarpOut &o,
                              float *gx, float *gflow, void *workspace, int B, int C, int H, int W, cudaStream_t st) {
    const int tiles_x = (W + 31) / 32, tiles_y = (H + 15) / 16;
    const long ntiles = warp_concat_tiles(B, H, W);
    if (ntiles >= (1L << 31)) return fail(FN2B200_EINVAL, "warp_concat_backward: %ld tiles exceed the grid limit", ntiles);
    // workspace: [the scatter scratch T, when gx is wanted][the bilinear per-tile partials, when gflow is wanted]
    float *T = gx ? static_cast<float *>(workspace) : nullptr;
    float *P = (fs.mode == 1 && gflow)
                   ? reinterpret_cast<float *>(static_cast<char *>(workspace) + (gx ? resample2d_backward_workspace_bytes(B, H, W) : 0))
                   : nullptr;
    if (T) {
        cudaError_t e = cudaMemsetAsync(T, 0, resample2d_backward_workspace_bytes(B, H, W), st);
        if (e != cudaSuccess) return fail((int)e, "warp_concat_backward: workspace memset failed (%s)", cudaGetErrorString(e));
    }
    const ImgView v = view_of(x, xs);
    const unsigned grid = (unsigned)ntiles;
    float *gf = P ? P : gflow;
#define FN2_WB(CT, UP, NX, NF) warp_concat_bwd_tile<CT, 2, UP, NX, NF><<<grid, 256, 0, st>>>(v, fs, gcat, o, gx, T, gf, H, W, tiles_x, tiles_y)
#define FN2_WBN(CT, UP)                                                                                                  \
    do {                                                                                                               \
        if (gx && gflow) FN2_WB(CT, UP, true, true);                                                                   \
        else if (gx) FN2_WB(CT, UP, true, false);                                                                      \
        else FN2_WB(CT, UP, false, true);                                                                              \
    } while (0)
#define FN2_WBC(UP)                                                                                                      \
    switch (C) {                                                                                                       \
        case 1: FN2_WBN(1, UP); break;                                                                                 \
        case 2: FN2_WBN(2, UP); break;                                                                                 \
        default: FN2_WBN(3, UP); break;                                                                                \
    }
    if (fs.mode == 1) { FN2_WBC(1) } else if (fs.mode == 2) { FN2_WBC(2) } else { FN2_WBC(0) }
#undef FN2_WBC
#undef FN2_WBN
#undef FN2_WB
    count_launch();
    if (int rc = check_launch("warp_concat_backward")) return rc;
    if (P) {
        const long n = (long)B * 2 * fs.fh * fs.fw;
        warp_concat_up_finish<4, 8><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(P, gflow, fs.fh, fs.fw, tiles_x, tiles_y,
                                                                                   fs.mul, n);
        count_launch();
        if (int rc = check_launch("warp_concat_backward (flow upsample adjoint)")) return rc;
    }
    if (!T) return 0;
    // gx[:, C:2C] += T
    return resample2d_backward_finish(T, gx + (long)C * H * W, 1, B, C, H, W, st, (long)2 * C * H * W);
}

}  // namespace fn2

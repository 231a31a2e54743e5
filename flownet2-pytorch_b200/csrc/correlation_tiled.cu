// correlation_tiled.cu -- TMA-tiled FP32-FMA correlation (cost volume) forward and backward.
//
// Replaces, for kernel_size == 1 / stride1 == 1 (FlowNetC's configuration, networks/FlowNetC.py:28):
//   channels_first x2 + correlation_forward            (correlation_cuda_kernel.cu:46-70, :73-147)
//   channels_first x2 + correlation_backward_input1/2  (correlation_cuda_kernel.cu:150-241, :243-334,
//                                                        launched once per sample, :519-554)
//
// Design (not a translation):
//   * No padded NHWC scratch copies and no memsets: TMA tensor maps over the ORIGINAL NCHW tensors,
//     signed box coordinates + out-of-bounds zero fill give the zero padding for free.
//   * One launch covers the whole batch (the reference loops over samples on the host in backward).
//   * Operands are staged global -> shared by cp.async.bulk.tensor (UTMALDG) through a 3-stage
//     mbarrier ring; compute threads never issue global loads.
//   * Forward: every thread owns 8 consecutive output pixels x all (2*dr+1) x-displacements of ONE
//     (pixel row, y-displacement) pair = 168 fp32 accumulators in registers, kept live across the
//     whole channel reduction.  Per channel it reads 8 f1 words + a 48-word f2 window with 14
//     LDS.128 for 168 FMAs (3 FMA/word).  The 4 lane groups of a warp hold 4 pixel rows that
//     need the SAME f2 row (rows y+2k with tj = s-k), so their window loads are shared-memory
//     broadcasts.  A CTA = 4 pixel rows x 4 f2 rows x 128 pixels; the 24 f2-row offsets a row
//     quad needs are split over 6 CTAs, each writing disjoint displacement planes (no atomics).
//   * Backward: every thread owns 8 pixels x 4 channels of the input gradient and keeps the 21x8
//     gradOutput values of the current y-displacement in registers; per step it streams 4 channel
//     windows (48 words each) from shared memory: 672 FMAs per 90 LDS.128.  gradInput1 and
//     gradInput2 use the same kernel with mirrored displacement signs.  Outputs are written once
//     (no zero-filled accumulation buffers, no atomics).
//   * fp32 products, fp32 accumulation, result divided by k*k*C as in the reference (:143).
#include "common.cuh"

namespace fn2 {

constexpr int kPX = 8;     // pixels per thread along x
constexpr int kTW = 128;   // tile width in pixels (16 x-blocks)
constexpr int kNST = 3;    // pipeline stages

__host__ __device__ constexpr int round_up(int a, int b) { return (a + b - 1) / b * b; }

// ------------------------------------------------------------------------------------------------
// Forward
// ------------------------------------------------------------------------------------------------
template <int S2, int DR>
struct FwdCfg {
    static constexpr int DS = 2 * DR + 1;
    static constexpr int KR = 4;                                   // pixel rows per CTA
    static constexpr int SR = 4;                                   // f2 rows per CTA
    static constexpr int CK = 8;                                   // channels per stage
    static constexpr int HALO = DR * S2;                           // one-sided x halo
    static constexpr int WINP = round_up(kPX + 2 * HALO, 4);       // per-thread f2 window (words)
    static constexpr int F2W = kTW - kPX + WINP;                   // f2 box width (multiple of 4)
    static constexpr int NSG = (KR + 2 * DR + SR - 1) / SR;        // f2-row groups per row quad
    static constexpr int F1_STAGE = KR * CK * kTW;                 // floats
    static constexpr int F2_STAGE = SR * CK * F2W;                 // floats
    static constexpr int STAGE = F1_STAGE + F2_STAGE;              // floats
    static constexpr uint32_t STAGE_BYTES = STAGE * 4u;
    static constexpr size_t SMEM = (size_t)kNST * STAGE * 4 + 128 + kNST * 8;
};

template <int S2, int DR>
__global__ void __launch_bounds__(256, 1)
corr_fwd_tiled_kernel(const __grid_constant__ CUtensorMap map1,
                      const __grid_constant__ CUtensorMap map2, float *__restrict__ out,
                      CorrParams p) {
    using Cfg = FwdCfg<S2, DR>;
    constexpr int DS = Cfg::DS, KR = Cfg::KR, SR = Cfg::SR, CK = Cfg::CK;
    constexpr int HALO = Cfg::HALO, WINP = Cfg::WINP, F2W = Cfg::F2W;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *smem = reinterpret_cast<float *>(smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u));
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + (size_t)kNST * Cfg::STAGE);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int kk = lane >> 3;                      // pixel row within the quad (shares f2 row)
    const int xb = (warp & 1) * 8 + (lane & 7);    // x-block (8 px)
    const int sl = warp >> 1;                      // f2 row within the CTA's group

    const int sg = blockIdx.x % Cfg::NSG, xt = blockIdx.x / Cfg::NSG;
    const int cls = blockIdx.y % S2, grp = blockIdx.y / S2;
    const int n = blockIdx.z;
    const int Y0 = cls + S2 * KR * grp;            // first output row of the quad
    const int x0 = xt * kTW;                       // first output column of the tile
    const int off = p.md - p.pad;                  // output -> input coordinate shift
    const int s = -DR + sg * SR + sl;              // f2 row offset (units of S2) rel. to Y0
    const int tj = s - kk;
    const int oy = Y0 + S2 * kk;
    const bool active = (tj >= -DR) && (tj <= DR) && (oy < p.oH) && (x0 + kPX * xb < p.oW);

    const int nchunks = (p.C + CK - 1) / CK;

    if (tid == 0) {
        prefetch_tensormap(&map1);
        prefetch_tensormap(&map2);
        for (int i = 0; i < kNST; ++i) mbar_init(&full[i], 1);
        fence_barrier_init();
    }
    __syncthreads();

    auto issue = [&](int chunk) {
        const int st = chunk % kNST;
        float *f1s = smem + (size_t)st * Cfg::STAGE;
        float *f2s = f1s + Cfg::F1_STAGE;
        mbar_arrive_expect_tx(&full[st], Cfg::STAGE_BYTES);
#pragma unroll
        for (int k = 0; k < KR; ++k)
            tma_load_4d(f1s + k * CK * kTW, &map1, &full[st], x0 + off, Y0 + S2 * k + off,
                        chunk * CK, n);
#pragma unroll
        for (int r = 0; r < SR; ++r)
            tma_load_4d(f2s + r * CK * F2W, &map2, &full[st], x0 + off - HALO,
                        Y0 + off + S2 * (-DR + sg * SR + r), chunk * CK, n);
    };
    if (tid == 0)
        for (int c = 0; c < kNST && c < nchunks; ++c) issue(c);

    float acc[kPX][DS];
#pragma unroll
    for (int i = 0; i < kPX; ++i)
#pragma unroll
        for (int t = 0; t < DS; ++t) acc[i][t] = 0.f;

    for (int chunk = 0; chunk < nchunks; ++chunk) {
        const int st = chunk % kNST;
        mbar_wait(&full[st], (chunk / kNST) & 1);
        if (active) {
            const float *f1p = smem + (size_t)st * Cfg::STAGE + kk * CK * kTW + kPX * xb;
            const float *f2p = smem + (size_t)st * Cfg::STAGE + Cfg::F1_STAGE + sl * CK * F2W + kPX * xb;
#pragma unroll 2
            for (int c = 0; c < CK; ++c) {
                float a[kPX];
                {
                    float4 v0 = *reinterpret_cast<const float4 *>(f1p + c * kTW);
                    float4 v1 = *reinterpret_cast<const float4 *>(f1p + c * kTW + 4);
                    a[0] = v0.x; a[1] = v0.y; a[2] = v0.z; a[3] = v0.w;
                    a[4] = v1.x; a[5] = v1.y; a[6] = v1.z; a[7] = v1.w;
                }
#pragma unroll
                for (int m4 = 0; m4 < WINP / 4; ++m4) {
                    float4 wv = *reinterpret_cast<const float4 *>(f2p + c * F2W + 4 * m4);
                    const float w[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        // window word m holds f2[x + m - HALO]; pixel i pairs with ti = (m-HALO-i)/S2
#pragma unroll
                        for (int i = 0; i < kPX; ++i) {
                            const int d = 4 * m4 + e - HALO - i;
                            if (d % S2 == 0 && d / S2 >= -DR && d / S2 <= DR)
                                acc[i][d / S2 + DR] = fmaf(a[i], w[e], acc[i][d / S2 + DR]);
                        }
                    }
                }
            }
        }
        __syncthreads();  // every thread is done reading this stage -> it may be refilled
        if (tid == 0 && chunk + kNST < nchunks) issue(chunk + kNST);
    }

    if (active) {
        const float nelems = (float)(p.k * p.k * p.C);
        const int ox = x0 + kPX * xb;
        const long plane = (long)p.oH * p.oW;
        float *o = out + (long)n * p.out_bstride + (((long)(tj + DR) * DS) * p.oH + oy) * p.oW + ox;
        const float slope = p.leaky;          // 1 = no activation; otherwise nn.LeakyReLU(slope) (FlowNetC.py:87)
        auto fin = [nelems, slope](float a) {
            const float v = a / nelems;
            return v > 0.f ? v : v * slope;    // v * 1 == v bit for bit
        };
        if ((p.oW & 3) == 0 && ox + kPX <= p.oW) {
#pragma unroll
            for (int t = 0; t < DS; ++t) {
                float4 v0 = make_float4(fin(acc[0][t]), fin(acc[1][t]), fin(acc[2][t]), fin(acc[3][t]));
                float4 v1 = make_float4(fin(acc[4][t]), fin(acc[5][t]), fin(acc[6][t]), fin(acc[7][t]));
                stg_stream4(o + t * plane, v0);
                stg_stream4(o + t * plane + 4, v1);
            }
        } else {
#pragma unroll
            for (int t = 0; t < DS; ++t)
#pragma unroll
                for (int i = 0; i < kPX; ++i)
                    if (ox + i < p.oW) o[t * plane + i] = fin(acc[i][t]);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Backward (WHICH == 1: gradInput1 from input2; WHICH == 2: gradInput2 from input1).
// ACT: each stage also holds the forward's activated output at the gradOutput box's coordinates, and every gradOutput
// value g becomes (act > 0 ? g : g * p.leaky) as it moves to registers (fn2b200_correlation_backward_cat).
// ------------------------------------------------------------------------------------------------
template <int S2, int DR, int WHICH, bool ACT = false>
struct BwdCfg {
    static constexpr int DS = 2 * DR + 1;
    static constexpr int CB = 64;                                  // channels per CTA
    static constexpr int CC = 4;                                   // channels per thread
    static constexpr int HALO = DR * S2;
    static constexpr int WINP = round_up(kPX + 2 * HALO, 4);
    static constexpr int FW0 = kTW - kPX + WINP;
    // row pitch with pitch % 8 == 4 -> 8 consecutive channels hit 8 distinct 16-byte bank groups
    static constexpr int FW = FW0 + ((4 - FW0 % 8) + 8) % 8;
    static constexpr int GW = (WHICH == 1) ? kTW : FW0;            // gradOutput row width staged
    static constexpr int F_STAGE = CB * FW;                        // floats
    static constexpr int G_STAGE = round_up(DS * GW, 32);          // floats (128-B multiple)
    static constexpr int NG = ACT ? 2 : 1;                          // gradOutput (+ activation) boxes per stage
    static constexpr int STAGE = F_STAGE + NG * G_STAGE;
    static constexpr uint32_t STAGE_BYTES = (CB * FW + NG * DS * GW) * 4u;
    static constexpr size_t SMEM = (size_t)kNST * STAGE * 4 + 128 + kNST * 8;
};

// 8 consecutive floats from shared memory; `sh` = the row's word offset, a compile-time constant after unrolling,
// picks the widest aligned access
__device__ __forceinline__ void lds_row8(const float *q, int sh, float *d) {
    if ((sh & 3) == 0) {
        float4 v0 = *reinterpret_cast<const float4 *>(q);
        float4 v1 = *reinterpret_cast<const float4 *>(q + 4);
        d[0] = v0.x; d[1] = v0.y; d[2] = v0.z; d[3] = v0.w;
        d[4] = v1.x; d[5] = v1.y; d[6] = v1.z; d[7] = v1.w;
    } else if ((sh & 1) == 0) {
#pragma unroll
        for (int h = 0; h < 4; ++h) {
            float2 v = *reinterpret_cast<const float2 *>(q + 2 * h);
            d[2 * h] = v.x; d[2 * h + 1] = v.y;
        }
    } else {
#pragma unroll
        for (int i = 0; i < kPX; ++i) d[i] = q[i];
    }
}

template <int S2, int DR, int WHICH, bool ACT>
__global__ void __launch_bounds__(256, 1)
corr_bwd_tiled_kernel(const __grid_constant__ CUtensorMap map_other,
                      const __grid_constant__ CUtensorMap map_g, const __grid_constant__ CUtensorMap map_a,
                      float *__restrict__ gin, CorrParams p) {
    using Cfg = BwdCfg<S2, DR, WHICH, ACT>;
    constexpr int DS = Cfg::DS, CB = Cfg::CB, CC = Cfg::CC;
    constexpr int HALO = Cfg::HALO, WINP = Cfg::WINP, FW = Cfg::FW, GW = Cfg::GW;
    constexpr int SGN = (WHICH == 1) ? 1 : -1;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *smem = reinterpret_cast<float *>(smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u));
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + (size_t)kNST * Cfg::STAGE);

    const int tid = threadIdx.x;
    const int cl = tid & 15;   // channel lane: channels cl, cl+16, cl+32, cl+48 of the block
    const int xb = tid >> 4;   // x-block (8 px)

    const int nxt = (p.W + kTW - 1) / kTW;
    const int xt = blockIdx.x % nxt, cb = blockIdx.x / nxt;
    const int y = blockIdx.y, n = blockIdx.z;
    const int x0 = xt * kTW, c0 = cb * CB;
    const int off = p.md - p.pad;

    if (tid == 0) {
        prefetch_tensormap(&map_other);
        prefetch_tensormap(&map_g);
        if (ACT) prefetch_tensormap(&map_a);
        for (int i = 0; i < kNST; ++i) mbar_init(&full[i], 1);
        fence_barrier_init();
    }
    __syncthreads();

    // step t <-> tj = t - DR.  other row: y + SGN*tj*S2.  gO row: WHICH==1: y - off; else y - tj*S2 - off.
    auto issue = [&](int t) {
        const int st = t % kNST;
        const int tj = t - DR;
        float *fs = smem + (size_t)st * Cfg::STAGE;
        float *gs = fs + Cfg::F_STAGE;
        mbar_arrive_expect_tx(&full[st], Cfg::STAGE_BYTES);
        tma_load_4d(fs, &map_other, &full[st], x0 - HALO, y + SGN * tj * S2, c0, n);
        if (WHICH == 1) {
            tma_load_4d(gs, &map_g, &full[st], x0 - off, y - off, t * DS, n);
            if (ACT) tma_load_4d(gs + Cfg::G_STAGE, &map_a, &full[st], x0 - off, y - off, t * DS, n);
        } else {
            tma_load_4d(gs, &map_g, &full[st], x0 - off - HALO, y - tj * S2 - off, t * DS, n);
            if (ACT) tma_load_4d(gs + Cfg::G_STAGE, &map_a, &full[st], x0 - off - HALO, y - tj * S2 - off, t * DS, n);
        }
    };
    if (tid == 0)
        for (int t = 0; t < kNST && t < DS; ++t) issue(t);

    float acc[CC][kPX];
#pragma unroll
    for (int j = 0; j < CC; ++j)
#pragma unroll
        for (int i = 0; i < kPX; ++i) acc[j][i] = 0.f;

    for (int t = 0; t < DS; ++t) {
        const int st = t % kNST;
        mbar_wait(&full[st], (t / kNST) & 1);
        const float *fs = smem + (size_t)st * Cfg::STAGE + kPX * xb;
        const float *gs = smem + (size_t)st * Cfg::STAGE + Cfg::F_STAGE + kPX * xb;
        // gradOutput values for this y-displacement: g[ti][i]
        float g[DS][kPX];
#pragma unroll
        for (int ti = 0; ti < DS; ++ti) {
            // WHICH == 2: gO[(tj,ti)][..][x' - (ti-DR)*S2 - off]; staged row starts at x0 - off - HALO
            const int sh = (WHICH == 1) ? 0 : (2 * DR - ti) * S2;
            lds_row8(gs + ti * GW + sh, sh, g[ti]);
            if (ACT) {
                float a[kPX];
                lds_row8(gs + Cfg::G_STAGE + ti * GW + sh, sh, a);
#pragma unroll
                for (int i = 0; i < kPX; ++i) g[ti][i] = a[i] > 0.f ? g[ti][i] : g[ti][i] * p.leaky;
            }
        }
#pragma unroll
        for (int j = 0; j < CC; ++j) {
            const float *wrow = fs + (cl + 16 * j) * FW;
#pragma unroll
            for (int m4 = 0; m4 < WINP / 4; ++m4) {
                float4 wv = *reinterpret_cast<const float4 *>(wrow + 4 * m4);
                const float w[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    // window word m holds other[x + m - HALO]; pixel i pairs with ti where
                    // m - HALO - i = SGN * ti * S2
#pragma unroll
                    for (int i = 0; i < kPX; ++i) {
                        const int d = SGN * (4 * m4 + e - HALO - i);
                        if (d % S2 == 0 && d / S2 >= -DR && d / S2 <= DR)
                            acc[j][i] = fmaf(g[d / S2 + DR][i], w[e], acc[j][i]);
                    }
                }
            }
        }
        __syncthreads();
        if (tid == 0 && t + kNST < DS) issue(t + kNST);
    }

    const float nelems = (float)(p.k * p.k * p.C);
    const int x = x0 + kPX * xb;
    if (x < p.W) {
#pragma unroll
        for (int j = 0; j < CC; ++j) {
            const int c = c0 + cl + 16 * j;
            if (c >= p.C) continue;
            float *o = gin + (((long)n * p.C + c) * p.H + y) * p.W + x;
            if (x + kPX <= p.W) {  // W % 4 == 0 is a precondition of the tiled path
                stg_stream4(o, make_float4(acc[j][0] / nelems, acc[j][1] / nelems, acc[j][2] / nelems, acc[j][3] / nelems));
                stg_stream4(o + 4, make_float4(acc[j][4] / nelems, acc[j][5] / nelems, acc[j][6] / nelems, acc[j][7] / nelems));
            } else {
#pragma unroll
                for (int i = 0; i < kPX; ++i)
                    if (x + i < p.W) o[i] = acc[j][i] / nelems;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------
// (stride2, displacement radius) pairs with a compiled tiled kernel; the x halo dr*s2 must be a
// multiple of 4 (TMA traps on a dim-0 start coordinate that is not 16-byte aligned -- measured).
#define FN2_TILED_CONFIGS(X) X(2, 10) X(2, 4) X(1, 4) X(2, 2)

bool corr_tiled_supported(const CorrParams &p) {
    if (p.k != 1 || p.s1 != 1) return false;
    if (p.W % 4 != 0) return false;  // TMA global strides must be multiples of 16 bytes
    if (p.oW % 4 != 0) return false;  // gradOutput is a TMA source in backward
    if ((p.md - p.pad) % 4 != 0) return false;  // box x start = tile + (md - pad): must stay 16-B aligned
#define X(S2_, DR_) if (p.s2 == S2_ && p.dr == DR_) return true;
    FN2_TILED_CONFIGS(X)
#undef X
    return false;
}

// bstride: elements between samples (0 = C*H*W, dense; larger = a channel range of a wider tensor)
static int make_nchw_map(CUtensorMap *m, const float *base, int B, int C, int H, int W, int bw,
                         int bc, long bstride = 0) {
    uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)C, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)W * 4, (uint64_t)W * H * 4, (uint64_t)(bstride ? bstride : (long)W * H * C) * 4};
    uint32_t box[4] = {(uint32_t)bw, 1u, (uint32_t)bc, 1u};
    return make_tensor_map_f32(m, base, 4, dims, strides, box);
}

template <int S2, int DR>
static int launch_fwd(const float *in1, const float *in2, float *out, const CorrParams &p,
                      cudaStream_t st) {
    using Cfg = FwdCfg<S2, DR>;
    CUtensorMap m1, m2;
    int rc = make_nchw_map(&m1, in1, p.B, p.C, p.H, p.W, kTW, Cfg::CK);
    if (rc) return rc;
    rc = make_nchw_map(&m2, in2, p.B, p.C, p.H, p.W, Cfg::F2W, Cfg::CK);
    if (rc) return rc;
    auto kern = corr_fwd_tiled_kernel<S2, DR>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
    if (e != cudaSuccess) return fail((int)e, "correlation_forward: smem attribute (%s)", cudaGetErrorString(e));
    const int nxt = (p.oW + kTW - 1) / kTW;
    const int ngrp = ((p.oH + S2 - 1) / S2 + Cfg::KR - 1) / Cfg::KR;
    dim3 grid(Cfg::NSG * nxt, S2 * ngrp, p.B);
    kern<<<grid, 256, Cfg::SMEM, st>>>(m1, m2, out, p);
    count_launch();
    return check_launch("correlation_forward(tiled)");
}

template <int S2, int DR, int WHICH, bool ACT>
static int launch_bwd(const float *other, const float *gout, float *gin, const CorrParams &p,
                      cudaStream_t st) {
    using Cfg = BwdCfg<S2, DR, WHICH, ACT>;
    static_assert(Cfg::SMEM <= 232448, "tiled backward stage ring exceeds the 227 KB of shared memory per block");
    // gradOutput (and activation) maps: D planes per sample, p.g_bstride elements apart
    CUtensorMap mo, mg, ma;
    int rc = make_nchw_map(&mo, other, p.B, p.C, p.H, p.W, Cfg::FW, Cfg::CB);
    if (rc) return rc;
    rc = make_nchw_map(&mg, gout, p.B, p.D, p.oH, p.oW, Cfg::GW, Cfg::DS, p.g_bstride);
    if (rc) return rc;
    if (ACT && (rc = make_nchw_map(&ma, p.act, p.B, p.D, p.oH, p.oW, Cfg::GW, Cfg::DS, p.g_bstride))) return rc;
    if (!ACT) ma = mg;                           // not read
    auto kern = corr_bwd_tiled_kernel<S2, DR, WHICH, ACT>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM);
    if (e != cudaSuccess) return fail((int)e, "correlation_backward: smem attribute (%s)", cudaGetErrorString(e));
    const int nxt = (p.W + kTW - 1) / kTW;
    const int ncb = (p.C + Cfg::CB - 1) / Cfg::CB;
    dim3 grid(nxt * ncb, p.H, p.B);
    kern<<<grid, 256, Cfg::SMEM, st>>>(mo, mg, ma, gin, p);
    count_launch();
    return check_launch("correlation_backward(tiled)");
}

template <int S2, int DR, bool ACT>
static int launch_bwd_both(const float *in1, const float *in2, const float *gout, float *gin1, float *gin2,
                           const CorrParams &p, cudaStream_t st) {
    int rc = 0;
    if (gin1) rc = launch_bwd<S2, DR, 1, ACT>(in2, gout, gin1, p, st);
    if (!rc && gin2) rc = launch_bwd<S2, DR, 2, ACT>(in1, gout, gin2, p, st);
    return rc;
}

int corr_forward_tiled(const float *in1, const float *in2, float *out, const CorrParams &p,
                       cudaStream_t st) {
#define X(S2_, DR_) if (p.s2 == S2_ && p.dr == DR_) return launch_fwd<S2_, DR_>(in1, in2, out, p, st);
    FN2_TILED_CONFIGS(X)
#undef X
    return fail(FN2B200_EUNSUPPORTED, "correlation_forward(tiled): no kernel for stride2=%d, dr=%d", p.s2, p.dr);
}

int corr_backward_tiled(const float *in1, const float *in2, const float *gout, float *gin1,
                        float *gin2, const CorrParams &p, cudaStream_t st) {
#define X(S2_, DR_)                                                                                                     \
    if (p.s2 == S2_ && p.dr == DR_)                                                                                     \
        return p.act ? launch_bwd_both<S2_, DR_, true>(in1, in2, gout, gin1, gin2, p, st)                               \
                     : launch_bwd_both<S2_, DR_, false>(in1, in2, gout, gin1, gin2, p, st);
    FN2_TILED_CONFIGS(X)
#undef X
    return fail(FN2B200_EUNSUPPORTED, "correlation_backward(tiled): no kernel for stride2=%d, dr=%d", p.s2, p.dr);
}

}  // namespace fn2

// correlation_tc.cu -- tensor-core (wgmma) correlation FORWARD and BACKWARD for FlowNetC's configuration
// (kernel_size 1, stride1 1, stride2 2, displacement radius 10, pad == max_displacement).
//
// Formulation (DESIGN.md section 6).  stride2 = 2 means output pixel (y,x) only meets f2 pixels of
// the same (y mod 2, x mod 2) parity class, so each of the 4 classes is a stride-1 correlation on a
// half-resolution grid (Hc x Wc) with displacements tj,ti in [-10,10].  For a tile of 8 x 16 class
// pixels (M = 128 rows) the needed f2 pixels are the 28 x 36 halo; the cost volume is the band
// |tj|,|ti| <= 10 of the dense product
//        S[p, q] = sum_c f1[c, p] * f2[c, q]        (p in tile, q in halo),
// computed as a GEMM in 7 "units" of 4 halo rows (N = 144 columns) over K = C channels.
// fp32 accuracy on bf16 tensor cores: every operand is split x = hi + lo (two bf16, 16 significand
// bits); S = hi*hi + hi*lo + lo*hi (3 MMAs, fp32 accumulate in registers), dropped lo*lo ~ 2^-18 relative.
//
// Forward pipeline (one persistent CTA per SM, warp-specialised, 288 threads):
//   prepass kernel : NCHW fp32 -> [n][class][yc][xc][c] bf16 hi / lo (channels contiguous = K-major)
//   warp 8         : TMA producer: f1 tile  -> smem A [hi|lo][C/64][128 rows x 128 B]  (resident for the tile's units)
//                                  f2 units -> smem B ring, one slot = hi OR lo of a unit x 64 channels
//                    [144 rows x 128 B] = one 18-KB box, 128-byte swizzle; halo outside the image = TMA
//                    out-of-bounds zero fill = the layer's zero padding
//   warps 0-7      : two warpgroups, one per 64 tile pixels: wgmma m64n144k16 (hi slot: hi*hi and lo*hi, lo slot:
//                    hi*lo, 4 k-steps each) into an fp32 register accumulator, then each thread stores the band entries
//                    of its fragment, scaled by 1/C, to out[n][(tj,ti)][y][x]
#include "wgmma.cuh"
#include <cuda_bf16.h>
#include <stdlib.h>

namespace fn2 {

constexpr int TC_TH = 8, TC_TW = 16, TC_DR = 10;
constexpr int TC_HH = TC_TH + 2 * TC_DR;      // 28 halo rows
constexpr int TC_HW = TC_TW + 2 * TC_DR;      // 36 halo cols
constexpr int TC_UR = 4;                       // halo rows per unit
constexpr int TC_NU = TC_HH / TC_UR;           // 7 units per tile
constexpr int TC_N = TC_UR * TC_HW;            // 144 accumulator columns per unit
constexpr int TC_KB = 64;                      // channels per k-block (128 B of bf16)
constexpr int TC_MAXKB = 4;                    // C <= 256
constexpr int TC_MAXBST = 12;                  // B ring slots (one per hi / lo half-stage): as many as shared memory allows (runtime)
constexpr int TC_DS = 2 * TC_DR + 1;           // 21
constexpr int TC_ABLK = 128 * 128;             // bytes of one A k-block (128 rows x 128 B)
constexpr int TC_BBLK = TC_N * 128;            // bytes of one B k-block (144 rows x 128 B)
constexpr int TC_NBAR = 2 * TC_MAXKB + 2 * TC_MAXBST;
constexpr int TC_SMEM_MAX = 232448;            // 227 KB opt-in limit per CTA (sm_90)
// A_hi and A_lo blocks, then bst ring slots of one 18-KB box each (+ 1 KB for the 1024-byte alignment of the swizzle atoms)
__host__ __device__ constexpr int tc_smem_bytes(int nkb, int bst) {
    return 2 * nkb * TC_ABLK + bst * TC_BBLK + TC_NBAR * 8 + 1024;
}

// ------------------------------------------------------------------------------------------------
// Prepass: NCHW fp32 -> parity-class-separated NHWC bf16 hi / lo
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
corr_tc_split_kernel(const float *__restrict__ in0, const float *__restrict__ in1,
                     __nv_bfloat16 *__restrict__ hi0, __nv_bfloat16 *__restrict__ lo0,
                     __nv_bfloat16 *__restrict__ hi1, __nv_bfloat16 *__restrict__ lo1, int C, int H, int W) {
    __shared__ float tile[64][65];
    const int tid = threadIdx.x;
    const int ncb = C / 64;
    const int which = blockIdx.y / ncb, c0 = (blockIdx.y % ncb) * 64;
    const float *__restrict__ in = which ? in1 : in0;
    __nv_bfloat16 *__restrict__ hi = which ? hi1 : hi0;
    __nv_bfloat16 *__restrict__ lo = which ? lo1 : lo0;
    // grid: x = (sample, row) -- the only dimension that may exceed 65535 --, y = (input, channel block), z = 64-px column block
    const int x0 = blockIdx.z * 64;
    const int n = blockIdx.x / H, y = blockIdx.x % H;
    const int Hc = H >> 1, Wc = W >> 1;
    {
        const int xo = tid & 63, cs = tid >> 6;
        const float *src = in + (((long)n * C + c0) * H + y) * W + x0 + xo;
        const bool ok = x0 + xo < W;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int c = i * 4 + cs;
            tile[c][xo] = ok ? ldg_stream1(src + (long)c * H * W) : 0.f;
        }
    }
    __syncthreads();
    // thread -> (pixel, channels [8 cg, 8 cg + 8) and [32 + 8 cg, 40 + 8 cg)): the 4 threads of a pixel write 64
    // contiguous bytes per store instruction (whole 32-byte sectors; 16 channels per thread in one run made
    // every store touch only half of each sector)
    const int xo = tid >> 2, cg = tid & 3, x = x0 + xo;
    if (x < W) {
        const int cls = (y & 1) * 2 + (x & 1);
        const long row = (((long)(n * 4 + cls) * Hc + (y >> 1)) * Wc + (x >> 1)) * C + c0;
        uint32_t hw[8], lw[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int c = (i >> 2) * 32 + cg * 8 + 2 * (i & 3);
            const float v0 = tile[c][xo], v1 = tile[c + 1][xo];
            const __nv_bfloat16 h0 = __float2bfloat16_rn(v0), h1 = __float2bfloat16_rn(v1);
            const __nv_bfloat16 l0 = __float2bfloat16_rn(v0 - __bfloat162float(h0));
            const __nv_bfloat16 l1 = __float2bfloat16_rn(v1 - __bfloat162float(h1));
            hw[i] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
            lw[i] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
        }
        uint4 *ph = reinterpret_cast<uint4 *>(hi + row + cg * 8), *pl = reinterpret_cast<uint4 *>(lo + row + cg * 8);
        ph[0] = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        ph[4] = make_uint4(hw[4], hw[5], hw[6], hw[7]);      // + 32 channels = 64 bytes
        pl[0] = make_uint4(lw[0], lw[1], lw[2], lw[3]);
        pl[4] = make_uint4(lw[4], lw[5], lw[6], lw[7]);
    }
}

// ------------------------------------------------------------------------------------------------
// Main kernel
// ------------------------------------------------------------------------------------------------
struct TcTile {
    int n, py, px, yc0, xc0;
};
__device__ __forceinline__ TcTile tc_decode(int t, int nxt, int nyt) {
    TcTile r;
    r.px = t & 1;
    int q = t >> 1;
    r.xc0 = (q % nxt) * TC_TW;
    q /= nxt;
    r.yc0 = (q % nyt) * TC_TH;
    q /= nyt;
    r.py = q & 1;
    r.n = q >> 1;
    return r;
}

// A CTA's work list: whole tiles tn, tn + grid, ... below `full`, then its share [w, w1) of the
// (tile, unit) pairs of the last partial round (tile = full + w / 7).
struct TcSeg {
    int t, ua, ub;
};
__device__ __forceinline__ bool tc_next_seg(int &tn, int &w, int full, int w1, TcSeg &sg) {
    if (tn < full) {
        sg.t = tn; sg.ua = 0; sg.ub = TC_NU;
        tn += gridDim.x;
        return true;
    }
    if (w < w1) {
        sg.t = full + w / TC_NU; sg.ua = w % TC_NU;
        sg.ub = (TC_NU - sg.ua < w1 - w) ? TC_NU : sg.ua + (w1 - w);
        w += sg.ub - sg.ua;
        return true;
    }
    return false;
}

// Warps 0-7: two consumer warpgroups; warpgroup wg owns tile pixels [64 wg, 64 wg + 64) (tile rows 4 wg .. 4 wg + 3) and
// keeps their m64 x n144 accumulator of the current unit in registers.  Warp 8: the TMA producer (one lane issues).
constexpr int TC_CONSUMERS = 256;
constexpr int TC_THREADS = TC_CONSUMERS + 32;
__global__ void __launch_bounds__(TC_THREADS, 1)
corr_fwd_tc_kernel(const __grid_constant__ CUtensorMap m1h, const __grid_constant__ CUtensorMap m1l,
                   const __grid_constant__ CUtensorMap m2h, const __grid_constant__ CUtensorMap m2l,
                   float *__restrict__ out, long out_bstride, float leaky, int B, int C, int H, int W, int ntiles,
                   int bst) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int Hc = H >> 1, Wc = W >> 1;
    const int nxt = (Wc + TC_TW - 1) / TC_TW, nyt = (Hc + TC_TH - 1) / TC_TH;
    const int nkb = C / TC_KB;
    // Whole tiles round-robin over the CTAs (neighbouring tiles run concurrently and share their halos in L2) for as
    // many full rounds as there are; the tiles of the last, partial round are dealt out by (tile, unit) pairs -- the 7
    // units of a tile write disjoint displacement rows -- so that the last round costs a few units, not a whole tile.
    const int full = (ntiles / (int)gridDim.x) * (int)gridDim.x;
    const int wtotal = (ntiles - full) * TC_NU, wper = (wtotal + (int)gridDim.x - 1) / (int)gridDim.x;
    const int w0 = (int)blockIdx.x * wper < wtotal ? (int)blockIdx.x * wper : wtotal;
    const int w1 = (w0 + wper < wtotal) ? w0 + wper : wtotal;
    unsigned char *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    unsigned char *sA = smem;                              // A_hi [kb][128 rows x 128 B], resident for a tile's units
    unsigned char *sAlo = smem + nkb * TC_ABLK;            // A_lo [kb][128 rows x 128 B]
    unsigned char *sB = smem + 2 * nkb * TC_ABLK;          // ring [slot][144 rows x 128 B]
    uint64_t *bars = reinterpret_cast<uint64_t *>(sB + bst * TC_BBLK);
    uint64_t *a_full = bars, *a_empty = bars + TC_MAXKB;
    uint64_t *b_full = bars + 2 * TC_MAXKB, *b_empty = b_full + TC_MAXBST;

    if (tid == 0) {
        prefetch_tensormap(&m1h); prefetch_tensormap(&m1l);
        prefetch_tensormap(&m2h); prefetch_tensormap(&m2l);
        for (int i = 0; i < TC_MAXKB; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], TC_CONSUMERS); }
        for (int i = 0; i < TC_MAXBST; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], TC_CONSUMERS); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == TC_CONSUMERS / 32) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            uint32_t bcount = 0;
            int it = 0;
            const uint64_t pol = l2_policy_evict_last();
            TcSeg sg;
            for (int tn = blockIdx.x, w = w0; tc_next_seg(tn, w, full, w1, sg); ++it) {
                const TcTile T = tc_decode(sg.t, nxt, nyt);
                const int img = T.n * 4 + T.py * 2 + T.px;
                // the tile's A blocks: one k-block is refilled as soon as the previous segment's last unit has read it
                for (int kb = 0; kb < nkb; ++kb) {
                    mbar_wait(&a_empty[kb], (it & 1) ^ 1);
                    mbar_arrive_expect_tx(&a_full[kb], 2 * TC_ABLK);
                    tma_load_4d_hint(sA + kb * TC_ABLK, &m1h, &a_full[kb], kb * TC_KB, T.xc0, T.yc0, img, pol);
                    tma_load_4d_hint(sAlo + kb * TC_ABLK, &m1l, &a_full[kb], kb * TC_KB, T.xc0, T.yc0, img, pol);
                }
                // B: one 18-KB box per half-stage (hi, then lo, of one unit x k-block); halo outside the image = TMA
                // out-of-bounds zero fill = the layer's zero padding
                for (int u = sg.ua; u < sg.ub; ++u)
                    for (int kb = 0; kb < nkb; ++kb)
                        for (int hl = 0; hl < 2; ++hl, ++bcount) {
                            const int s = bcount % bst;
                            mbar_wait(&b_empty[s], ((bcount / bst) & 1) ^ 1);
                            mbar_arrive_expect_tx(&b_full[s], TC_BBLK);
                            tma_load_4d_hint(sB + s * TC_BBLK, hl ? &m2l : &m2h, &b_full[s], kb * TC_KB, T.xc0 - TC_DR,
                                             T.yc0 - TC_DR + u * TC_UR, img, pol);
                        }
            }
        }
    } else {
        // ===================== consumers: wgmma + epilogue =====================
        const int wg = warp >> 2, wq = warp & 3;
        // accumulator fragment: rows 16 wq + lane / 4 (+ 8) of the warpgroup = tile row 4 wg + wq, columns pxa (+ 8)
        const int py_t = 4 * wg + wq, pxa = lane >> 2, q = lane & 3;
        // 1/(k*k*C): exact for power-of-two C (FlowNetC: 256) -> bit-identical to the reference's divide; otherwise
        // within 1 ulp.
        const float inv_nelems = 1.0f / (float)C;
        const long plane = (long)H * W;
        const bool act = leaky != 1.f;
        uint32_t bcount = 0;
        int it = 0;
        TcSeg sg;
        for (int tn = blockIdx.x, w = w0; tc_next_seg(tn, w, full, w1, sg); ++it) {
            const int ua = sg.ua, ub = sg.ub;
            const TcTile T = tc_decode(sg.t, nxt, nyt);
            const int yc = T.yc0 + py_t, xc = T.xc0 + pxa;
            const bool ok0 = (yc < Hc) && (xc < Wc), ok1 = (yc < Hc) && (xc + 8 < Wc);
            float *ob = out + (long)T.n * out_bstride + (long)(2 * yc + T.py) * W + (2 * xc + T.px);
            for (int u = ua; u < ub; ++u) {
                float acc[TC_N / 2];
#pragma unroll
                for (int i = 0; i < TC_N / 2; ++i) acc[i] = 0.f;
                wgmma_fence_operands(acc);
                int prev = -1, prev_a = -1;            // ring slot (and A block) read by the wgmma group in flight
                for (int kb = 0; kb < nkb; ++kb) {
                    if (u == ua) mbar_wait(&a_full[kb], it & 1);
                    const uint64_t dh = wgmma_desc_k_sw128(smem_u32(sA + kb * TC_ABLK + wg * (TC_ABLK / 2)));
                    const uint64_t dl = wgmma_desc_k_sw128(smem_u32(sAlo + kb * TC_ABLK + wg * (TC_ABLK / 2)));
#pragma unroll
                    for (int hl = 0; hl < 2; ++hl, ++bcount) {
                        const int s = bcount % bst;
                        mbar_wait(&b_full[s], (bcount / bst) & 1);
                        const uint64_t bd = wgmma_desc_k_sw128(smem_u32(sB + s * TC_BBLK));
                        wgmma_fence();
#pragma unroll
                        for (int ks = 0; ks < TC_KB / 16; ++ks) {
                            wgmma_m64n144k16_k(acc, dh + 2 * ks, bd + 2 * ks);             // hi x hi | hi x lo
                            if (hl == 0) wgmma_m64n144k16_k(acc, dl + 2 * ks, bd + 2 * ks); // lo x hi
                        }
                        wgmma_commit();
                        wgmma_wait<1>();
                        if (prev >= 0) {
                            mbar_arrive(&b_empty[prev]);
                            if (prev_a >= 0) mbar_arrive(&a_empty[prev_a]);
                        }
                        prev = s;
                        prev_a = (hl == 1 && u == ub - 1) ? kb : -1;       // A block free for the next segment
                    }
                }
                wgmma_wait<0>();
                wgmma_fence_operands(acc);
                mbar_arrive(&b_empty[prev]);
                if (prev_a >= 0) mbar_arrive(&a_empty[prev_a]);
                // accumulator column c = hrl * 36 + qx (halo row hrl of the unit, halo column qx) of tile pixel
                // (py_t, px) is displacement (tj, ti) = (u * 4 + hrl - py_t, qx - px) - (10, 10), if inside the band
                const int tjb = u * TC_UR - py_t;
#pragma unroll
                for (int i = 0; i < TC_N / 8; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int c = 8 * i + 2 * q + (j & 1);
                        const int hrl = c / TC_HW;
                        const int ti = c - hrl * TC_HW - pxa - 8 * (j >> 1), tj = tjb + hrl;
                        if (((j >> 1) ? ok1 : ok0) && (unsigned)ti < (unsigned)TC_DS && (unsigned)tj < (unsigned)TC_DS) {
                            float v = acc[4 * i + j] * inv_nelems;
                            if (act) v = v > 0.f ? v : v * leaky;      // fused nn.LeakyReLU (FlowNetC.py:87), warp-uniform
                            __stcs(ob + 16 * (j >> 1) + (long)(tj * TC_DS + ti) * plane, v);
                        }
                    }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Backward on tensor cores: gradInput1 tiles (other = input2) and gradInput2 tiles (other = input1).
//
//   gI1[c, p] = 1/C sum_q G1[p, q] f2[c, q],   G1[p, q] = gO[(q - p), p]          (|q - p| <= 10)
//   gI2[c, q] = 1/C sum_p G2[q, p] f1[c, p],   G2[q, p] = gO[(q - p), p]
// per parity class: D[128 tile px][C] += A[128][144] * B[144 halo px][C] over the 7 halo-row units, accumulated in
// registers (warpgroup wg: tile pixels [64 wg, 64 wg + 64), an m64 x nC fragment) for the whole tile.
//   A = the banded gradOutput matrix, built per unit by the warpgroup's own threads straight from the fp32 gradOutput
//       planes (bf16 hi/lo split on the fly) into an MN-major SW128 layout [k][64 pixels] (two buffers per warpgroup,
//       so that building unit u + 1 overlaps the last wgmma group of unit u, and each warpgroup's building overlaps
//       the other's MMAs);
//   B = the other input's halo chunk from the prepass copy ([pixel][channel] bf16 = MN-major operand), one ring slot =
//       hi OR lo of a K-group (48 halo pixels) x all channel blocks;
//   3 products (hi*hi, lo*hi | hi*lo) per k-step, N = C <= 256 per instruction.
// Two threads per tile pixel build A: halo rows {2 hp, 2 hp + 1} x all 21 displacements each.  Loads stay coalesced
// (lanes = pixels, one displacement plane per instruction); the band positions a pixel row writes are the same for
// every unit, so the zero columns of A are written ONCE at kernel start and the scatter offsets live in registers.
// ------------------------------------------------------------------------------------------------
constexpr int TB_AHL = TC_N * 128;                 // 18432 B: hi (or lo) of a warpgroup's A, [k][64 pixels] (MN-major, SW128)
constexpr int TB_ASTG = 2 * TB_AHL;                // hi + lo
constexpr int TB_NAST = 2;                         // A buffers per warpgroup
constexpr int TB_SMEM_A = 2 * TB_NAST * TB_ASTG;   // 147456
// byte offset of A element (pixel p of the warpgroup's 64, k): pixels contiguous, 16-byte chunk index XOR (k & 7)
__host__ __device__ constexpr uint32_t tb_a_offset(uint32_t p, uint32_t k) {
    return k * 128u + ((((p >> 3) ^ (k & 7u))) << 4) + (p & 7u) * 2u;
}
constexpr int TB_MAXBST = 6;
constexpr int TB_NBAR = 2 * TB_MAXBST;
// B staging: the unit's 144 K indices in 3 groups of 48 (12 halo columns x 4 rows); one ring slot = the hi (or the lo)
// copy of one group x ALL channel blocks = up to 4 boxes of 6 KB, so every wgmma covers N = C columns.
constexpr int TB_NG = 3, TB_GW = TC_HW / TB_NG, TB_GK = TC_UR * TB_GW;   // 3 groups, 12 columns, 48 K
constexpr int TB_GBLK = TB_GK * 128;               // 6144 B: one 64-channel block of a group's rows
constexpr int TB_BSTAGE = 4 * TB_GBLK;             // 24576 B: [<= 4 channel blocks][48 rows x 128 B]
__host__ __device__ constexpr uint32_t tb_kindex(uint32_t hrl, uint32_t qx) {
    return (qx / TB_GW) * TB_GK + hrl * TB_GW + (qx % TB_GW);
}
// warps 0-7: two warpgroups (build A, wgmma, epilogue) with 232 registers a thread (setmaxnreg: the m64 x n256 accumulator
// alone is 128); warps 8-11: a producer warpgroup lowered to 40 registers, of which warp 8 issues the TMA loads
constexpr int TB_THREADS = TC_CONSUMERS + 128;
__host__ __device__ constexpr int tb_smem_bytes(int bst) {
    return TB_SMEM_A + bst * TB_BSTAGE + TB_NBAR * 8 + 1024;
}

template <int NKB>
__device__ __forceinline__ void wgmma_bwd(float (&d)[NKB * 32], uint64_t da, uint64_t db);
template <> __device__ __forceinline__ void wgmma_bwd<1>(float (&d)[32], uint64_t da, uint64_t db) { wgmma_m64n64k16_mn(d, da, db); }
template <> __device__ __forceinline__ void wgmma_bwd<2>(float (&d)[64], uint64_t da, uint64_t db) { wgmma_m64n128k16_mn(d, da, db); }
template <> __device__ __forceinline__ void wgmma_bwd<3>(float (&d)[96], uint64_t da, uint64_t db) { wgmma_m64n192k16_mn(d, da, db); }
template <> __device__ __forceinline__ void wgmma_bwd<4>(float (&d)[128], uint64_t da, uint64_t db) { wgmma_m64n256k16_mn(d, da, db); }

// Both gradients in ONE launch: global tiles [t_begin, t_end) of [0, 2 ntiles).  One gradient only: tile g < ntiles
// is tile g of gradInput1 (B = input2's halo, maps m2h / m2l), tile g >= ntiles is tile g - ntiles of gradInput2
// (B = input1's halo); both: g = 2 tile + (0 = gradInput1, 1 = gradInput2).
template <int NKB>
__global__ void __launch_bounds__(TB_THREADS, 1)
corr_bwd_tc_kernel(const __grid_constant__ CUtensorMap m2h, const __grid_constant__ CUtensorMap m2l,
                   const __grid_constant__ CUtensorMap m1h, const __grid_constant__ CUtensorMap m1l,
                   const float *__restrict__ gout, float *__restrict__ gin1, float *__restrict__ gin2, int B,
                   int H, int W, int ntiles, int t_begin, int t_end, int bst) {
    constexpr int C = NKB * TC_KB;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    unsigned char *sA = smem;                          // [warpgroup][buffer][hi | lo][144 k x 128 B]
    unsigned char *sB = smem + TB_SMEM_A;              // [slot][channel block][48 rows x 128 B] (SW128, MN-major)
    uint64_t *bars = reinterpret_cast<uint64_t *>(sB + bst * TB_BSTAGE);
    uint64_t *b_full = bars, *b_empty = bars + TB_MAXBST;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int Hc = H >> 1, Wc = W >> 1;
    const int nxt = (Wc + TC_TW - 1) / TC_TW, nyt = (Hc + TC_TH - 1) / TC_TH;
    const long plane = (long)H * W;
    // both gradients requested: even global tiles are gradInput1 tiles, odd ones the gradInput2 tile of the same
    // location, so the two readers of a gradOutput region run side by side and the second one finds it in L2
    const bool both = (t_begin == 0) && (t_end == 2 * ntiles);

    if (tid == 0) {
        prefetch_tensormap(&m2h); prefetch_tensormap(&m2l);
        prefetch_tensormap(&m1h); prefetch_tensormap(&m1l);
        for (int i = 0; i < TB_MAXBST; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], TC_CONSUMERS); }
        fence_barrier_init();
    }
    // columns of A outside a pixel row's band are zero for every unit: written once, here
    for (int i = tid; i < TB_SMEM_A / 16; i += TB_THREADS) reinterpret_cast<uint4 *>(sA)[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async();
    __syncthreads();

    if (warp >= TC_CONSUMERS / 32) {
        // ===================== TMA producer: the other input's halo chunks =====================
        setmaxnreg_dec<40>();
        if (warp == TC_CONSUMERS / 32 && lane == 0) {
            uint32_t bcount = 0;
            const uint64_t pol = l2_policy_evict_last();
            for (int g = t_begin + blockIdx.x; g < t_end; g += gridDim.x) {
                const bool second = both ? (g & 1) : (g >= ntiles);
                const TcTile T = tc_decode(both ? (g >> 1) : (second ? g - ntiles : g), nxt, nyt);
                const int img = T.n * 4 + T.py * 2 + T.px;
                const CUtensorMap *moh = second ? &m1h : &m2h, *mol = second ? &m1l : &m2l;
                for (int u = 0; u < TC_NU; ++u)
                    for (int gr = 0; gr < TB_NG; ++gr)
                        for (int hl = 0; hl < 2; ++hl, ++bcount) {
                            const int s = bcount % bst;
                            mbar_wait(&b_empty[s], ((bcount / bst) & 1) ^ 1);
                            mbar_arrive_expect_tx(&b_full[s], (uint32_t)(NKB * TB_GBLK));
                            unsigned char *dst = sB + s * TB_BSTAGE;
#pragma unroll
                            for (int j = 0; j < NKB; ++j)
                                tma_load_4d_hint(dst + j * TB_GBLK, hl ? mol : moh, &b_full[s], j * TC_KB,
                                                 T.xc0 - TC_DR + gr * TB_GW, T.yc0 - TC_DR + u * TC_UR, img, pol);
                        }
            }
        }
        return;
    }
    setmaxnreg_inc<232>();

    const int wg = warp >> 2, wq = warp & 3;
    // builder role: pixel bp of the warpgroup's 64 (a warp covers 4 tile rows x 8 pixels: its 32 two-byte stores of
    // one (halo row, displacement) hit 32 different banks), halo rows {2 hp, 2 hp + 1}
    const int hp = wq >> 1;
    const int bp = (lane >> 3) * TC_TW + (wq & 1) * 8 + (lane & 7);
    const int bpy = 4 * wg + (bp >> 4), bpx = bp & 15;
    // accumulator fragment role: rows 16 wq + lane / 4 (+ 8) of the warpgroup
    const int py_t = 4 * wg + wq, pxa = lane >> 2, q = lane & 3;
    const int iplane = (int)plane;             // all tensors < 2^31 elements (checked by the C ABI)
    unsigned char *aw = sA + wg * TB_NAST * TB_ASTG;
    const float inv_nelems = 1.0f / (float)C;
    uint32_t bcount = 0, ucount = 0;
    for (int g = t_begin + blockIdx.x; g < t_end; g += gridDim.x) {
        const bool second = both ? (g & 1) : (g >= ntiles);           // gradInput2 tile (block-uniform)
        const TcTile T = tc_decode(both ? (g >> 1) : (second ? g - ntiles : g), nxt, nyt);
        const int nbase = T.n * (TC_DS * TC_DS);
        // Per-tile address set-up of the builder pixel (element offsets fit in 32 bits): for unit u the band row of
        // halo row hrl = 2hp+hh starts at off[hh] + u * dstep; consecutive displacements are `step` apart.
        int off[2], dstep, step, ystep, tj0[2], ys0[2];
        uint32_t colmask = 0;                                  // displacements to load (gradInput2: source columns inside the image)
        {
            const int yc = T.yc0 + bpy, xc = T.xc0 + bpx;
            const bool pix_ok = (yc < Hc) && (xc < Wc);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int hrl = 2 * hp + hh;
                tj0[hh] = hrl - bpy;                               // tj + 10 at u = 0 (+4 per unit)
                if (!second) {
                    ys0[hh] = pix_ok ? 0 : Hc;                     // gO at the output pixel itself
                    off[hh] = ((nbase + tj0[hh] * TC_DS) * H + (2 * yc + T.py)) * W + (2 * xc + T.px);
                } else {
                    ys0[hh] = T.yc0 - TC_DR + hrl;                 // source pixel row at u = 0 (+4 per unit)
                    const int xs0 = T.xc0 - TC_DR + bpx;           // source column for j = 0
                    off[hh] = ((nbase + (TC_DS - 1 - tj0[hh]) * TC_DS + (TC_DS - 1)) * H + (2 * ys0[hh] + T.py)) * W +
                              (2 * xs0 + T.px);
                    if (hh == 0)
#pragma unroll
                        for (int j = 0; j < TC_DS; ++j)
                            if ((unsigned)(xs0 + j) < (unsigned)Wc) colmask |= 1u << j;
                }
            }
            if (!second) {
                step = iplane;                                     // next ti -> next plane
                dstep = TC_UR * TC_DS * iplane;                    // next unit -> tj + 4
                ystep = 0;
                colmask = (1u << TC_DS) - 1u;
            } else {
                ystep = TC_UR;
                step = 2 - iplane;                                 // j -> j+1: -1 plane, +2 in x
                dstep = -TC_UR * TC_DS * iplane + 2 * TC_UR * W;   // next unit: tj + 4 -> -84 planes; source row + 4 -> +8 rows
            }
        }
        float acc[C / 2];
#pragma unroll
        for (int i = 0; i < C / 2; ++i) acc[i] = 0.f;
        wgmma_fence_operands(acc);
        int prev = -1;                                         // ring slot read by the wgmma group in flight
        for (int u = 0; u < TC_NU; ++u, ++ucount) {
            // buffer ucount & 1 was last read by unit ucount - 2, complete since unit ucount - 1's first wait
            unsigned char *ah = aw + (ucount & 1) * TB_ASTG, *al = ah + TB_AHL;
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int tjp = tj0[hh] + u * TC_UR;
                const bool row_ok = ((unsigned)tjp < (unsigned)TC_DS) && ((unsigned)(ys0[hh] + u * ystep) < (unsigned)Hc);
                const int base = off[hh] + u * dstep;          // only dereferenced under `ok`
                float v[TC_DS];
#pragma unroll
                for (int j = 0; j < TC_DS; ++j) {
                    const bool ok = row_ok && ((colmask >> j) & 1u);
                    v[j] = ok ? __ldg(gout + (base + j * step)) : 0.f;
                }
#pragma unroll
                for (int j = 0; j < TC_DS; ++j) {
                    const __nv_bfloat16 h = __float2bfloat16_rn(v[j]);
                    const __nv_bfloat16 l = __float2bfloat16_rn(v[j] - __bfloat162float(h));
                    const uint32_t o = tb_a_offset(bp, tb_kindex(2 * hp + hh, bpx + j));   // unit-invariant
                    *reinterpret_cast<unsigned short *>(ah + o) = __bfloat16_as_ushort(h);
                    *reinterpret_cast<unsigned short *>(al + o) = __bfloat16_as_ushort(l);
                }
            }
            fence_proxy_async();                               // generic-proxy writes -> visible to the tensor core
            named_barrier_sync(1 + wg, 128);                   // the warpgroup's whole A is written
            const uint32_t ah32 = smem_u32(ah), al32 = smem_u32(al);
            for (int gr = 0; gr < TB_NG; ++gr)
#pragma unroll
                for (int hl = 0; hl < 2; ++hl, ++bcount) {
                    const int s = bcount % bst;
                    mbar_wait(&b_full[s], (bcount / bst) & 1);
                    const uint32_t bb = smem_u32(sB + s * TB_BSTAGE);
                    wgmma_fence();
#pragma unroll
                    for (int ks = 0; ks < TB_GK / 16; ++ks) {
                        const uint32_t ko = (gr * TB_GK + ks * 16) * 128;
                        const uint64_t bd = wgmma_desc_mn_sw128(bb + ks * 16 * 128, TB_GBLK);
                        wgmma_bwd<NKB>(acc, wgmma_desc_mn_sw128(ah32 + ko, TB_AHL), bd);           // hi x hi | hi x lo
                        if (hl == 0) wgmma_bwd<NKB>(acc, wgmma_desc_mn_sw128(al32 + ko, TB_AHL), bd);  // lo x hi
                    }
                    wgmma_commit();
                    wgmma_wait<1>();
                    if (prev >= 0) mbar_arrive(&b_empty[prev]);
                    prev = s;
                }
        }
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
        mbar_arrive(&b_empty[prev]);
        // epilogue: fragment rows = tile pixels (py_t, pxa) and (py_t, pxa + 8), columns = channels
        const int yc = T.yc0 + py_t, xc = T.xc0 + pxa;
        const bool ok0 = (yc < Hc) && (xc < Wc), ok1 = (yc < Hc) && (xc + 8 < Wc);
        float *o = (second ? gin2 : gin1) + (long)T.n * C * plane + (long)(2 * yc + T.py) * W + (2 * xc + T.px);
#pragma unroll
        for (int i = 0; i < C / 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if ((j >> 1) ? ok1 : ok0)
                    __stcs(o + 16 * (j >> 1) + (long)(8 * i + 2 * q + (j & 1)) * plane, acc[4 * i + j] * inv_nelems);
    }
}

// ------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------
bool corr_tc_supported(const CorrParams &p) {
    return p.k == 1 && p.s1 == 1 && p.s2 == 2 && p.dr == TC_DR && p.pad == p.md && (p.H % 2 == 0) &&
           (p.W % 2 == 0) && (p.C % TC_KB == 0) && p.C <= TC_KB * TC_MAXKB && p.H >= 2 && p.W >= 2 &&
           (p.W + 63) / 64 <= 65535;          // the split pass's grid z extent (x carries B * H)
}

size_t corr_tc_workspace_bytes(const CorrParams &p) {
    return corr_tc_supported(p) ? (size_t)4 * p.B * p.C * p.H * p.W * sizeof(__nv_bfloat16) : 0;
}

// workspace layout: [hi(in1) | lo(in1) | hi(in2) | lo(in2)], each B*C*H*W bf16
static int corr_tc_split(const float *in1, const float *in2, __nv_bfloat16 *w, const CorrParams &p, cudaStream_t st) {
    const size_t per = (size_t)p.B * p.C * p.H * p.W;
    dim3 sgrid(p.B * p.H, 2 * (p.C / 64), (p.W + 63) / 64);
    corr_tc_split_kernel<<<sgrid, 256, 0, st>>>(in1, in2, w, w + per, w + 2 * per, w + 3 * per, p.C, p.H, p.W);
    count_launch();
    return check_launch("correlation(tc split)");
}

static int make_class_map(CUtensorMap *m, const void *base, const CorrParams &p, int box_w, int box_h) {
    const int Hc = p.H / 2, Wc = p.W / 2;
    uint64_t dims[4] = {(uint64_t)p.C, (uint64_t)Wc, (uint64_t)Hc, (uint64_t)p.B * 4};
    uint64_t strides[3] = {(uint64_t)p.C * 2, (uint64_t)Wc * p.C * 2, (uint64_t)Hc * Wc * p.C * 2};
    uint32_t box[4] = {(uint32_t)TC_KB, (uint32_t)box_w, (uint32_t)box_h, 1u};
    return make_tensor_map_bf16_sw128(m, base, 4, dims, strides, box);
}

int corr_forward_tc(const float *in1, const float *in2, float *out, const CorrParams &p, void *workspace,
                    size_t workspace_bytes, cudaStream_t st) {
    const size_t need = corr_tc_workspace_bytes(p);
    if (need == 0) return fail(FN2B200_EUNSUPPORTED, "correlation_forward(tc): configuration not supported");
    if (!workspace || workspace_bytes < need)
        return fail(FN2B200_EINVAL, "correlation_forward(tc): workspace of %zu bytes required, got %zu", need,
                    workspace_bytes);
    if (reinterpret_cast<uintptr_t>(workspace) & 127)
        return fail(FN2B200_EINVAL, "correlation_forward(tc): workspace must be 128-byte aligned");
    const size_t per = (size_t)p.B * p.C * p.H * p.W;
    __nv_bfloat16 *w = static_cast<__nv_bfloat16 *>(workspace);
    __nv_bfloat16 *h1 = w, *l1 = w + per, *h2 = w + 2 * per, *l2 = w + 3 * per;
    int rc = corr_tc_split(in1, in2, w, p, st);
    if (rc) return rc;

    CUtensorMap m1h, m1l, m2h, m2l;
    if ((rc = make_class_map(&m1h, h1, p, TC_TW, TC_TH))) return rc;
    if ((rc = make_class_map(&m1l, l1, p, TC_TW, TC_TH))) return rc;
    if ((rc = make_class_map(&m2h, h2, p, TC_HW, TC_UR))) return rc;
    if ((rc = make_class_map(&m2l, l2, p, TC_HW, TC_UR))) return rc;

    const int Hc = p.H / 2, Wc = p.W / 2;
    const int nxt = (Wc + TC_TW - 1) / TC_TW, nyt = (Hc + TC_TH - 1) / TC_TH;
    const int ntiles = p.B * 4 * nxt * nyt;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int nkb = p.C / TC_KB;
    int bst = 2;
    while (bst < TC_MAXBST && tc_smem_bytes(nkb, bst + 1) <= TC_SMEM_MAX) ++bst;
    const int smem = tc_smem_bytes(nkb, bst);
    cudaError_t e = cudaFuncSetAttribute(corr_fwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return fail((int)e, "correlation_forward(tc): smem attribute (%s)", cudaGetErrorString(e));
    const int grid = ntiles < sms ? ntiles : sms;
    corr_fwd_tc_kernel<<<grid, TC_THREADS, smem, st>>>(m1h, m1l, m2h, m2l, out, p.out_bstride, p.leaky, p.B, p.C, p.H, p.W,
                                                       ntiles, bst);
    count_launch();
    return check_launch("correlation_forward(tc)");
}

template <int NKB>
static int launch_bwd_tc_nkb(const CUtensorMap &m2h, const CUtensorMap &m2l, const CUtensorMap &m1h, const CUtensorMap &m1l,
                             const float *gout, float *gin1, float *gin2, const CorrParams &p, int ntiles, int t_begin,
                             int t_end, int grid, cudaStream_t st) {
    int bst = 2;
    while (bst < TB_MAXBST && tb_smem_bytes(bst + 1) <= TC_SMEM_MAX) ++bst;
    const int smem = tb_smem_bytes(bst);
    cudaError_t e = cudaFuncSetAttribute(corr_bwd_tc_kernel<NKB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return fail((int)e, "correlation_backward(tc): smem attribute (%s)", cudaGetErrorString(e));
    corr_bwd_tc_kernel<NKB><<<grid, TB_THREADS, smem, st>>>(m2h, m2l, m1h, m1l, gout, gin1, gin2, p.B, p.H, p.W, ntiles,
                                                            t_begin, t_end, bst);
    count_launch();
    return check_launch("correlation_backward(tc)");
}

static int launch_bwd_tc(const __nv_bfloat16 *h1, const __nv_bfloat16 *l1, const __nv_bfloat16 *h2, const __nv_bfloat16 *l2,
                         const float *gout, float *gin1, float *gin2, const CorrParams &p, cudaStream_t st) {
    CUtensorMap m1h, m1l, m2h, m2l;
    int rc;
    if ((rc = make_class_map(&m1h, h1, p, TB_GW, TC_UR))) return rc;     // one K group: 12 halo columns x 4 rows
    if ((rc = make_class_map(&m1l, l1, p, TB_GW, TC_UR))) return rc;
    if ((rc = make_class_map(&m2h, h2, p, TB_GW, TC_UR))) return rc;
    if ((rc = make_class_map(&m2l, l2, p, TB_GW, TC_UR))) return rc;
    const int Hc = p.H / 2, Wc = p.W / 2;
    const int nxt = (Wc + TC_TW - 1) / TC_TW, nyt = (Hc + TC_TH - 1) / TC_TH;
    const int ntiles = p.B * 4 * nxt * nyt;
    const int t_begin = gin1 ? 0 : ntiles, t_end = gin2 ? 2 * ntiles : ntiles;
    if (t_end <= t_begin) return 0;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int grid = (t_end - t_begin) < sms ? (t_end - t_begin) : sms;
    switch (p.C / TC_KB) {
    case 1: return launch_bwd_tc_nkb<1>(m2h, m2l, m1h, m1l, gout, gin1, gin2, p, ntiles, t_begin, t_end, grid, st);
    case 2: return launch_bwd_tc_nkb<2>(m2h, m2l, m1h, m1l, gout, gin1, gin2, p, ntiles, t_begin, t_end, grid, st);
    case 3: return launch_bwd_tc_nkb<3>(m2h, m2l, m1h, m1l, gout, gin1, gin2, p, ntiles, t_begin, t_end, grid, st);
    default: return launch_bwd_tc_nkb<4>(m2h, m2l, m1h, m1l, gout, gin1, gin2, p, ntiles, t_begin, t_end, grid, st);
    }
}

// have_split != 0: the workspace already holds the hi/lo copies of (in1, in2) written by
// corr_forward_tc on the same inputs (the autograd wrapper keeps it alive between forward and backward).
int corr_backward_tc(const float *in1, const float *in2, const float *gout, float *gin1, float *gin2,
                     const CorrParams &p, void *workspace, size_t workspace_bytes, int have_split, cudaStream_t st) {
    const size_t need = corr_tc_workspace_bytes(p);
    if (need == 0) return fail(FN2B200_EUNSUPPORTED, "correlation_backward(tc): configuration not supported");
    if (!workspace || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 127))
        return fail(FN2B200_EINVAL, "correlation_backward(tc): 128-byte-aligned workspace of %zu bytes required", need);
    const size_t per = (size_t)p.B * p.C * p.H * p.W;
    __nv_bfloat16 *w = static_cast<__nv_bfloat16 *>(workspace);
    int rc = 0;
    if (!have_split && (rc = corr_tc_split(in1, in2, w, p, st))) return rc;
    return launch_bwd_tc(w, w + per, w + 2 * per, w + 3 * per, gout, gin1, gin2, p, st);
}

}  // namespace fn2

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
// bits); S = hi*hi + hi*lo + lo*hi (3 MMAs, fp32 accumulate in registers), dropped lo*lo ~ 2^-18 relative
// (tc_split_hi: finite x splits into finite halves, the bf16 overflow window included).
//
// Forward pipeline (one persistent CTA per SM, warp-specialised, 384 threads):
//   prepass kernel : NCHW fp32 -> [n][class][yc][xc][c] bf16 hi / lo (channels contiguous = K-major)
//   warps 8-11     : TMA producer (one lane of warp 8):
//                                  f1 tile  -> smem A [hi|lo][C/64][128 rows x 128 B]  (resident for the tile's units)
//                                  f2 units -> smem B ring, one slot = hi OR lo of a unit x 64 channels
//                    [144 rows x 128 B] = one 18-KB box, 128-byte swizzle; halo outside the image = TMA
//                    out-of-bounds zero fill = the layer's zero padding
//   warps 0-7      : two warpgroups, ping-pong by unit: the k-th unit of a CTA is computed by warpgroup k & 1 for all
//                    128 tile pixels, wgmma m64n144k16 per 64-pixel half (hi slot: hi*hi and lo*hi, lo slot: hi*lo,
//                    4 k-steps each) into two fp32 register accumulators; each warp then moves the band entries of
//                    its two fragment rows, scaled by 1/C, through a private shared-memory buffer to
//                    out[n][(tj,ti)][y][x], 16 pixels x 2 displacement planes per store instruction, while the other
//                    warpgroup's wgmmas for the next unit run
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
constexpr int TC_NBAR = 2 * TC_MAXKB + 2 * TC_MAXBST + 2;    // A full / empty, B full / empty, the 2 turn barriers
constexpr int TC_SMEM_MAX = 232448;            // 227 KB opt-in limit per CTA (sm_90)
// Forward epilogue staging: each consumer warp transposes its band through a private buffer [ti][px] of its 16 tile
// pixels, one displacement row ti every TC_SPITCH floats.  The pitch makes the fill conflict-free: for one
// accumulator register, lane (pxa, q) writes float (2q - pxa + k) * 20 + pxa, and 8q + 13 pxa is distinct mod 32 for
// all 32 lanes (pitch 16 would put the 4 lanes of a pixel in one bank).
constexpr int TC_SPITCH = 20;
constexpr int TC_SBUF = (TC_DS - 1) * TC_SPITCH + TC_TW;     // floats per warp
// A_hi and A_lo blocks, then bst ring slots of one 18-KB box each, the mbarriers, the 8 staging buffers (+ 1 KB for
// the 1024-byte alignment of the swizzle atoms)
__host__ __device__ constexpr int tc_smem_bytes(int nkb, int bst) {
    return 2 * nkb * TC_ABLK + bst * TC_BBLK + TC_NBAR * 8 + 8 * TC_SBUF * 4 + 1024;
}

// The hi half of the split x = hi + lo: rn_bf16(x), saturated to the largest finite bf16.  A finite x in the bf16
// overflow window (|x| in [0x7F7F8000, 0x7F7FFFFF]) would round to a bf16 infinity and make lo = -inf; saturated, lo =
// rn(x - hi) stays finite and |x - hi - lo| <= 2^-16 |x| still holds.  ±inf splits into (±max, ±inf) and NaN into NaN.
// One cvt.satfinite replaces the cvt.rn: a window test beside it added six instructions per gradOutput value to the
// backward's builder and slowed corr_bwd_tc_kernel by ~6 %.
__device__ __forceinline__ __nv_bfloat16 tc_split_hi(float x) {
    unsigned short h;
    asm("cvt.rn.satfinite.bf16.f32 %0, %1;" : "=h"(h) : "f"(x));
    return __ushort_as_bfloat16(h);
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
            const __nv_bfloat16 h0 = tc_split_hi(v0), h1 = tc_split_hi(v1);
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

// Ring slots [b, b + n) that the calling warpgroup does not read (the forward's A blocks of a segment without a unit of
// the warpgroup, as a ring of nkb slots): wait for each fill, then release it.  Releasing a slot before its fill has landed
// would complete the previous phase, and a slot refilled before this warpgroup saw its current phase would make the
// parity of its next wait on the slot ambiguous.
__device__ __forceinline__ void tc_skip_slots(uint64_t *full, uint64_t *empty, uint32_t b, int n, int bst) {
    for (int i = 0; i < n; ++i, ++b) {
        const int s = b % bst;
        mbar_wait(&full[s], (b / bst) & 1);
        mbar_arrive(&empty[s]);
    }
}

// Warps 0-7: two consumer warpgroups that take the CTA's units in turn (ping-pong): the k-th unit the CTA runs belongs
// to warpgroup k & 1, which keeps the unit's two m64 x n144 accumulators (tile rows 0-3 and 4-7) in registers and then
// stores the unit's band while the other warpgroup's wgmmas for unit k + 1 run.  Warps 8-11: the producer warpgroup, of
// which one lane of warp 8 issues the TMA loads.  Register budgets (setmaxnreg) fill the 64 K register file: the two
// accumulators alone are 144 registers, more than ptxas grants a thread of a 288-thread kernel without spilling.
constexpr int TC_CONSUMERS = 256;
constexpr int TC_THREADS = TC_CONSUMERS + 128;
constexpr int TC_REG_MMA = 232, TC_REG_PROD = 40;
static_assert(128 * (2 * TC_REG_MMA + TC_REG_PROD) <= 65536, "register budgets exceed the register file");
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
    uint64_t *turn = b_empty + TC_MAXBST;                     // [warpgroup]: the previous unit's wgmmas are issued
    float *stage = reinterpret_cast<float *>(bars + TC_NBAR);  // [consumer warp][TC_SBUF]

    if (tid == 0) {
        prefetch_tensormap(&m1h); prefetch_tensormap(&m1l);
        prefetch_tensormap(&m2h); prefetch_tensormap(&m2l);
        // A: both warpgroups arrive once per segment; B: a slot has one reader, the warpgroup of its unit
        for (int i = 0; i < TC_MAXKB; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], TC_CONSUMERS); }
        for (int i = 0; i < TC_MAXBST; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], TC_CONSUMERS / 2); }
        for (int i = 0; i < 2; ++i) mbar_init(&turn[i], TC_CONSUMERS / 2);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp >= TC_CONSUMERS / 32) {
        // ===================== TMA producer =====================
        setmaxnreg_dec<TC_REG_PROD>();
        if (warp == TC_CONSUMERS / 32 && lane == 0) {
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
        setmaxnreg_inc<TC_REG_MMA>();
        const int wg = warp >> 2, wq = warp & 3;
        // accumulator fragment of half h: rows 16 wq + lane / 4 (+ 8) of the half = tile row 4 h + wq, columns pxa (+ 8)
        const int pxa = lane >> 2, q = lane & 3;
        // store role: tile pixel sx of the fragment row, displacement column ti = t + sd of a store pair
        const int sx = lane & 15, sd = lane >> 4;
        float *sbuf = stage + warp * TC_SBUF;
        // 1/(k*k*C): exact for power-of-two C (FlowNetC: 256) -> bit-identical to the reference's divide; otherwise
        // within 1 ulp.
        const float inv_nelems = 1.0f / (float)C;
        const long plane = (long)H * W;
        const bool act = leaky != 1.f;
        // Barrier phases.  Both warpgroups walk all segments and count every unit (k) and ring slot (bcount) of the CTA
        // in the producer's order; each waits on and releases only the slots of its own units.  A wait for fill P of a
        // slot is unambiguous only if fill P - 1 has landed (otherwise the slot's last completed phase, P - 2, has the
        // parity waited for), and fill P - 1 may belong to the other warpgroup's unit.  So unit k starts only after the
        // warpgroup of unit k - 1 has passed all of that unit's b_full waits: it then arrives on turn[k & 1], and by
        // induction every fill of the units before k has landed.  turn[w] completes its j-th phase when unit 2 j + 1 - w
        // has been issued, so unit k waits for phase ((k + 1) >> 1) - 1 of turn[k & 1]; unit 0 waits for phase -1, which
        // a fresh barrier reports complete.  The turns alternate, so neither turn barrier can run a phase ahead of its
        // waiter.  A fill P + 1 needs the reader's release of fill P, so a slot cannot run ahead of its reader either.
        // A is resident for a segment and read by both warpgroups: each waits for a_full and arrives on a_empty once per
        // segment and k-block, after its last unit of the segment, or at once if it has no unit there (a one-unit
        // segment of the last round), so that its wait in the next segment again sees the phase before.
        uint32_t bcount = 0, k = 0;
        int it = 0;
        TcSeg sg;
        for (int tn = blockIdx.x, w = w0; tc_next_seg(tn, w, full, w1, sg); ++it) {
            const int ua = sg.ua, ub = sg.ub;
            const TcTile T = tc_decode(sg.t, nxt, nyt);
            const int xc = T.xc0 + sx;
            const int uf = ua + (int)((k ^ (uint32_t)wg) & 1u);       // this warpgroup's first unit of the segment
            if (uf >= ub) tc_skip_slots(a_full, a_empty, (uint32_t)it * nkb, nkb, nkb);
            for (int u = uf; u < ub; u += 2) {
                const uint32_t ku = k + (uint32_t)(u - ua);
                uint32_t b = bcount + (uint32_t)(u - ua) * 2 * nkb;
                mbar_wait(&turn[wg], (((ku + 1) >> 1) & 1) ^ 1);
                float acc[2][TC_N / 2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int i = 0; i < TC_N / 2; ++i) acc[h][i] = 0.f;
                    wgmma_fence_operands(acc[h]);
                }
                // the unit's wgmmas into the halves h with live[h]; called with constants, so that no wgmma sits on a
                // path of its own (ptxas would serialise them all)
                auto mma = [&](const bool live0, const bool live1) {
                    const bool live[2] = {live0, live1};
                    int prev = -1, prev_a = -1;            // ring slot (and A block) read by the wgmma group in flight
                    for (int kb = 0; kb < nkb; ++kb) {
                        if (u == uf) mbar_wait(&a_full[kb], it & 1);
                        // A descriptors of the two halves (tile rows 0-3, 4-7): hi, then lo
                        uint64_t da[2][2];
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            da[0][h] = wgmma_desc_k_sw128(smem_u32(sA + kb * TC_ABLK + h * (TC_ABLK / 2)));
                            da[1][h] = wgmma_desc_k_sw128(smem_u32(sAlo + kb * TC_ABLK + h * (TC_ABLK / 2)));
                        }
#pragma unroll
                        for (int hl = 0; hl < 2; ++hl, ++b) {
                            const int s = b % bst;
                            mbar_wait(&b_full[s], (b / bst) & 1);
                            const uint64_t bd = wgmma_desc_k_sw128(smem_u32(sB + s * TC_BBLK));
                            wgmma_fence();
                            // each accumulator: hi x hi | hi x lo, then (hi slot) lo x hi, k-step by k-step
#pragma unroll
                            for (int ks = 0; ks < TC_KB / 16; ++ks) {
#pragma unroll
                                for (int lo = 0; lo <= (hl == 0); ++lo)
#pragma unroll
                                    for (int h = 0; h < 2; ++h)
                                        if (live[h]) wgmma_m64n144k16_k(acc[h], da[lo][h] + 2 * ks, bd + 2 * ks);
                            }
                            wgmma_commit();
                            if (hl == 1 && kb == nkb - 1) mbar_arrive(&turn[wg ^ 1]);   // unit k + 1 may start
                            wgmma_wait<1>();
                            if (prev >= 0) {
                                mbar_arrive(&b_empty[prev]);
                                if (prev_a >= 0) mbar_arrive(&a_empty[prev_a]);
                            }
                            prev = s;
                            prev_a = (hl == 1 && u + 2 >= ub) ? kb : -1;       // A block free for the next segment
                        }
                    }
                    wgmma_wait<0>();
                    wgmma_fence_operands(acc[0]);
                    wgmma_fence_operands(acc[1]);
                    mbar_arrive(&b_empty[prev]);
                    if (prev_a >= 0) mbar_arrive(&a_empty[prev_a]);
                };
                // unit 0 only meets tile rows 0-3 and unit 6 only tile rows 4-7: the other half's products would only
                // reach out-of-band columns, which are never stored
                if (u == 0) mma(true, false);
                else if (u == TC_NU - 1) mma(false, true);
                else mma(true, true);
                // accumulator column c = hrl * 36 + qx (halo row hrl of the unit, halo column qx) of tile pixel
                // (py_t, px) is displacement (tj, ti) = (u * 4 + hrl - py_t, qx - px) - (10, 10), if inside the band.
                // Per halo row, tj is the same for the whole warp (its fragment rows of a half are one tile row), and
                // each of its 16 pixels has exactly 21 in-band columns among the row's 36, so the warp's buffer [ti][px]
                // is wholly rewritten by each pass.  Storing from the buffer writes 16 consecutive pixels of 2
                // displacement planes per instruction (2 lines), where storing from the fragment wrote one value
                // per lane to up to 32 different planes.  A dead half has no displacement row in the band.
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int py_t = 4 * h + wq, yc = T.yc0 + py_t;
                    const bool ok = (yc < Hc) && (xc < Wc);
                    float *ob = out + (long)T.n * out_bstride + (long)(2 * yc + T.py) * W + (2 * xc + T.px);
                    const int tjb = u * TC_UR - py_t;
#pragma unroll
                    for (int hrl = 0; hrl < TC_UR; ++hrl) {
                        const int tj = tjb + hrl;
                        if ((unsigned)tj >= (unsigned)TC_DS) continue;     // warp-uniform
#pragma unroll
                        for (int i = TC_HW * hrl / 8; i <= (TC_HW * hrl + TC_HW - 1) / 8; ++i)
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const int x = pxa + 8 * (j >> 1);
                                const int ti = 8 * i + 2 * q + (j & 1) - TC_HW * hrl - x;
                                if ((unsigned)ti < (unsigned)TC_DS) {           // implies the column lies in halo row hrl
                                    float v = acc[h][4 * i + j] * inv_nelems;
                                    if (act) v = v > 0.f ? v : v * leaky;      // fused nn.LeakyReLU (FlowNetC.py:87), warp-uniform
                                    sbuf[ti * TC_SPITCH + x] = v;
                                }
                            }
                        __syncwarp();
                        float *o = ob + (long)(tj * TC_DS + sd) * plane;
#pragma unroll
                        for (int t = 0; t < TC_DS; t += 2)
                            if (ok && t + sd < TC_DS) __stcs(o + (long)t * plane, sbuf[(t + sd) * TC_SPITCH + sx]);
                        __syncwarp();                                   // read before the next pass overwrites
                    }
                }
            }
            k += (uint32_t)(ub - ua);
            bcount += (uint32_t)(ub - ua) * 2 * nkb;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Backward on tensor cores: gradInput1 tiles (other = input2) and gradInput2 tiles (other = input1).
//
//   gI1[c, p] = 1/C sum_q G1[p, q] f2[c, q],   G1[p, q] = gO[(q - p), p]          (|q - p| <= 10)
//   gI2[c, q] = 1/C sum_p G2[q, p] f1[c, p],   G2[q, p] = gO[(q - p), p]
// per parity class: D[128 tile px][C] += A[128][144] * B[144 halo px][C] over the halo-row units, accumulated in
// registers (warpgroup wg: tile pixels [64 wg, 64 wg + 64), an m64 x nC fragment) for the whole tile.
//   A = the banded gradOutput matrix, built per unit by a builder warpgroup straight from the fp32 gradOutput planes
//       (bf16 hi/lo split on the fly) into an MN-major SW128 layout [k][64 pixels], two buffers per MMA warpgroup
//       handed over through mbarriers (a_full: built, a_empty: the wgmmas that read it are complete), so that the
//       builders load and build up to two units ahead of the MMAs and across the MMA warpgroups' gradient stores;
//   B = the other input's halo chunk from the prepass copy ([pixel][channel] bf16 = MN-major operand), one ring slot =
//       hi OR lo of a K-group (48 halo pixels) x all channel blocks;
//   3 products (hi*hi, lo*hi | hi*lo) per k-step, N = C per instruction (two n128 halves at C = 256).
// One builder thread per tile pixel: all 4 halo rows x 21 displacements of the unit.  Loads stay coalesced (lanes =
// pixels, one displacement plane per instruction); the band positions a pixel writes are the same for every unit, so
// the zero columns of A are written ONCE at kernel start.
// Epilogue: each MMA warp stores its tile row's 16 pixels x C channels, scaled by 1/C, 16 pixels x 2 channel planes per
// store instruction (a register swap between lane pairs, no shared memory).  Each warpgroup releases only the
// ring slots it reads, so one warpgroup's stores run under the other's wgmmas (phases: at the MMA warpgroups' loop).
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
// B ring full / empty, A full [warpgroup][buffer], A empty [warpgroup][buffer], then the 2 turn barriers
constexpr int TB_NBAR = 2 * TB_MAXBST + 2 * 2 * TB_NAST + 2;
// B staging: the unit's 144 K indices in 3 groups of 48 (12 halo columns x 4 rows); one ring slot = the hi (or the lo)
// copy of one group x ALL channel blocks = up to 4 boxes of 6 KB, so one k-step covers N = C columns.
constexpr int TB_NG = 3, TB_GW = TC_HW / TB_NG, TB_GK = TC_UR * TB_GW;   // 3 groups, 12 columns, 48 K
constexpr int TB_GBLK = TB_GK * 128;               // 6144 B: one 64-channel block of a group's rows
constexpr int TB_BSTAGE = 4 * TB_GBLK;             // 24576 B: [<= 4 channel blocks][48 rows x 128 B]
__host__ __device__ constexpr uint32_t tb_kindex(uint32_t hrl, uint32_t qx) {
    return (qx / TB_GW) * TB_GK + hrl * TB_GW + (qx % TB_GW);
}
// A offset of halo row h from that of halo row 0: + 12 h k-rows, and an odd h flips bit 2 of k & 7 (the swizzle)
__host__ __device__ constexpr uint32_t tb_row_offset(uint32_t ao0, uint32_t h) {
    return (ao0 ^ ((h & 1u) << 6)) + h * TB_GW * 128u;
}
__host__ __device__ constexpr bool tb_row_offsets_hold() {
    for (uint32_t p = 0; p < 64; ++p)
        for (uint32_t x = 0; x < TC_HW; ++x)
            for (uint32_t h = 0; h < TC_UR; ++h)
                if (tb_a_offset(p, tb_kindex(h, x)) != tb_row_offset(tb_a_offset(p, tb_kindex(0, x)), h)) return false;
    return true;
}
static_assert(tb_row_offsets_hold(), "tb_row_offset must match tb_a_offset");
// warps 0-7: two MMA warpgroups (wgmma, epilogue); warps 8-11: the builder warpgroup (A); warps 12-15: the producer
// warpgroup, of which warp 12 issues the TMA loads.  Register budgets (setmaxnreg) fill the 64 K register file: the
// m64 x n256 accumulator alone is 128 registers, a builder thread holds its unit's 84 gradOutput values.
constexpr int TB_THREADS = TC_CONSUMERS + 256;
constexpr int TB_REG_MMA = 168, TB_REG_BUILD = 152, TB_REG_PROD = 24;
static_assert(128 * (2 * TB_REG_MMA + TB_REG_BUILD + TB_REG_PROD) <= 65536, "register budgets exceed the register file");
__host__ __device__ constexpr int tb_smem_bytes(int bst) {
    return TB_SMEM_A + bst * TB_BSTAGE + TB_NBAR * 8 + 1024;
}

template <int NKB>
__device__ __forceinline__ void wgmma_bwd(float (&d)[NKB * 32], uint64_t da, uint64_t db);
template <> __device__ __forceinline__ void wgmma_bwd<1>(float (&d)[32], uint64_t da, uint64_t db) { wgmma_m64n64k16_mn(d, da, db); }
template <> __device__ __forceinline__ void wgmma_bwd<2>(float (&d)[64], uint64_t da, uint64_t db) { wgmma_m64n128k16_mn(d, da, db); }
template <> __device__ __forceinline__ void wgmma_bwd<3>(float (&d)[96], uint64_t da, uint64_t db) { wgmma_m64n192k16_mn(d, da, db); }
// C = 256: two n128 halves (channel blocks 0-1, then 2-3).  ptxas places the operands of one instruction within the
// kernel-wide register limit, 128 at 512 threads, which an n256 accumulator alone fills.  Each accumulator element still
// receives the same k16 products in the same order.
template <> __device__ __forceinline__ void wgmma_bwd<4>(float (&d)[128], uint64_t da, uint64_t db) {
    wgmma_m64n128k16_mn(*reinterpret_cast<float (*)[64]>(&d[0]), da, db);
    wgmma_m64n128k16_mn(*reinterpret_cast<float (*)[64]>(&d[64]), da, db + ((2 * TB_GBLK) >> 4));
}

// Both gradients in ONE launch: global tiles [t_begin, t_end) of [0, 2 ntiles).  One gradient only: tile g < ntiles
// is tile g of gradInput1 (B = input2's halo, maps m2h / m2l), tile g >= ntiles is tile g - ntiles of gradInput2
// (B = input1's halo); both: g = 2 tile + (0 = gradInput1, 1 = gradInput2).
// CAT (fn2b200_correlation_backward_cat): sample n's gradOutput planes start at gout + n * gplanes planes (a channel
// range of a concat gradient), and with act != NULL every gradOutput value g is replaced by (act > 0 ? g : g * slope),
// act read at g's offset, before the bf16 split.  !CAT: gplanes = 441, no activation (act, slope unused).
template <int NKB, bool CAT>
__global__ void __launch_bounds__(TB_THREADS, 1)
corr_bwd_tc_kernel(const __grid_constant__ CUtensorMap m2h, const __grid_constant__ CUtensorMap m2l,
                   const __grid_constant__ CUtensorMap m1h, const __grid_constant__ CUtensorMap m1l,
                   const float *__restrict__ gout, const float *__restrict__ act, int gplanes, float slope,
                   float *__restrict__ gin1, float *__restrict__ gin2, int B,
                   int H, int W, int ntiles, int t_begin, int t_end, int bst) {
    constexpr int C = NKB * TC_KB;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    unsigned char *sA = smem;                          // [warpgroup][buffer][hi | lo][144 k x 128 B]
    unsigned char *sB = smem + TB_SMEM_A;              // [slot][channel block][48 rows x 128 B] (SW128, MN-major)
    uint64_t *bars = reinterpret_cast<uint64_t *>(sB + bst * TB_BSTAGE);
    uint64_t *b_full = bars, *b_empty = bars + TB_MAXBST;
    uint64_t *a_full = bars + 2 * TB_MAXBST, *a_empty = a_full + 2 * TB_NAST;
    uint64_t *turn = a_empty + 2 * TB_NAST;             // [warpgroup]: the other warpgroup has passed its solo unit's waits

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
        for (int i = 0; i < 2 * TB_NAST; ++i) { mbar_init(&a_full[i], 64); mbar_init(&a_empty[i], 128); }
        for (int i = 0; i < 2; ++i) mbar_init(&turn[i], 128);
        fence_barrier_init();
    }
    // columns of A outside a pixel row's band are zero for every unit: written once, here
    for (int i = tid; i < TB_SMEM_A / 16; i += TB_THREADS) reinterpret_cast<uint4 *>(sA)[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async();
    __syncthreads();

    if (warp >= TC_CONSUMERS / 32 + 4) {
        // ===================== TMA producer: the other input's halo chunks =====================
        setmaxnreg_dec<TB_REG_PROD>();
        if (warp == TC_CONSUMERS / 32 + 4 && lane == 0) {
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

    // warpgroup wg's pixel rows 4 wg .. 4 wg + 3 only meet units wg .. wg + 5: the other unit's A would be all zero.
    // Builders and MMA warpgroups walk the same tiles and units, so the A buffer of a warpgroup's ucount-th unit is
    // ucount & 1, in its (ucount >> 1)-th use.
    if (warp >= TC_CONSUMERS / 32) {
        // ===================== builders: the banded gradOutput matrix A =====================
        setmaxnreg_inc<TB_REG_BUILD>();
        // builder warp bw serves MMA warpgroup wg = bw / 2 and covers 4 tile rows x 8 pixels of it (its 32 two-byte
        // stores of one (halo row, displacement) hit 32 different banks); thread = pixel bp of the warpgroup's 64
        const int bw = warp - TC_CONSUMERS / 32, wg = bw >> 1;
        const int bp = (lane >> 3) * TC_TW + (bw & 1) * 8 + (lane & 7);
        const int bpy = 4 * wg + (bp >> 4), bpx = bp & 15;
        const int iplane = (int)plane;         // all tensors < 2^31 elements (checked by the C ABI)
        unsigned char *aw = sA + wg * TB_NAST * TB_ASTG;
        uint64_t *full = a_full + wg * TB_NAST, *empty = a_empty + wg * TB_NAST;
        // A offsets of halo row 0 (unit- and tile-invariant, < 2^16), two per register: displacement j in bits
        // [16 (j & 1), 16 (j & 1) + 16) of ao[j / 2]
        uint32_t ao[(TC_DS + 1) / 2];
#pragma unroll
        for (int j = 0; j < TC_DS; j += 2)
            ao[j / 2] = tb_a_offset(bp, tb_kindex(0, bpx + j)) | (j + 1 < TC_DS ? tb_a_offset(bp, tb_kindex(0, bpx + j + 1)) << 16 : 0u);
        uint32_t ucount = 0;
        for (int g = t_begin + blockIdx.x; g < t_end; g += gridDim.x) {
            const bool second = both ? (g & 1) : (g >= ntiles);       // gradInput2 tile (block-uniform)
            const TcTile T = tc_decode(both ? (g >> 1) : (second ? g - ntiles : g), nxt, nyt);
            const int nbase = T.n * (CAT ? gplanes : TC_DS * TC_DS);
            // Per-tile address set-up (element offsets fit in 32 bits): the band row of the tile's halo row r (unit
            // r / 4) starts at off + r * rstep; consecutive displacements are `step` apart; the row is loaded when
            // tj = r - bpy is a displacement and source row ys0 + r * ystep lies inside the image.
            int off, rstep, step, ys0, ystep;
            uint32_t colmask = (1u << TC_DS) - 1u;             // displacements to load (gradInput2: source columns inside the image)
            {
                const int yc = T.yc0 + bpy, xc = T.xc0 + bpx;
                if (!second) {
                    ys0 = ((yc < Hc) && (xc < Wc)) ? 0 : Hc;       // gO at the output pixel itself
                    ystep = 0;
                    off = ((nbase - bpy * TC_DS) * H + (2 * yc + T.py)) * W + (2 * xc + T.px);
                    step = iplane;                                 // next ti -> next plane
                    rstep = TC_DS * iplane;                        // next halo row -> tj + 1
                } else {
                    ys0 = T.yc0 - TC_DR;                           // source pixel row of halo row 0
                    ystep = 1;
                    const int xs0 = T.xc0 - TC_DR + bpx;           // source column for j = 0
                    off = ((nbase + (TC_DS - 1 + bpy) * TC_DS + (TC_DS - 1)) * H + (2 * ys0 + T.py)) * W + (2 * xs0 + T.px);
                    step = 2 - iplane;                             // j -> j+1: -1 plane, +2 in x
                    rstep = 2 * W - TC_DS * iplane;                // next halo row: tj + 1 -> -21 planes, source row + 2
                    colmask = 0;
#pragma unroll
                    for (int j = 0; j < TC_DS; ++j)
                        if ((unsigned)(xs0 + j) < (unsigned)Wc) colmask |= 1u << j;
                }
            }
            for (int u = wg; u < TC_NU - 1 + wg; ++u, ++ucount) {
                bool row_ok[TC_UR];
#pragma unroll
                for (int h = 0; h < TC_UR; ++h) {
                    const int r = u * TC_UR + h;
                    row_ok[h] = ((unsigned)(r - bpy) < (unsigned)TC_DS) && ((unsigned)(ys0 + r * ystep) < (unsigned)Hc);
                }
                // CAT with activation: the activations are folded to a bit per displacement (act > 0) before the
                // gradOutput loads are issued
                uint32_t pos[TC_UR];
#pragma unroll
                for (int h = 0; h < TC_UR; ++h) pos[h] = ~0u;
                if (CAT && act) {
                    // all 84 loads issue before the first compare: one round trip per unit, not one per halo row
                    float a[TC_UR][TC_DS];
#pragma unroll
                    for (int h = 0; h < TC_UR; ++h) {
                        const int base = off + (u * TC_UR + h) * rstep;    // only dereferenced under `ok`
#pragma unroll
                        for (int j = 0; j < TC_DS; ++j) {       // predicated, not branched: all loads in flight
                            const bool ok = row_ok[h] && ((colmask >> j) & 1u);
                            a[h][j] = ok ? __ldg(act + (base + j * step)) : 1.f;
                        }
                    }
#pragma unroll
                    for (int h = 0; h < TC_UR; ++h) {
                        pos[h] = 0u;
#pragma unroll
                        for (int j = 0; j < TC_DS; ++j) pos[h] |= a[h][j] > 0.f ? 1u << j : 0u;
                    }
                }
                // the unit's 84 gradOutput loads go out before the wait for the buffer
                float v[TC_UR][TC_DS];
#pragma unroll
                for (int h = 0; h < TC_UR; ++h) {
                    const int base = off + (u * TC_UR + h) * rstep;
#pragma unroll
                    for (int j = 0; j < TC_DS; ++j) {
                        const bool ok = row_ok[h] && ((colmask >> j) & 1u);
                        v[h][j] = ok ? __ldg(gout + (base + j * step)) : 0.f;
                        if (CAT) v[h][j] = ((pos[h] >> j) & 1u) ? v[h][j] : v[h][j] * slope;
                    }
                }
                const int ab = ucount & 1;
                mbar_wait(&empty[ab], ((ucount >> 1) & 1) ^ 1);   // the wgmmas that read this buffer are complete
                unsigned char *ah = aw + ab * TB_ASTG, *al = ah + TB_AHL;
#pragma unroll
                for (int h = 0; h < TC_UR; ++h)
#pragma unroll
                    for (int j = 0; j < TC_DS; ++j) {
                        const __nv_bfloat16 hv = tc_split_hi(v[h][j]);
                        const __nv_bfloat16 lv = __float2bfloat16_rn(v[h][j] - __bfloat162float(hv));
                        const uint32_t o = tb_row_offset((ao[j / 2] >> (16 * (j & 1))) & 0xFFFFu, h);
                        *reinterpret_cast<unsigned short *>(ah + o) = __bfloat16_as_ushort(hv);
                        *reinterpret_cast<unsigned short *>(al + o) = __bfloat16_as_ushort(lv);
                    }
                fence_proxy_async();                               // generic-proxy writes -> visible to the tensor core
                mbar_arrive(&full[ab]);
            }
        }
        return;
    }

    // ===================== MMA warpgroups: wgmma + epilogue =====================
    setmaxnreg_inc<TB_REG_MMA>();
    const int wg = warp >> 2, wq = warp & 3;
    // accumulator fragment role: rows 16 wq + lane / 4 (+ 8) of the warpgroup
    const int py_t = 4 * wg + wq, pxa = lane >> 2, q = lane & 3;
    const uint32_t aw32 = smem_u32(sA + wg * TB_NAST * TB_ASTG);
    uint64_t *full = a_full + wg * TB_NAST, *empty = a_empty + wg * TB_NAST;
    const float inv_nelems = 1.0f / (float)C;
    // Barrier phases.  Units 1-5 of a tile are read by both warpgroups; unit 0 only by warpgroup 0 and unit 6 only by
    // warpgroup 1.  That is each warpgroup's solo unit su, whose ring slots it releases alone, with 2 arrivals per thread.
    // Both warpgroups count every ring slot (bcount) in the producer's order.  A wait for fill P of a slot is
    // unambiguous only if fill P - 1 has landed (otherwise the slot's last completed phase, P - 2, has the parity
    // waited for), and a warpgroup does not see the fills of the other one's solo unit.  So each waits, before its
    // first unit of a tile, until the other has passed all its b_full waits of the solo unit just before: warpgroup 1
    // before unit 1 of tile it for warpgroup 0's unit 0 of tile it, warpgroup 0 before unit 0 of tile it for
    // warpgroup 1's unit 6 of tile it - 1.  turn[w] completes its j-th phase when the other warpgroup has passed the
    // waits of its j-th solo unit, so warpgroup 1 waits for phase it of turn[1] and warpgroup 0 for phase it - 1 of
    // turn[0]; the first tile's phase -1 is one a fresh barrier reports complete.  Neither turn barrier can run a phase
    // ahead of its waiter: its next phase needs the other warpgroup to pass its own turn wait, which needs this
    // warpgroup's arrival after the wait.  A fill P + 1 needs the readers' release of fill P, so a slot cannot run
    // ahead of a reader either.  These waits are the only coupling, so warpgroup 0's gradient stores run under
    // warpgroup 1's unit 6, and warpgroup 1's under warpgroup 0's unit 0 of the next tile and the start of its unit 1.
    const int su = wg * (TC_NU - 1);
    uint32_t bcount = 0, ucount = 0, it = 0;
    for (int g = t_begin + blockIdx.x; g < t_end; g += gridDim.x, ++it) {
        const bool second = both ? (g & 1) : (g >= ntiles);           // gradInput2 tile (block-uniform)
        const TcTile T = tc_decode(both ? (g >> 1) : (second ? g - ntiles : g), nxt, nyt);
        float acc[C / 2];
#pragma unroll
        for (int i = 0; i < C / 2; ++i) acc[i] = 0.f;
        wgmma_fence_operands(acc);
        int prev = -1, prev_a = -1;                            // ring slot (and A buffer) read by the wgmma group in flight
        uint32_t prev_n = 1;                                   // arrivals that release it: 2 in the solo unit
        if (wg == 1) bcount += 2 * TB_NG;                      // unit 0: warpgroup 0's alone
        for (int u = wg; u < TC_NU - 1 + wg; ++u, ++ucount) {
            const int ab = ucount & 1;
            mbar_wait(&full[ab], (ucount >> 1) & 1);
            if (u == wg) mbar_wait(&turn[wg], (it & 1) ^ (uint32_t)wg ^ 1u);
            const uint32_t ah32 = aw32 + ab * TB_ASTG, al32 = ah32 + TB_AHL;
            for (int gr = 0; gr < TB_NG; ++gr)
#pragma unroll
                for (int hl = 0; hl < 2; ++hl, ++bcount) {
                    const int s = bcount % bst;
                    mbar_wait(&b_full[s], (bcount / bst) & 1);
                    if (u == su && gr == TB_NG - 1 && hl == 1) mbar_arrive(&turn[wg ^ 1]);   // the solo unit has landed
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
                    if (prev >= 0) {
                        mbar_arrive_cnt(&b_empty[prev], prev_n);
                        if (prev_a >= 0) mbar_arrive(&empty[prev_a]);
                    }
                    prev = s;
                    prev_n = u == su ? 2u : 1u;
                    prev_a = (gr == TB_NG - 1 && hl == 1) ? ab : -1;   // the unit's last read of its A buffer
                }
        }
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
        mbar_arrive_cnt(&b_empty[prev], prev_n);
        mbar_arrive(&empty[prev_a]);
        if (wg == 0) bcount += 2 * TB_NG;                      // unit 6: warpgroup 1's alone
        // epilogue: fragment rows = tile pixels (py_t, pxa) and (py_t, pxa + 8), columns = channels 8 i + 2 q (+ 1).  The
        // lane pair q = 2 m, 2 m + 1 swaps halves (one shfl.xor per channel parity), so that lane q holds pixel
        // sx = pxa + 8 (q & 1) of the four channels 8 i + 4 m + k; each store instruction then writes 16 consecutive
        // tile pixels of 2 channel planes (2 lines), where storing the fragment as it is wrote 8 pixels of 4 planes.
        const int sx = pxa + 8 * (q & 1), yc = T.yc0 + py_t, xc = T.xc0 + sx;
        const bool ok = (yc < Hc) && (xc < Wc), odd = q & 1;
        float *o = (second ? gin2 : gin1) + ((long)T.n * C + 4 * (q >> 1)) * plane + (long)(2 * yc + T.py) * W + (2 * xc + T.px);
#pragma unroll
        for (int i = 0; i < C / 8; ++i) {
            const float *a = acc + 4 * i;          // [pixel half][channel parity] of channels 8 i + 2 q (+ 1)
            const float r0 = __shfl_xor_sync(0xffffffffu, odd ? a[0] : a[2], 1);
            const float r1 = __shfl_xor_sync(0xffffffffu, odd ? a[1] : a[3], 1);
            const float v[4] = {odd ? r0 : a[0], odd ? r1 : a[1], odd ? a[2] : r0, odd ? a[3] : r1};
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (ok) __stcs(o + (long)(8 * i + k) * plane, v[k] * inv_nelems);
        }
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

template <int NKB, bool CAT>
static int launch_bwd_tc_nkb(const CUtensorMap &m2h, const CUtensorMap &m2l, const CUtensorMap &m1h, const CUtensorMap &m1l,
                             const float *gout, float *gin1, float *gin2, const CorrParams &p, int ntiles, int t_begin,
                             int t_end, int grid, cudaStream_t st) {
    int bst = 2;
    while (bst < TB_MAXBST && tb_smem_bytes(bst + 1) <= TC_SMEM_MAX) ++bst;
    const int smem = tb_smem_bytes(bst);
    cudaError_t e = cudaFuncSetAttribute(corr_bwd_tc_kernel<NKB, CAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return fail((int)e, "correlation_backward(tc): smem attribute (%s)", cudaGetErrorString(e));
    // gradOutput planes per sample: the 2^31-element check on the gradient buffer keeps every offset in 32 bits
    const int gplanes = (int)(p.g_bstride / ((long)p.oH * p.oW));
    corr_bwd_tc_kernel<NKB, CAT><<<grid, TB_THREADS, smem, st>>>(m2h, m2l, m1h, m1l, gout, p.act, gplanes, p.leaky, gin1,
                                                                 gin2, p.B, p.H, p.W, ntiles, t_begin, t_end, bst);
    count_launch();
    return check_launch("correlation_backward(tc)");
}

template <bool CAT>
static int launch_bwd_tc_c(const CUtensorMap &m2h, const CUtensorMap &m2l, const CUtensorMap &m1h, const CUtensorMap &m1l,
                           const float *gout, float *gin1, float *gin2, const CorrParams &p, int ntiles, int t_begin,
                           int t_end, int grid, cudaStream_t st) {
    switch (p.C / TC_KB) {
    case 1: return launch_bwd_tc_nkb<1, CAT>(m2h, m2l, m1h, m1l, gout, gin1, gin2, p, ntiles, t_begin, t_end, grid, st);
    case 2: return launch_bwd_tc_nkb<2, CAT>(m2h, m2l, m1h, m1l, gout, gin1, gin2, p, ntiles, t_begin, t_end, grid, st);
    case 3: return launch_bwd_tc_nkb<3, CAT>(m2h, m2l, m1h, m1l, gout, gin1, gin2, p, ntiles, t_begin, t_end, grid, st);
    default: return launch_bwd_tc_nkb<4, CAT>(m2h, m2l, m1h, m1l, gout, gin1, gin2, p, ntiles, t_begin, t_end, grid, st);
    }
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
    // the dense, activation-free gradient of fn2b200_correlation_backward keeps the original instantiations
    if (p.act || p.g_bstride != (long)p.D * p.oH * p.oW)
        return launch_bwd_tc_c<true>(m2h, m2l, m1h, m1l, gout, gin1, gin2, p, ntiles, t_begin, t_end, grid, st);
    return launch_bwd_tc_c<false>(m2h, m2l, m1h, m1l, gout, gin1, gin2, p, ntiles, t_begin, t_end, grid, st);
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

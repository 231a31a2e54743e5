// wgmma_selftest.cu -- hardware self-test of the wgmma / TMA-swizzle plumbing in wgmma.cuh: bf16 GEMMs with every operand
// form the tensor-core correlation kernels rely on, plus the descriptor forms around them, compared with a CPU product by
// tests/test_gpu_umma.py (through libfn2b200_test.so, csrc_test/fn2b200_test.h).  One CTA of two warpgroups; warpgroup wg
// computes rows [64 wg, 64 wg + 64) of D.
#include "../csrc/wgmma.cuh"
#include <cuda_bf16.h>

namespace fn2 {

// A K-major, B MN-major (the _mn test: A written by the threads, B^T = [K][N] loaded by TMA)
__device__ __forceinline__ void wgmma_m64n64k16_ak_bmn(float (&d)[32], uint64_t da, uint64_t db) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
        "%32, %33, 1, 1, 1, 0, 1;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db));
}

__device__ __forceinline__ void wgmma_m64n144k16_rs(float (&d)[72], const uint32_t (&a)[4], uint64_t db) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n144k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71}, "
        "{%72, %73, %74, %75}, %76, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}

constexpr int ST_M = 128, ST_N = 144, ST_KB = 64;
constexpr int ST_THREADS = 256;

// store an m64 x nN accumulator fragment of warpgroup wg to row-major D[128 x N]
template <int N>
__device__ __forceinline__ void st_store(float *D, const float (&acc)[N / 2], int tid) {
    const int wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31;
#pragma unroll
    for (int i = 0; i < N / 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int row = 64 * wg + 16 * w + (lane >> 2) + 8 * (j >> 1), col = 8 * i + 2 * (lane & 3) + (j & 1);
            D[row * N + col] = acc[4 * i + j];
        }
}

// A fragment of one K = 16 step (rows 16 w + lane/4 (+8) of the warpgroup; k pairs 2 (lane % 4) (+8)), read by `ld`
template <typename LD>
__device__ __forceinline__ void st_afrag(uint32_t (&a)[4], int tid, int k0, LD ld) {
    const int wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31;
    const int r0 = 64 * wg + 16 * w + (lane >> 2), kk = k0 + 2 * (lane & 3);
    a[0] = ld(r0, kk);
    a[1] = ld(r0 + 8, kk);
    a[2] = ld(r0, kk + 8);
    a[3] = ld(r0 + 8, kk + 8);
}

// mode 0: A and B K-major SW128 from shared memory (TMA) -- the forward's operands.
// mode 1: A from registers, read from global memory; B as mode 0.
// mode 2: A from registers, read from the TMA-swizzled shared-memory tile; B as mode 0.
__global__ void __launch_bounds__(ST_THREADS, 1)
wgmma_selftest_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                      const unsigned short *__restrict__ A, float *__restrict__ D, int K, int mode) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    unsigned char *sA = smem;                         // [128 rows][128 B], SW128
    unsigned char *sB = smem + ST_M * 128;            // [144 rows][128 B], SW128
    uint64_t *bar = reinterpret_cast<uint64_t *>(sB + ST_N * 128);
    const int tid = threadIdx.x, wg = tid >> 7;
    if (tid == 0) {
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    float acc[ST_N / 2];
#pragma unroll
    for (int i = 0; i < ST_N / 2; ++i) acc[i] = 0.f;
    wgmma_fence_operands(acc);
    for (int kb = 0; kb < K / ST_KB; ++kb) {
        if (tid == 0) {
            mbar_arrive_expect_tx(bar, (mode == 1 ? ST_N : ST_M + ST_N) * 128);
            if (mode != 1) tma_load_2d(sA, &mapA, bar, kb * ST_KB, 0);
            tma_load_2d(sB, &mapB, bar, kb * ST_KB, 0);
        }
        mbar_wait(bar, kb & 1);
        const uint64_t db = wgmma_desc_k_sw128(smem_u32(sB));
        if (mode == 0) {
            const uint64_t da = wgmma_desc_k_sw128(smem_u32(sA + wg * 64 * 128));
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < ST_KB / 16; ++ks) wgmma_m64n144k16_k(acc, da + 2 * ks, db + 2 * ks);
        } else {
            uint32_t a[ST_KB / 16][4];
#pragma unroll
            for (int ks = 0; ks < ST_KB / 16; ++ks) {
                if (mode == 1)
                    st_afrag(a[ks], tid, kb * ST_KB + ks * 16, [&](int r, int k) {
                        return *reinterpret_cast<const uint32_t *>(A + (size_t)r * K + k);
                    });
                else          // element (r, k) of a 128-byte-swizzled row: 16-byte chunk index XOR (r & 7)
                    st_afrag(a[ks], tid, ks * 16, [&](int r, int k) {
                        return *reinterpret_cast<const uint32_t *>(sA + r * 128 + ((((k >> 3) ^ (r & 7))) << 4) + (k & 7) * 2);
                    });
            }
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < ST_KB / 16; ++ks) wgmma_m64n144k16_rs(acc, a[ks], db + 2 * ks);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
        __syncthreads();                              // shared memory may be overwritten by the next block
    }
    st_store<ST_N>(D, acc, tid);
}

static int wgmma_selftest(const void *A, const void *B, float *D, int K, int mode, cudaStream_t st) {
    if (K <= 0 || K % ST_KB) return fail(FN2B200_EINVAL, "wgmma_selftest: K must be a positive multiple of 64");
    CUtensorMap ma, mb;
    uint64_t dimsA[2] = {(uint64_t)K, ST_M}, dimsB[2] = {(uint64_t)K, ST_N};
    uint64_t str[1] = {(uint64_t)K * 2};
    uint32_t boxA[2] = {ST_KB, ST_M}, boxB[2] = {ST_KB, ST_N};
    int rc = make_tensor_map_bf16_sw128(&ma, A, 2, dimsA, str, boxA);
    if (rc) return rc;
    rc = make_tensor_map_bf16_sw128(&mb, B, 2, dimsB, str, boxB);
    if (rc) return rc;
    const int smem = (ST_M + ST_N) * 128 + 1024 + 64;
    cudaError_t e = cudaFuncSetAttribute(wgmma_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return fail((int)e, "wgmma_selftest: smem attribute (%s)", cudaGetErrorString(e));
    wgmma_selftest_kernel<<<1, ST_THREADS, smem, st>>>(ma, mb, static_cast<const unsigned short *>(A), D, K, mode);
    count_launch();
    return check_launch("wgmma_selftest");
}
int wgmma_selftest_ss(const void *A, const void *B, float *D, int K, cudaStream_t st) { return wgmma_selftest(A, B, D, K, 0, st); }
int wgmma_selftest_rs_global(const void *A, const void *B, float *D, int K, cudaStream_t st) { return wgmma_selftest(A, B, D, K, 1, st); }
int wgmma_selftest_rs_smem(const void *A, const void *B, float *D, int K, cudaStream_t st) { return wgmma_selftest(A, B, D, K, 2, st); }

// D[128 x 64] = A[128 x 144] * Bt[144 x 64]: A written to shared memory by the threads, K-major without swizzle
// (a_sw32 = 0: 8-row x 16-byte core matrices, LBO = 2048 B between the two K chunks of a step, SBO = 128 B between
// 8-row groups) or with the 32-byte swizzle (a_sw32 = 1: 32-byte rows, 256-byte atoms); Bt ([K][N] row-major) loaded by
// TMA as an MN-major SW128 operand, the backward kernel's B form.
constexpr int ST2_K = 144, ST2_N = 64;
__host__ __device__ constexpr uint32_t sw32_offset(uint32_t r, uint32_t k) {
    return r * 32u + ((((k >> 3) & 1u) ^ ((r >> 2) & 1u)) << 4) + (k & 7u) * 2u;
}

__global__ void __launch_bounds__(ST_THREADS, 1)
wgmma_selftest_mn_kernel(const unsigned short *__restrict__ A, const __grid_constant__ CUtensorMap mapB, float *__restrict__ D,
                         int a_sw32) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    unsigned char *sB = smem;                              // [144 rows (K)][128 B], SW128 (MN-major)
    unsigned char *sA = smem + ST2_K * 128;                // 9 k-steps x 4096 B
    uint64_t *bar = reinterpret_cast<uint64_t *>(sA + 9 * 4096);
    const int tid = threadIdx.x, wg = tid >> 7;
    if (tid == 0) {
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    if (tid < ST_M) {                                      // thread p writes row p of A
        const int p = tid;
        for (int k = 0; k < ST2_K; ++k) {
            const int ks = k >> 4, c = (k >> 3) & 1, e = k & 7;
            const uint32_t off = a_sw32 ? ks * 4096 + sw32_offset(p, k & 15) : ks * 4096 + c * 2048 + (p >> 3) * 128 + (p & 7) * 16 + e * 2;
            *reinterpret_cast<unsigned short *>(sA + off) = A[(size_t)p * ST2_K + k];
        }
    }
    fence_proxy_async();          // generic-proxy smem writes -> visible to the tensor core (async proxy)
    __syncthreads();
    if (tid == 0) {
        mbar_arrive_expect_tx(bar, ST2_K * 128);
        tma_load_2d(sB, &mapB, bar, 0, 0);
    }
    mbar_wait(bar, 0);
    float acc[ST2_N / 2];
#pragma unroll
    for (int i = 0; i < ST2_N / 2; ++i) acc[i] = 0.f;
    wgmma_fence_operands(acc);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < ST2_K / 16; ++ks) {
        const uint32_t a = smem_u32(sA + ks * 4096);
        uint64_t da;
        if (a_sw32) {             // 64 rows per warpgroup x 32 B
            da = (uint64_t)(((a + wg * 64 * 32) & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(256 >> 4) << 32) |
                 ((uint64_t)3 << 62);
        } else {                  // 8 row groups per warpgroup x 128 B
            da = (uint64_t)(((a + wg * 8 * 128) & 0x3FFFF) >> 4) | ((uint64_t)(2048 >> 4) << 16) | ((uint64_t)(128 >> 4) << 32);
        }
        wgmma_m64n64k16_ak_bmn(acc, da, wgmma_desc_mn_sw128(smem_u32(sB) + ks * 16 * 128, ST2_K * 128));
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    st_store<ST2_N>(D, acc, tid);
}

int wgmma_selftest_mn(const void *A, const void *Bt, float *D, int a_sw32, cudaStream_t st) {
    CUtensorMap mb;
    uint64_t dims[2] = {ST2_N, ST2_K};
    uint64_t str[1] = {ST2_N * 2};
    uint32_t box[2] = {ST2_N, ST2_K};
    int rc = make_tensor_map_bf16_sw128(&mb, Bt, 2, dims, str, box);
    if (rc) return rc;
    const int smem = ST2_K * 128 + 9 * 4096 + 1024 + 64;
    cudaError_t e = cudaFuncSetAttribute(wgmma_selftest_mn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return fail((int)e, "wgmma_selftest_mn: smem attribute (%s)", cudaGetErrorString(e));
    wgmma_selftest_mn_kernel<<<1, ST_THREADS, smem, st>>>(static_cast<const unsigned short *>(A), mb, D, a_sw32);
    count_launch();
    return check_launch("wgmma_selftest_mn");
}

}  // namespace fn2

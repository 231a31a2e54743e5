/*
 * fn2b200_test.h -- C ABI of libfn2b200_test.so: hardware self-tests and micro-benchmarks of the building blocks
 * (wgmma / TMA descriptors, reduction flavours).  NOT part of the product:
 * libfn2b200.so neither contains nor links any of this; only tests/ load this library.
 * Same conventions as include/fn2b200.h (device pointers, stream handle, 0 = success, thread-local error text).
 */
#ifndef FN2B200_TEST_H_
#define FN2B200_TEST_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

const char *fn2b200_test_last_error(void);

/* D[128 x 144] (fp32, row-major) = A[128 x K] * B[144 x K]^T; A, B bf16 row-major, K a positive multiple of 64.
 * Both operands from shared memory (K-major, 128-byte swizzle, loaded by TMA) -- the forward kernel's forms. */
int fn2b200_test_wgmma_gemm_ss(const void *A_bf16, const void *B_bf16, float *D, int K, void *stream);

/* D[128 x 64] = A[128 x 144] * Bt[144 x 64]: A written to shared memory by the threads, K-major (a_sw32 = 0: no-swizzle
 * core-matrix layout, 1: 32-byte swizzle), Bt ([K][N] row-major) loaded as an MN-major SW128 operand -- the backward
 * kernel's B form. */
int fn2b200_test_wgmma_gemm_mn(const void *A_bf16, const void *Bt_bf16, float *D, int a_sw32, void *stream);

/* The _ss product with A taken from registers (wgmma's register-A form), the fragments read from global memory. */
int fn2b200_test_wgmma_gemm_rs(const void *A_bf16, const void *B_bf16, float *D, int K, void *stream);

/* The _rs product with A brought into shared memory by TMA (K-major SW128) and read from there into the fragments. */
int fn2b200_test_wgmma_gemm_rs_tma(const void *A_bf16, const void *B_bf16, float *D, int K, void *stream);

/* Reduction-flavour micro-benchmark (csrc_test/atomics_bench.cu): mode 0 red.global.f32,
 * 1 red.global.v2, 2 red.global.v4, 3 red.shared.f32, 4 plain shared RMW, 5 red.global.f32 with adjacent lane pairs.
 * buf holds grid * window floats (zeroed by the caller), cycles holds grid entries. */
int fn2b200_test_atomics_bench(float *buf, long long *cycles, int mode, int window, int iters, int grid, void *stream);

#ifdef __cplusplus
}
#endif
#endif

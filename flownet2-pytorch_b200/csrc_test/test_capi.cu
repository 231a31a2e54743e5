// test_capi.cu -- extern "C" boundary of libfn2b200_test.so (csrc_test/fn2b200_test.h).
#include "../csrc/common.cuh"
#include "fn2b200_test.h"

namespace fn2 {
int wgmma_selftest_ss(const void *A, const void *B, float *D, int K, cudaStream_t st);
int wgmma_selftest_rs_global(const void *A, const void *B, float *D, int K, cudaStream_t st);
int wgmma_selftest_rs_smem(const void *A, const void *B, float *D, int K, cudaStream_t st);
int wgmma_selftest_mn(const void *A, const void *Bt, float *D, int a_sw32, cudaStream_t st);
int atomics_bench(float *buf, long long *cycles, int mode, int window, int iters, int grid, cudaStream_t st);
}  // namespace fn2
using namespace fn2;

extern "C" {

const char *fn2b200_test_last_error(void) { return last_error_text(); }

int fn2b200_test_wgmma_gemm_ss(const void *A, const void *B, float *D, int K, void *stream) {
    if (!A || !B || !D) return fail(FN2B200_ENULL, "test_wgmma_gemm_ss: null pointer");
    if (int rc = bind_device_of(D)) return rc;
    return wgmma_selftest_ss(A, B, D, K, (cudaStream_t)stream);
}
int fn2b200_test_wgmma_gemm_mn(const void *A, const void *Bt, float *D, int a_sw32, void *stream) {
    if (!A || !Bt || !D) return fail(FN2B200_ENULL, "test_wgmma_gemm_mn: null pointer");
    if (int rc = bind_device_of(D)) return rc;
    return wgmma_selftest_mn(A, Bt, D, a_sw32 != 0, (cudaStream_t)stream);
}
int fn2b200_test_wgmma_gemm_rs(const void *A, const void *B, float *D, int K, void *stream) {
    if (!A || !B || !D) return fail(FN2B200_ENULL, "test_wgmma_gemm_rs: null pointer");
    if (int rc = bind_device_of(D)) return rc;
    return wgmma_selftest_rs_global(A, B, D, K, (cudaStream_t)stream);
}
int fn2b200_test_wgmma_gemm_rs_tma(const void *A, const void *B, float *D, int K, void *stream) {
    if (!A || !B || !D) return fail(FN2B200_ENULL, "test_wgmma_gemm_rs_tma: null pointer");
    if (int rc = bind_device_of(D)) return rc;
    return wgmma_selftest_rs_smem(A, B, D, K, (cudaStream_t)stream);
}

int fn2b200_test_atomics_bench(float *buf, long long *cycles, int mode, int window, int iters, int grid, void *stream) {
    if (!buf || !cycles) return fail(FN2B200_ENULL, "test_atomics_bench: null pointer");
    if (int rc = bind_device_of(buf)) return rc;
    return atomics_bench(buf, cycles, mode, window, iters, grid, (cudaStream_t)stream);
}

}  // extern "C"

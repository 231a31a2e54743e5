// runtime.cu -- host-side plumbing shared by libfn2b200.so and the test library: thread-local error text,
// launch counter, device binding by pointer, TMA descriptor encoding (driver entry point through the runtime).
#include <math.h>
#include <atomic>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace fn2 {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};  // statistics only; no behaviour depends on it

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }
int check_launch(const char *what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
        return fail((int)e, "%s: CUDA error %d (%s)", what, (int)e, cudaGetErrorString(e));
    return 0;
}

// Bind the calling thread to the device that owns `ptr`.  Worker threads (the autograd engine,
// nn.DataParallel replicas) may have no CUDA context current yet -- torch's device guard skips
// cudaSetDevice when the index already matches -- and driver calls such as
// cuTensorMapEncodeTiled then fail with CUDA_ERROR_INVALID_CONTEXT.
int bind_device_of(const void *ptr) {
    cudaPointerAttributes a;
    cudaError_t e = cudaPointerGetAttributes(&a, ptr);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail((int)e, "cudaPointerGetAttributes failed (%s)", cudaGetErrorString(e));
    }
    if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged)
        return fail(FN2B200_EINVAL, "pointer %p is not device memory (type %d): the C ABI takes device "
                    "pointers only", ptr, (int)a.type);
    e = cudaSetDevice(a.device);
    if (e != cudaSuccess) return fail((int)e, "cudaSetDevice(%d) failed (%s)", a.device, cudaGetErrorString(e));
    return 0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *,
                                  const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_tensor_map_f32(CUtensorMap *map, const void *base, int rank, const uint64_t *dims,
                        const uint64_t *strides_bytes, const uint32_t *box) {
    // Resolved per call (cheap, cached inside the runtime): keeps the library free of static
    // mutable state and of a link-time libcuda dependency.
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
    if (e != cudaSuccess || fn == nullptr || q != cudaDriverEntryPointSuccess)
        return fail(e != cudaSuccess ? (int)e : (int)cudaErrorNotSupported,
                    "cuTensorMapEncodeTiled entry point unavailable (err %d)", (int)e);
    cuuint64_t gdim[5], gstr[4];
    cuuint32_t bdim[5], estr[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bdim[i] = box[i];
        estr[i] = 1;
        if (i + 1 < rank) gstr[i] = strides_bytes[i];
    }
    CUresult r = ((EncodeTiledFn)fn)(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank,
                                     const_cast<void *>(base), gdim, gstr, bdim, estr,
                                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return fail((int)cudaErrorInvalidValue, "cuTensorMapEncodeTiled failed (CUresult %d)", (int)r);
    return 0;
}

int make_tensor_map_bf16_sw128(CUtensorMap *map, const void *base, int rank, const uint64_t *dims,
                               const uint64_t *strides_bytes, const uint32_t *box) {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
    if (e != cudaSuccess || fn == nullptr || q != cudaDriverEntryPointSuccess)
        return fail(e != cudaSuccess ? (int)e : (int)cudaErrorNotSupported,
                    "cuTensorMapEncodeTiled entry point unavailable (err %d)", (int)e);
    cuuint64_t gdim[5], gstr[4];
    cuuint32_t bdim[5], estr[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = dims[i];
        bdim[i] = box[i];
        estr[i] = 1;
        if (i + 1 < rank) gstr[i] = strides_bytes[i];
    }
    CUresult r = ((EncodeTiledFn)fn)(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank,
                                     const_cast<void *>(base), gdim, gstr, bdim, estr,
                                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return fail((int)cudaErrorInvalidValue, "cuTensorMapEncodeTiled(bf16, SW128) failed (CUresult %d)", (int)r);
    return 0;
}


uint64_t launches_so_far() { return g_launches.load(std::memory_order_relaxed); }
const char *last_error_text() { return g_err; }

}  // namespace fn2

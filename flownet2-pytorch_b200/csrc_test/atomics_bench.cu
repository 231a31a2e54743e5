// atomics_bench.cu -- micro-benchmark of the reduction flavours a bilinear scatter (Resample2d backward) can be
// built from.  Test / tuning hook only; lives in libfn2b200_test.so, not in the product.
//
// Every thread issues `iters` reductions to pseudo-random addresses inside a window of `window` floats that belongs
// to its CTA (global modes: window placed at cta * window inside `buf`; shared modes: the CTA's shared memory).
//   mode 0  red.global.add.f32            one float per lane
//   mode 1  red.global.add.v2.f32         8-byte aligned pairs
//   mode 2  red.global.add.v4.f32         16-byte aligned quads
//   mode 3  red.shared.add.f32            shared-memory reduction, random banks
//   mode 4  ld.shared + st.shared         non-atomic read-modify-write (the cost floor of an exclusive-owner scheme)
//   mode 5  red.global.add.f32            lanes 2i / 2i+1 hit adjacent floats (the xL/xR tap pair)
#include "../csrc/common.cuh"

namespace fn2 {

__device__ __forceinline__ uint32_t lcg(uint32_t &s) {
    s = s * 1664525u + 1013904223u;
    return s >> 8;
}

__global__ void __launch_bounds__(256)
atomics_bench_kernel(float *buf, long long *cycles, int mode, int window, int iters) {
    extern __shared__ float sm[];
    uint32_t s = (blockIdx.x * 256u + threadIdx.x) * 2654435761u + 12345u;
    float *base = buf + (size_t)blockIdx.x * window;
    if (mode == 3 || mode == 4) {
        for (int i = threadIdx.x; i < window; i += 256) sm[i] = 0.f;
        __syncthreads();
    }
    long long t0 = clock64();
    float v = 1.0f + threadIdx.x * 1e-3f;
    switch (mode) {
        case 0:
            for (int i = 0; i < iters; ++i) {
                float *p = base + lcg(s) % (uint32_t)window;
                asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
            }
            break;
        case 1:
            for (int i = 0; i < iters; ++i) {
                float *p = base + (lcg(s) % (uint32_t)(window / 2)) * 2;
                asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v), "f"(v) : "memory");
            }
            break;
        case 2:
            for (int i = 0; i < iters; ++i) {
                float *p = base + (lcg(s) % (uint32_t)(window / 4)) * 4;
                asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v), "f"(v), "f"(v), "f"(v) : "memory");
            }
            break;
        case 3:
            for (int i = 0; i < iters; ++i) {
                uint32_t a = smem_u32(sm + lcg(s) % (uint32_t)window);
                asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory");
            }
            break;
        case 4:
            for (int i = 0; i < iters; ++i) {
                volatile float *p = sm + lcg(s) % (uint32_t)window;
                *p = *p + v;
            }
            break;
        case 5:
            for (int i = 0; i < iters; ++i) {
                uint32_t r = lcg(s);
                r = __shfl_sync(0xffffffffu, r, threadIdx.x & 30);          // pairs of lanes share the draw
                float *p = base + (r % (uint32_t)(window - 1)) + (threadIdx.x & 1);
                asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
            }
            break;
    }
    __syncthreads();
    long long t1 = clock64();
    if (mode == 3 || mode == 4) {
        float acc = 0.f;
        for (int i = threadIdx.x; i < window; i += 256) acc += sm[i];
        if (acc == -1.f) buf[0] = acc;      // keep the shared-memory work observable
    }
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

int atomics_bench(float *buf, long long *cycles, int mode, int window, int iters, int grid, cudaStream_t st) {
    if (mode < 0 || mode > 5 || window < 8 || window % 4 || iters < 1 || grid < 1)
        return fail(FN2B200_EINVAL, "atomics_bench: mode %d window %d iters %d grid %d", mode, window, iters, grid);
    size_t smem = (mode == 3 || mode == 4) ? (size_t)window * 4 : 0;
    if (smem > 200 * 1024) return fail(FN2B200_EINVAL, "atomics_bench: window too large for shared memory");
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(atomics_bench_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return fail((int)e, "atomics_bench: smem attribute (%s)", cudaGetErrorString(e));
    }
    atomics_bench_kernel<<<grid, 256, smem, st>>>(buf, cycles, mode, window, iters);
    count_launch();
    return check_launch("atomics_bench");
}

}  // namespace fn2

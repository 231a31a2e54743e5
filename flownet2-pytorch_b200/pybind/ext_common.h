// ext_common.h -- shared by the three pybind extension modules (correlation_cuda / resample2d_cuda / channelnorm_cuda):
// thin ATen <-> C-ABI glue.  No arithmetic lives here; everything is forwarded to libfn2b200.so (include/fn2b200.h).
#pragma once
#include <torch/extension.h>

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include "fn2b200.h"

namespace fn2ext {

inline void check(int rc, const char *what) {
    // the reference raises AT_ERROR("CUDA call failed") (correlation_cuda.cc:81-83); we add the library's message
    TORCH_CHECK(rc == 0, what, " failed (status ", rc, "): ", fn2b200_last_error());
}
inline void need_cuda_f32(const at::Tensor &t, const char *name) {
    TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor (there is no CPU path; the reference has none either)");
    TORCH_CHECK(t.scalar_type() == at::kFloat, name, " must be float32 (got ", t.scalar_type(), ")");
}
inline void need_out(const at::Tensor &t, const char *name) {
    need_cuda_f32(t, name);
    TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
}
inline void *stream_of(const at::Tensor &t) { return at::cuda::getCurrentCUDAStream(t.get_device()).stream(); }
inline at::Tensor scratch(size_t bytes, const at::Tensor &like) {
    return at::empty({(int64_t)(bytes ? bytes : 16)}, like.options().dtype(at::kByte));
}
// the C ABI's dtype code of a 16-bit tensor (1 = fp16, 2 = bf16), 0 for anything else
inline int dtype16(const at::Tensor &t) { return t.scalar_type() == at::kHalf ? 1 : (t.scalar_type() == at::kBFloat16 ? 2 : 0); }

}  // namespace fn2ext

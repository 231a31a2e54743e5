// channelnorm_cuda.cc -- the reference's extension module `channelnorm_cuda` (channelnorm_package/channelnorm_cuda.cc:
// 6-30) on libfn2b200; float32 and, like the reference's dispatch (channelnorm_kernel.cu:111,152), half.
#include "ext_common.h"
using namespace fn2ext;

int channelnorm_cuda_forward(at::Tensor &input1, at::Tensor &output, int norm_deg) {
    TORCH_CHECK(input1.is_cuda() && output.is_cuda() && output.is_contiguous(), "CUDA tensors, contiguous output required");
    TORCH_CHECK(input1.scalar_type() == output.scalar_type(), "input1 / output dtype mismatch");
    if (!dtype16(input1)) need_cuda_f32(input1, "input1");
    int rc;
    {
        c10::cuda::CUDAGuard guard(input1.device());
        at::Tensor a = input1.contiguous();
        const int B = a.size(0), C = a.size(1), H = a.size(2), W = a.size(3);
        if (int dt = dtype16(a))
            rc = fn2b200_channelnorm_forward_16(a.data_ptr(), output.data_ptr(), B, C, H, W, norm_deg, dt, stream_of(a));
        else
            rc = fn2b200_channelnorm_forward(a.data_ptr<float>(), output.data_ptr<float>(), B, C, H, W, norm_deg, stream_of(a));
    }
    check(rc, "channelnorm_forward");
    return 1;
}

int channelnorm_cuda_backward(at::Tensor &input1, at::Tensor &output, at::Tensor &gradOutput, at::Tensor &gradInput1, int norm_deg) {
    TORCH_CHECK(input1.is_cuda() && gradInput1.is_cuda() && gradInput1.is_contiguous(), "CUDA tensors, contiguous gradInput1 required");
    TORCH_CHECK(input1.scalar_type() == output.scalar_type() && input1.scalar_type() == gradOutput.scalar_type() &&
                input1.scalar_type() == gradInput1.scalar_type(), "dtype mismatch");
    if (!dtype16(input1)) need_cuda_f32(input1, "input1");
    int rc;
    {
        c10::cuda::CUDAGuard guard(input1.device());
        at::Tensor a = input1.contiguous(), o = output.contiguous(), g = gradOutput.contiguous();
        const int B = a.size(0), C = a.size(1), H = a.size(2), W = a.size(3);
        if (int dt = dtype16(a))
            rc = fn2b200_channelnorm_backward_16(a.data_ptr(), o.data_ptr(), g.data_ptr(), gradInput1.data_ptr(), B, C, H, W, norm_deg, dt,
                                                 stream_of(a));
        else
            rc = fn2b200_channelnorm_backward(a.data_ptr<float>(), o.data_ptr<float>(), g.data_ptr<float>(), gradInput1.data_ptr<float>(),
                                              B, C, H, W, norm_deg, stream_of(a));
    }
    check(rc, "channelnorm_backward");
    return 1;
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.def("forward", &channelnorm_cuda_forward, "Channel norm forward (CUDA)");
    m.def("backward", &channelnorm_cuda_backward, "Channel norm backward (CUDA)");
}

// channelnorm_cuda.cc -- the reference's extension module `channelnorm_cuda` (channelnorm_package/channelnorm_cuda.cc:
// 6-30) on libfn2b200; float32 and, like the reference's dispatch (channelnorm_kernel.cu:111,152), half.
#include "ext_common.h"
using namespace fn2ext;

int channelnorm_cuda_forward(at::Tensor &input1, at::Tensor &output, int norm_deg) {
    if (!dtype16(input1)) need_cuda_f32(input1, "input1");
    channelnorm_forward(input1, output, norm_deg);          // output in input1's dtype
    return 1;
}

int channelnorm_cuda_backward(at::Tensor &input1, at::Tensor &output, at::Tensor &gradOutput, at::Tensor &gradInput1, int norm_deg) {
    if (!dtype16(input1)) need_cuda_f32(input1, "input1");
    TORCH_CHECK(output.scalar_type() == input1.scalar_type() && gradOutput.scalar_type() == input1.scalar_type(),
                "channelnorm_backward: output and grad_output must have input1's dtype ", input1.scalar_type());
    channelnorm_backward(input1, output, gradOutput, gradInput1, norm_deg);      // gradInput1 in input1's dtype
    return 1;
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.def("forward", &channelnorm_cuda_forward, "Channel norm forward (CUDA)");
    m.def("backward", &channelnorm_cuda_backward, "Channel norm backward (CUDA)");
}

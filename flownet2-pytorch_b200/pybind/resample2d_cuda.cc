// resample2d_cuda.cc -- the reference's extension module `resample2d_cuda` (resample2d_package/resample2d_cuda.cc:6-31)
// on libfn2b200.  The caller pre-allocates (and zero-fills) the outputs at their final shape (resample2d.py:18,31-32).
#include "ext_common.h"
using namespace fn2ext;

int resample2d_cuda_forward(at::Tensor &input1, at::Tensor &input2, at::Tensor &output, int kernel_size, bool bilinear) {
    need_cuda_f32(input1, "input1"); need_cuda_f32(input2, "input2"); need_cuda_f32(output, "output");
    resample2d_forward(input1, input2, output, kernel_size, bilinear, 0, 1.0);
    return 1;
}

int resample2d_cuda_backward(at::Tensor &input1, at::Tensor &input2, at::Tensor &gradOutput, at::Tensor &gradInput1,
                             at::Tensor &gradInput2, int kernel_size, bool bilinear) {
    need_cuda_f32(input1, "input1"); need_cuda_f32(input2, "input2"); need_cuda_f32(gradOutput, "grad_output");
    need_cuda_f32(gradInput1, "grad_input1"); need_cuda_f32(gradInput2, "grad_input2");
    // zero_grad_input1 = false: gradInput1 arrives zero-filled (resample2d.py:31) and is accumulated into
    resample2d_backward(input1, input2, gradOutput, kernel_size, bilinear, true, true, gradInput1, gradInput2, false);
    return 1;
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.def("forward", &resample2d_cuda_forward, "Resample2D forward (CUDA)");
    m.def("backward", &resample2d_cuda_backward, "Resample2D backward (CUDA)");
}

// correlation_cuda.cc -- the reference's extension module `correlation_cuda` (correlation_package/correlation_cuda.cc:
// 10-16, 89-96, 169-172: same function names, argument order, out-parameter convention, return value) on libfn2b200.
#include "ext_common.h"
using namespace fn2ext;

int correlation_forward_cuda(at::Tensor &input1, at::Tensor &input2, at::Tensor &rInput1, at::Tensor &rInput2,
                             at::Tensor &output, int pad_size, int kernel_size, int max_displacement, int stride1,
                             int stride2, int corr_type_multiply) {
    (void)rInput1; (void)rInput2;        // the reference's padded NHWC scratch (:36-41): not needed, left untouched
    need_cuda_f32(input1, "input1"); need_cuda_f32(input2, "input2"); need_cuda_f32(output, "output");
    const CorrShape s = corr_shape(input1, input2, pad_size, kernel_size, max_displacement, stride1, stride2);
    output.resize_({s.B, s.D, s.oH, s.oW});      // :38 (no fill_(0): every element is written)
    correlation_forward(input1, input2, output, false, 0, 1.0, pad_size, kernel_size, max_displacement, stride1, stride2,
                        corr_type_multiply);
    return 1;
}

int correlation_backward_cuda(at::Tensor &input1, at::Tensor &input2, at::Tensor &rInput1, at::Tensor &rInput2,
                              at::Tensor &gradOutput, at::Tensor &gradInput1, at::Tensor &gradInput2, int pad_size,
                              int kernel_size, int max_displacement, int stride1, int stride2, int corr_type_multiply) {
    (void)rInput1; (void)rInput2;
    need_cuda_f32(input1, "input1"); need_cuda_f32(input2, "input2"); need_cuda_f32(gradOutput, "grad_output");
    need_cuda_f32(gradInput1, "grad_input1"); need_cuda_f32(gradInput2, "grad_input2");
    gradInput1.resize_(input1.sizes());       // :109-110
    gradInput2.resize_(input2.sizes());
    // no workspace is handed over from the forward: the reference's Function keeps none
    correlation_backward(input1, input2, gradOutput, false, std::nullopt, 0, 1.0, std::nullopt, pad_size, kernel_size,
                         max_displacement, stride1, stride2, corr_type_multiply, true, true, gradInput1, gradInput2);
    return 1;
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.def("forward", &correlation_forward_cuda, "Correlation forward (CUDA)");
    m.def("backward", &correlation_backward_cuda, "Correlation backward (CUDA)");
}

// fn2b200_ops.cc -- the three layers and the fused ops as PyTorch operators, torch.ops.fn2b200.* (TORCH_LIBRARY), and,
// as the Python module of the same library, the host-side glue of every op (ext_common.h) that flownet2_b200.functional
// calls.  Every operator is functional: it allocates its outputs through torch's caching allocator, launches on the
// current stream and keeps no state between calls, so it can be traced by torch.compile, exported by torch.export and
// captured into a CUDA graph.  Fake kernels and autograd formulas are registered from Python (flownet2_b200.ops).  The
// library registers its schemas without a GPU; the kernels are CUDA only.
#include "ext_common.h"
using namespace fn2ext;

namespace op {

// a gradient that was not asked for: an empty fp32 tensor (the op's outputs are always tensors)
at::Tensor or_none(const at::Tensor &t, const at::Tensor &like) {
    return t.defined() ? t : at::empty({0}, like.options().dtype(at::kFloat));
}
Grads or_none(const Grads &g, const at::Tensor &like) { return {or_none(std::get<0>(g), like), or_none(std::get<1>(g), like)}; }

// ---- correlation -------------------------------------------------------------------------------------------------

std::tuple<at::Tensor, at::Tensor> correlation_forward(const at::Tensor &input1, const at::Tensor &input2, int64_t pad,
                                                       int64_t k, int64_t md, int64_t s1, int64_t s2, int64_t mul) {
    return fn2ext::correlation_forward(input1, input2, std::nullopt, false, 0, 1.0, pad, k, md, s1, s2, mul);
}

// `workspace` is what the forward returned for the same inputs (autograd's version counter rules out in-place changes
// of saved inputs), or an empty tensor.
Grads correlation_backward(const at::Tensor &input1, const at::Tensor &input2, const at::Tensor &grad_output,
                           const at::Tensor &workspace, int64_t pad, int64_t k, int64_t md, int64_t s1, int64_t s2,
                           int64_t mul, bool need1, bool need2) {
    return or_none(fn2ext::correlation_backward(input1, input2, grad_output, false, std::nullopt, 0, 1.0, workspace, pad,
                                                k, md, s1, s2, mul, need1, need2, std::nullopt, std::nullopt),
                   input1);
}

// [redir | LeakyReLU(leaky_slope)(correlation)] -> (cat, workspace)
std::tuple<at::Tensor, at::Tensor> correlation_forward_cat(const at::Tensor &redir, const at::Tensor &input1,
                                                           const at::Tensor &input2, int64_t pad, int64_t k, int64_t md,
                                                           int64_t s1, int64_t s2, int64_t mul, double leaky_slope) {
    need_cuda(redir, "redir"); need_cuda(input1, "input1"); need_cuda(input2, "input2");
    const CorrShape s = corr_shape(input1, input2, pad, k, md, s1, s2);
    TORCH_CHECK(redir.dim() == 4 && redir.size(0) == s.B && redir.size(2) == s.oH && redir.size(3) == s.oW,
                "CorrelationCat: redir ", redir.sizes(), " does not match the correlation output [", s.B, ", D, ", s.oH,
                ", ", s.oW, "]");
    const int64_t R = redir.size(1);
    c10::cuda::CUDAGuard guard(input1.device());
    at::Tensor cat = at::empty({s.B, R + s.D, s.oH, s.oW}, input1.options().dtype(at::kFloat));
    cat.narrow(1, 0, R).copy_(redir);
    return {cat, std::get<1>(fn2ext::correlation_forward(input1, input2, cat, true, R, leaky_slope, pad, k, md, s1, s2,
                                                         mul))};
}

Grads correlation_backward_cat(const at::Tensor &input1, const at::Tensor &input2, const at::Tensor &grad_cat,
                               const at::Tensor &cat, const at::Tensor &workspace, int64_t ch_offset, double leaky_slope,
                               int64_t pad, int64_t k, int64_t md, int64_t s1, int64_t s2, int64_t mul, bool need1,
                               bool need2) {
    return or_none(fn2ext::correlation_backward(input1, input2, grad_cat, true, cat, ch_offset, leaky_slope, workspace,
                                                pad, k, md, s1, s2, mul, need1, need2, std::nullopt, std::nullopt),
                   input1);
}

// ---- Resample2d and ChannelNorm ----------------------------------------------------------------------------------

at::Tensor resample2d_forward(const at::Tensor &input1, const at::Tensor &input2, int64_t kernel_size, bool bilinear) {
    return fn2ext::resample2d_forward(input1, input2, std::nullopt, kernel_size, bilinear, 0, 1.0);
}

Grads resample2d_backward(const at::Tensor &input1, const at::Tensor &input2, const at::Tensor &grad_output,
                          int64_t kernel_size, bool bilinear, bool need1, bool need2) {
    return or_none(fn2ext::resample2d_backward(input1, input2, grad_output, kernel_size, bilinear, need1, need2,
                                               std::nullopt, std::nullopt, true),
                   input2);
}

at::Tensor channelnorm_forward(const at::Tensor &input1, int64_t norm_deg) {
    return fn2ext::channelnorm_forward(input1, std::nullopt, norm_deg);
}

at::Tensor channelnorm_backward(const at::Tensor &input1, const at::Tensor &output, const at::Tensor &grad_output,
                                int64_t norm_deg) {
    return fn2ext::channelnorm_backward(input1, output, grad_output, std::nullopt, norm_deg);
}

// ---- warp -> diff -> channel-norm -> concat ----------------------------------------------------------------------

// the glue's input checks, and one more: the fake kernels take the batch from x
void same_batch(const at::Tensor &x, const at::Tensor &flow, int64_t C, const char *who) {
    warp_concat_inputs(x, flow, C, who);
    TORCH_CHECK(x.size(0) == flow.size(0), who, ": x ", x.sizes(), " and flow ", flow.sizes(), " must have one batch");
}

at::Tensor warp_concat_forward(const at::Tensor &x, const at::Tensor &flow, int64_t C, int64_t upsample_mode,
                               double flow_mul, double flow_div, int64_t cat_channels, int64_t ch_x, int64_t n_x,
                               int64_t ch_warped, int64_t ch_flow, int64_t ch_flow_norm, int64_t ch_diff_norm) {
    need_cuda(x, "x"); need_cuda(flow, "flow");
    same_batch(x, flow, C, "warp_concat_forward");
    c10::cuda::CUDAGuard guard(flow.device());
    // channels no product covers (the C ABI refuses overlapping ranges) are zero: the op's output is fully defined
    const int64_t covered = (ch_x >= 0 ? n_x : 0) + (ch_warped >= 0 ? C : 0) + (ch_flow >= 0 ? 2 : 0) +
                            (ch_flow_norm >= 0) + (ch_diff_norm >= 0);
    const auto opt = flow.options().dtype(at::kFloat);
    at::Tensor cat = covered < cat_channels ? at::zeros({x.size(0), cat_channels, x.size(2), x.size(3)}, opt)
                                            : at::empty({x.size(0), cat_channels, x.size(2), x.size(3)}, opt);
    return fn2ext::warp_concat_forward(x, flow, cat, C, upsample_mode, flow_mul, flow_div, cat_channels,
                                       {ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm});
}

Grads warp_concat_backward(const at::Tensor &x, const at::Tensor &flow, const at::Tensor &grad_cat, int64_t C,
                           int64_t upsample_mode, double flow_mul, double flow_div, int64_t ch_x, int64_t n_x,
                           int64_t ch_warped, int64_t ch_flow, int64_t ch_flow_norm, int64_t ch_diff_norm, bool need_x,
                           bool need_flow) {
    need_cuda(x, "x"); need_cuda(flow, "flow"); need_cuda(grad_cat, "grad_cat");
    same_batch(x, flow, C, "warp_concat_backward");
    return or_none(fn2ext::warp_concat_backward(x, flow, grad_cat, C, upsample_mode, flow_mul, flow_div,
                                                {ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm}, need_x,
                                                need_flow),
                   flow);
}

// concat3 of models.py:179: (img0 | sd flow | s2 flow | |sd flow| | |s2 flow| | sd diff norm | s2 diff norm), each flow
// the nearest x4 upsample of its quarter-resolution flow2 (sd: / div_flow, models.py:167; s2: * div_flow, :154)
constexpr WarpLayout FUSION_SD{0, 3, -1, 3, 7, 9}, FUSION_S2{-1, 0, -1, 5, 8, 10};
constexpr int64_t FUSION_CHANNELS = 11, NEAREST = 2;

at::Tensor fusion_concat(const at::Tensor &x, const at::Tensor &sd_flow2, const at::Tensor &s2_flow2, double div_flow) {
    need_cuda(x, "x"); need_cuda(sd_flow2, "sd_flow2"); need_cuda(s2_flow2, "s2_flow2");
    same_batch(x, sd_flow2, 3, "fusion_concat");
    same_batch(x, s2_flow2, 3, "fusion_concat");
    c10::cuda::CUDAGuard guard(x.device());
    at::Tensor cat = at::empty({x.size(0), FUSION_CHANNELS, x.size(2), x.size(3)}, x.options().dtype(at::kFloat));
    fn2ext::warp_concat_forward(x, sd_flow2, cat, 3, NEAREST, 1.0 / div_flow, 1.0, FUSION_CHANNELS, FUSION_SD);
    fn2ext::warp_concat_forward(x, s2_flow2, cat, 3, NEAREST, div_flow, 1.0, FUSION_CHANNELS, FUSION_S2);
    return cat;
}

// two warp_concat backward passes, each reading its own channels of grad_cat; the x gradients summed
std::tuple<at::Tensor, at::Tensor, at::Tensor> fusion_concat_backward(const at::Tensor &x, const at::Tensor &sd_flow2,
                                                                      const at::Tensor &s2_flow2, const at::Tensor &grad_cat,
                                                                      double div_flow, bool need_x, bool need_sd,
                                                                      bool need_s2) {
    need_cuda(x, "x"); need_cuda(sd_flow2, "sd_flow2"); need_cuda(s2_flow2, "s2_flow2"); need_cuda(grad_cat, "grad_cat");
    same_batch(x, sd_flow2, 3, "fusion_concat_backward");
    same_batch(x, s2_flow2, 3, "fusion_concat_backward");
    at::Tensor gx, g_sd, g_s2, gx2;
    if (need_x || need_sd)
        std::tie(gx, g_sd) = fn2ext::warp_concat_backward(x, sd_flow2, grad_cat, 3, NEAREST, 1.0 / div_flow, 1.0, FUSION_SD,
                                                          need_x, need_sd);
    if (need_x || need_s2) {
        std::tie(gx2, g_s2) = fn2ext::warp_concat_backward(x, s2_flow2, grad_cat, 3, NEAREST, div_flow, 1.0, FUSION_S2,
                                                           need_x, need_s2);
        if (need_x) gx.add_(gx2);
    }
    return {or_none(gx, x), or_none(g_sd, x), or_none(g_s2, x)};
}

}  // namespace op

TORCH_LIBRARY(fn2b200, m) {
    m.def("correlation_forward(Tensor input1, Tensor input2, int pad_size, int kernel_size, int max_displacement, "
          "int stride1, int stride2, int corr_multiply=1) -> (Tensor output, Tensor workspace)");
    m.def("correlation_backward(Tensor input1, Tensor input2, Tensor grad_output, Tensor workspace, int pad_size, "
          "int kernel_size, int max_displacement, int stride1, int stride2, int corr_multiply=1, bool need1=True, "
          "bool need2=True) -> (Tensor grad_input1, Tensor grad_input2)");
    m.def("correlation_forward_cat(Tensor redir, Tensor input1, Tensor input2, int pad_size, int kernel_size, "
          "int max_displacement, int stride1, int stride2, int corr_multiply=1, float leaky_slope=0.1) -> "
          "(Tensor cat, Tensor workspace)");
    m.def("correlation_backward_cat(Tensor input1, Tensor input2, Tensor grad_cat, Tensor cat, Tensor workspace, "
          "int ch_offset, float leaky_slope, int pad_size, int kernel_size, int max_displacement, int stride1, int stride2, "
          "int corr_multiply=1, bool need1=True, bool need2=True) -> (Tensor grad_input1, Tensor grad_input2)");
    m.def("resample2d_forward(Tensor input1, Tensor input2, int kernel_size=1, bool bilinear=True) -> Tensor");
    m.def("resample2d_backward(Tensor input1, Tensor input2, Tensor grad_output, int kernel_size=1, bool bilinear=True, "
          "bool need1=True, bool need2=True) -> (Tensor grad_input1, Tensor grad_input2)");
    m.def("channelnorm_forward(Tensor input1, int norm_deg=2) -> Tensor");
    m.def("channelnorm_backward(Tensor input1, Tensor output, Tensor grad_output, int norm_deg=2) -> Tensor");
    m.def("warp_concat_forward(Tensor x, Tensor flow, int C, int upsample_mode, float flow_mul, float flow_div, "
          "int cat_channels, int ch_x, int n_x, int ch_warped, int ch_flow, int ch_flow_norm, int ch_diff_norm) -> Tensor");
    m.def("warp_concat_backward(Tensor x, Tensor flow, Tensor grad_cat, int C, int upsample_mode, float flow_mul, "
          "float flow_div, int ch_x, int n_x, int ch_warped, int ch_flow, int ch_flow_norm, int ch_diff_norm, "
          "bool need_x=True, bool need_flow=True) -> (Tensor grad_x, Tensor grad_flow)");
    m.def("fusion_concat(Tensor x, Tensor sd_flow2, Tensor s2_flow2, float div_flow) -> Tensor");
    m.def("fusion_concat_backward(Tensor x, Tensor sd_flow2, Tensor s2_flow2, Tensor grad_cat, float div_flow, "
          "bool need_x=True, bool need_sd=True, bool need_s2=True) -> (Tensor grad_x, Tensor grad_sd, Tensor grad_s2)");
}

TORCH_LIBRARY_IMPL(fn2b200, CUDA, m) {
    m.impl("correlation_forward", &op::correlation_forward);
    m.impl("correlation_backward", &op::correlation_backward);
    m.impl("correlation_forward_cat", &op::correlation_forward_cat);
    m.impl("correlation_backward_cat", &op::correlation_backward_cat);
    m.impl("resample2d_forward", &op::resample2d_forward);
    m.impl("resample2d_backward", &op::resample2d_backward);
    m.impl("channelnorm_forward", &op::channelnorm_forward);
    m.impl("channelnorm_backward", &op::channelnorm_backward);
    m.impl("warp_concat_forward", &op::warp_concat_forward);
    m.impl("warp_concat_backward", &op::warp_concat_backward);
    m.impl("fusion_concat", &op::fusion_concat);
    m.impl("fusion_concat_backward", &op::fusion_concat_backward);
}

// the glue itself, for flownet2_b200.functional: caller-supplied outputs, absent gradients as None
PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.def("correlation_forward", &fn2ext::correlation_forward);
    m.def("correlation_backward", &fn2ext::correlation_backward);
    m.def("resample2d_forward", &fn2ext::resample2d_forward);
    m.def("resample2d_backward", &fn2ext::resample2d_backward);
    m.def("channelnorm_forward", &fn2ext::channelnorm_forward);
    m.def("channelnorm_backward", &fn2ext::channelnorm_backward);
    m.def("warp_concat_forward", [](const at::Tensor &x, const at::Tensor &flow, const Opt &out, int64_t C,
                                    int64_t upsample_mode, double flow_mul, double flow_div, int64_t cat_channels,
                                    int64_t ch_x, int64_t n_x, int64_t ch_warped, int64_t ch_flow, int64_t ch_flow_norm,
                                    int64_t ch_diff_norm) {
        return fn2ext::warp_concat_forward(x, flow, out, C, upsample_mode, flow_mul, flow_div, cat_channels,
                                           {ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm});
    });
    m.def("warp_concat_backward", [](const at::Tensor &x, const at::Tensor &flow, const at::Tensor &grad_cat, int64_t C,
                                     int64_t upsample_mode, double flow_mul, double flow_div, int64_t ch_x, int64_t n_x,
                                     int64_t ch_warped, int64_t ch_flow, int64_t ch_flow_norm, int64_t ch_diff_norm,
                                     bool need_x, bool need_flow) {
        return fn2ext::warp_concat_backward(x, flow, grad_cat, C, upsample_mode, flow_mul, flow_div,
                                            {ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm}, need_x,
                                            need_flow);
    });
}

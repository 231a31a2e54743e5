// fn2b200_ops.cc -- the three layers and the fused ops as PyTorch operators, torch.ops.fn2b200.* (TORCH_LIBRARY), on
// libfn2b200's C ABI.  Every op is functional: it allocates its outputs through torch's caching allocator, launches on
// the current stream and keeps no state between calls, so it can be traced by torch.compile, exported by torch.export
// and captured into a CUDA graph.  Fake kernels and autograd formulas are registered from Python (flownet2_b200.ops).
// The library registers its schemas without a GPU; the kernels are CUDA only.
#include "ext_common.h"
using namespace fn2ext;

namespace {

inline void *ptr(const at::Tensor &t) { return t.defined() && t.numel() ? t.data_ptr() : nullptr; }
inline float *fptr(const at::Tensor &t) { return static_cast<float *>(ptr(t)); }
inline at::Tensor f32(const at::Tensor &t) { return t.to(at::kFloat); }                  // strided views kept as they are
inline at::Tensor f32c(const at::Tensor &t) { return t.to(at::kFloat).contiguous(); }
inline void need_cuda(const at::Tensor &t, const char *name) {
    TORCH_CHECK(t.is_cuda(), "flownet2-pytorch_b200 runs on CUDA tensors only (", name, " is a ", t.device().type(),
                " tensor)");
}
// a gradient that was not asked for: an empty fp32 tensor (the op's outputs are always tensors)
inline at::Tensor none_like(const at::Tensor &t) { return at::empty({0}, t.options().dtype(at::kFloat)); }
inline std::array<int64_t, 4> strides4(const at::Tensor &t) { return {t.stride(0), t.stride(1), t.stride(2), t.stride(3)}; }

// ---- correlation -------------------------------------------------------------------------------------------------

struct CorrShape { int B, C, H, W, D, oH, oW; };

CorrShape corr_shape(const at::Tensor &input1, const at::Tensor &input2, int64_t pad, int64_t k, int64_t md, int64_t s1,
                     int64_t s2) {
    need_cuda(input1, "input1"); need_cuda(input2, "input2");
    TORCH_CHECK(input1.dim() == 4 && input1.sizes() == input2.sizes(),
                "correlation: input1/input2 must be 4-D with equal shapes, got ", input1.sizes(), " and ", input2.sizes());
    CorrShape s{(int)input1.size(0), (int)input1.size(1), (int)input1.size(2), (int)input1.size(3), 0, 0, 0};
    check(fn2b200_correlation_out_shape(s.C, s.H, s.W, pad, k, md, s1, s2, &s.D, &s.oH, &s.oW), "correlation_out_shape");
    TORCH_CHECK(s.oH > 0 && s.oW > 0, "correlation: empty output (", s.oH, " x ", s.oW, ") for input ", s.H, "x", s.W,
                ", pad_size=", pad, ", max_displacement=", md, ", kernel_size=", k);
    return s;
}

// [redir | LeakyReLU(leaky)(correlation)] -> (cat, workspace); no redir: the plain correlation [B, D, oH, oW].
std::tuple<at::Tensor, at::Tensor> corr_forward(const at::Tensor *redir, const at::Tensor &input1, const at::Tensor &input2,
                                                int64_t pad, int64_t k, int64_t md, int64_t s1, int64_t s2, int64_t mul,
                                                double leaky, const char *who) {
    const CorrShape s = corr_shape(input1, input2, pad, k, md, s1, s2);
    const int R = redir ? (int)redir->size(1) : 0;
    if (redir) {
        need_cuda(*redir, "redir");
        TORCH_CHECK(redir->dim() == 4 && redir->size(0) == s.B && redir->size(2) == s.oH && redir->size(3) == s.oW,
                    "CorrelationCat: redir ", redir->sizes(), " does not match the correlation output [", s.B, ", D, ",
                    s.oH, ", ", s.oW, "]");
    }
    at::Tensor cat, ws;
    int rc;
    {
        c10::cuda::CUDAGuard guard(input1.device());
        at::Tensor a = f32c(input1), b = f32c(input2);
        cat = at::empty({s.B, R + s.D, s.oH, s.oW}, a.options());
        if (redir) cat.narrow(1, 0, R).copy_(*redir);
        // the tensor-core path's bf16 hi/lo operands (the analogue of the reference's rbot1/rbot2, correlation.py:20-21);
        // returned so that the backward can skip the split pass
        const size_t wsb = fn2b200_correlation_forward_workspace(s.B, s.C, s.H, s.W, pad, k, md, s1, s2);
        ws = at::empty({(int64_t)wsb}, a.options().dtype(at::kByte));
        rc = fn2b200_correlation_forward_cat(fptr(a), fptr(b), fptr(cat), R + s.D, R, (float)leaky, s.B, s.C, s.H, s.W, pad,
                                             k, md, s1, s2, mul, ptr(ws), wsb, stream_of(a));
    }
    check(rc, who);
    return {cat, ws};
}

// Input gradients of cat[:, ch_offset : ch_offset + D] = LeakyReLU(leaky)(correlation); no cat: the plain correlation.
// `workspace` is what the forward returned for the same inputs (autograd's version counter rules out in-place changes
// of saved inputs), or an empty tensor: the split pass is skipped when it is large enough.
std::tuple<at::Tensor, at::Tensor> corr_backward(const at::Tensor &input1, const at::Tensor &input2, const at::Tensor &grad,
                                                 const at::Tensor *cat, const at::Tensor &workspace, int64_t ch_offset,
                                                 double leaky, int64_t pad, int64_t k, int64_t md, int64_t s1, int64_t s2,
                                                 int64_t mul, bool need1, bool need2, const char *who) {
    const CorrShape s = corr_shape(input1, input2, pad, k, md, s1, s2);
    need_cuda(grad, "grad");
    if (cat) {
        TORCH_CHECK(grad.dim() == 4 && grad.size(0) == s.B && grad.size(2) == s.oH && grad.size(3) == s.oW, who,
                    ": grad_cat shape ", grad.sizes(), " does not match [", s.B, ", channels, ", s.oH, ", ", s.oW, "]");
        need_out(*cat, "cat");
        TORCH_CHECK(cat->sizes() == grad.sizes() && cat->device() == input1.device(), who, ": cat ", cat->sizes(),
                    " must have grad_cat's shape ", grad.sizes());
    } else {
        TORCH_CHECK(grad.dim() == 4 && grad.size(0) == s.B && grad.size(1) == s.D && grad.size(2) == s.oH &&
                    grad.size(3) == s.oW, who, ": grad_output shape ", grad.sizes(), " != expected [", s.B, ", ", s.D,
                    ", ", s.oH, ", ", s.oW, "]");
    }
    at::Tensor g1, g2;
    int rc;
    {
        c10::cuda::CUDAGuard guard(input1.device());
        at::Tensor a = f32c(input1), b = f32c(input2), g = f32c(grad);
        g1 = need1 ? at::empty_like(a) : none_like(a);
        g2 = need2 ? at::empty_like(b) : none_like(b);
        const size_t wsb = fn2b200_correlation_backward_workspace(s.B, s.C, s.H, s.W, pad, k, md, s1, s2);
        const bool have = wsb && workspace.scalar_type() == at::kByte && workspace.device() == a.device() &&
                          (size_t)workspace.numel() >= wsb;
        at::Tensor ws = have ? workspace : at::empty({(int64_t)wsb}, a.options().dtype(at::kByte));
        rc = fn2b200_correlation_backward_cat(fptr(a), fptr(b), fptr(g), cat ? fptr(*cat) : nullptr,
                                              cat ? (int)grad.size(1) : s.D, ch_offset, (float)leaky, fptr(g1), fptr(g2),
                                              s.B, s.C, s.H, s.W, pad, k, md, s1, s2, mul, ptr(ws), wsb, have ? 1 : 0,
                                              stream_of(a));
    }
    check(rc, who);
    return {g1, g2};
}

std::tuple<at::Tensor, at::Tensor> correlation_forward(const at::Tensor &input1, const at::Tensor &input2, int64_t pad,
                                                       int64_t k, int64_t md, int64_t s1, int64_t s2, int64_t mul) {
    return corr_forward(nullptr, input1, input2, pad, k, md, s1, s2, mul, 1.0, "correlation_forward");
}

std::tuple<at::Tensor, at::Tensor> correlation_backward(const at::Tensor &input1, const at::Tensor &input2,
                                                        const at::Tensor &grad_output, const at::Tensor &workspace,
                                                        int64_t pad, int64_t k, int64_t md, int64_t s1, int64_t s2,
                                                        int64_t mul, bool need1, bool need2) {
    return corr_backward(input1, input2, grad_output, nullptr, workspace, 0, 1.0, pad, k, md, s1, s2, mul, need1, need2,
                         "correlation_backward");
}

std::tuple<at::Tensor, at::Tensor> correlation_forward_cat(const at::Tensor &redir, const at::Tensor &input1,
                                                           const at::Tensor &input2, int64_t pad, int64_t k, int64_t md,
                                                           int64_t s1, int64_t s2, int64_t mul, double leaky_slope) {
    return corr_forward(&redir, input1, input2, pad, k, md, s1, s2, mul, leaky_slope, "correlation_forward_cat");
}

std::tuple<at::Tensor, at::Tensor> correlation_backward_cat(const at::Tensor &input1, const at::Tensor &input2,
                                                            const at::Tensor &grad_cat, const at::Tensor &cat,
                                                            const at::Tensor &workspace, int64_t ch_offset,
                                                            double leaky_slope, int64_t pad, int64_t k, int64_t md,
                                                            int64_t s1, int64_t s2, int64_t mul, bool need1, bool need2) {
    return corr_backward(input1, input2, grad_cat, &cat, workspace, ch_offset, leaky_slope, pad, k, md, s1, s2, mul, need1,
                         need2, "correlation_backward_cat");
}

// ---- Resample2d --------------------------------------------------------------------------------------------------

at::Tensor resample2d_forward(const at::Tensor &input1, const at::Tensor &input2, int64_t kernel_size, bool bilinear) {
    need_cuda(input1, "input1"); need_cuda(input2, "input2");
    TORCH_CHECK(input1.dim() == 4 && input2.dim() == 4 && input2.size(1) == 2,
                "resample2d: expected image [B,C,H,W] and flow [B,2,H,W], got ", input1.sizes(), " and ", input2.sizes());
    TORCH_CHECK(input1.size(0) >= input2.size(0), "resample2d: image batch ", input1.size(0), " smaller than flow batch ",
                input2.size(0));
    at::Tensor out;
    int rc;
    {
        c10::cuda::CUDAGuard guard(input2.device());
        at::Tensor img = f32(input1), flow = f32c(input2);
        const int B = flow.size(0), C = img.size(1), H = flow.size(2), W = flow.size(3);
        out = at::empty({B, C, H, W}, flow.options());
        rc = fn2b200_resample2d_forward(fptr(img), strides4(img).data(), fptr(flow), fptr(out), B, C, img.size(2),
                                        img.size(3), H, W, kernel_size, bilinear ? 1 : 0, stream_of(flow));
    }
    check(rc, "resample2d_forward");
    return out;
}

std::tuple<at::Tensor, at::Tensor> resample2d_backward(const at::Tensor &input1, const at::Tensor &input2,
                                                       const at::Tensor &grad_output, int64_t kernel_size, bool bilinear,
                                                       bool need1, bool need2) {
    need_cuda(input1, "input1"); need_cuda(input2, "input2"); need_cuda(grad_output, "grad_output");
    TORCH_CHECK(input1.dim() == 4 && input2.dim() == 4 && input2.size(1) == 2,
                "resample2d_backward: expected image [B,C,H,W] and flow [B,2,H,W], got ", input1.sizes(), " and ",
                input2.sizes());
    const int64_t B = input2.size(0), C = input1.size(1), H = input2.size(2), W = input2.size(3);
    TORCH_CHECK(grad_output.sizes() == at::IntArrayRef({B, C, H, W}), "resample2d_backward: grad_output shape ",
                grad_output.sizes(), " != expected [", B, ", ", C, ", ", H, ", ", W, "]");
    at::Tensor g1, g2;
    int rc;
    {
        c10::cuda::CUDAGuard guard(input2.device());
        at::Tensor img = f32(input1), flow = f32c(input2), g = f32c(grad_output);
        const int iH = img.size(2), iW = img.size(3);
        g1 = need1 ? at::empty(img.sizes(), flow.options()) : none_like(flow);
        if (need1 && img.size(0) != B) g1.zero_();     // rows the flow batch does not touch stay zero
        g2 = need2 ? at::empty_like(flow) : none_like(flow);
        const auto is = strides4(img);
        // pixel-interleaved accumulator of the image gradient (the library zero-fills it on the stream)
        const size_t wsb = need1 ? fn2b200_resample2d_backward_workspace(is.data(), B, C, iH, iW, H, W) : 0;
        at::Tensor ws = at::empty({(int64_t)wsb}, flow.options().dtype(at::kByte));
        rc = fn2b200_resample2d_backward_ws(fptr(img), is.data(), fptr(flow), fptr(g), fptr(g1), fptr(g2), B, C, iH, iW, H,
                                            W, kernel_size, bilinear ? 1 : 0, 1, ptr(ws), wsb, stream_of(flow));
    }
    check(rc, "resample2d_backward");
    return {g1, g2};
}

// ---- ChannelNorm (fp32, and fp16 / bf16 storage natively) ---------------------------------------------------------

at::Tensor channelnorm_forward(const at::Tensor &input1, int64_t norm_deg) {
    need_cuda(input1, "input1");
    TORCH_CHECK(input1.dim() == 4, "channelnorm: expected a 4-D tensor, got ", input1.sizes());
    at::Tensor out;
    int rc;
    {
        c10::cuda::CUDAGuard guard(input1.device());
        const int dt = dtype16(input1);
        at::Tensor a = dt ? input1.contiguous() : f32c(input1);
        const int B = a.size(0), C = a.size(1), H = a.size(2), W = a.size(3);
        out = at::empty({B, 1, H, W}, a.options());
        rc = dt ? fn2b200_channelnorm_forward_16(ptr(a), ptr(out), B, C, H, W, norm_deg, dt, stream_of(a))
                : fn2b200_channelnorm_forward(fptr(a), fptr(out), B, C, H, W, norm_deg, stream_of(a));
    }
    check(rc, "channelnorm_forward");
    return out;
}

at::Tensor channelnorm_backward(const at::Tensor &input1, const at::Tensor &output, const at::Tensor &grad_output,
                                int64_t norm_deg) {
    need_cuda(input1, "input1"); need_cuda(output, "output"); need_cuda(grad_output, "grad_output");
    TORCH_CHECK(input1.dim() == 4 && output.dim() == 4 && grad_output.sizes() == output.sizes() &&
                output.size(0) == input1.size(0) && output.size(1) == 1 && output.size(2) == input1.size(2) &&
                output.size(3) == input1.size(3), "channelnorm_backward: shapes input1 ", input1.sizes(), ", output ",
                output.sizes(), ", grad_output ", grad_output.sizes(), " do not match");
    at::Tensor gi;
    int rc;
    {
        c10::cuda::CUDAGuard guard(input1.device());
        const int dt = output.scalar_type() == input1.scalar_type() && grad_output.scalar_type() == input1.scalar_type()
                       ? dtype16(input1) : 0;
        at::Tensor a = dt ? input1.contiguous() : f32c(input1), o = dt ? output.contiguous() : f32c(output),
                   g = dt ? grad_output.contiguous() : f32c(grad_output);
        const int B = a.size(0), C = a.size(1), H = a.size(2), W = a.size(3);
        gi = at::empty_like(a);
        rc = dt ? fn2b200_channelnorm_backward_16(ptr(a), ptr(o), ptr(g), ptr(gi), B, C, H, W, norm_deg, dt, stream_of(a))
                : fn2b200_channelnorm_backward(fptr(a), fptr(o), fptr(g), fptr(gi), B, C, H, W, norm_deg, stream_of(a));
    }
    check(rc, "channelnorm_backward");
    return gi;
}

// ---- warp -> diff -> channel-norm -> concat (include/fn2b200.h: fn2b200_warp_concat_forward) ------------------------

struct WarpLayout { int64_t ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm; };

void warp_concat_into(at::Tensor &cat, const at::Tensor &x, const at::Tensor &flow, int64_t C, int64_t mode, double flow_mul,
                      double flow_div, const WarpLayout &l) {
    at::Tensor xx = f32(x), fl = f32c(flow);
    check(fn2b200_warp_concat_forward(fptr(xx), strides4(xx).data(), C, fptr(fl), fl.size(2), fl.size(3), mode,
                                      (float)flow_mul, fptr(cat), cat.size(1), l.ch_x, l.n_x, l.ch_warped, l.ch_flow,
                                      (float)flow_div, l.ch_flow_norm, l.ch_diff_norm, cat.size(0), cat.size(2),
                                      cat.size(3), stream_of(fl)),
          "warp_concat_forward");
}

void warp_concat_args(const at::Tensor &x, const at::Tensor &flow, int64_t C, const char *who) {
    need_cuda(x, "x"); need_cuda(flow, "flow");
    TORCH_CHECK(x.dim() == 4 && flow.dim() == 4 && flow.size(1) == 2 && x.size(1) >= 2 * C && x.size(0) == flow.size(0), who,
                ": expected x [B,>=2C,H,W] and flow [B,2,h,w], got ", x.sizes(), " and ", flow.sizes());
}

at::Tensor warp_concat_forward(const at::Tensor &x, const at::Tensor &flow, int64_t C, int64_t upsample_mode,
                               double flow_mul, double flow_div, int64_t cat_channels, int64_t ch_x, int64_t n_x,
                               int64_t ch_warped, int64_t ch_flow, int64_t ch_flow_norm, int64_t ch_diff_norm) {
    warp_concat_args(x, flow, C, "warp_concat_forward");
    c10::cuda::CUDAGuard guard(flow.device());
    // channels no product covers (the C ABI refuses overlapping ranges) are zero: the op's output is fully defined
    const int64_t covered = (ch_x >= 0 ? n_x : 0) + (ch_warped >= 0 ? C : 0) + (ch_flow >= 0 ? 2 : 0) +
                            (ch_flow_norm >= 0) + (ch_diff_norm >= 0);
    const auto opt = flow.options().dtype(at::kFloat);
    at::Tensor cat = covered < cat_channels ? at::zeros({x.size(0), cat_channels, x.size(2), x.size(3)}, opt)
                                            : at::empty({x.size(0), cat_channels, x.size(2), x.size(3)}, opt);
    warp_concat_into(cat, x, flow, C, upsample_mode, flow_mul, flow_div,
                     {ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm});
    return cat;
}

std::tuple<at::Tensor, at::Tensor> warp_concat_backward_impl(const at::Tensor &x, const at::Tensor &flow,
                                                             const at::Tensor &grad_cat, int64_t C, int64_t mode,
                                                             double flow_mul, double flow_div, const WarpLayout &l,
                                                             bool need_x, bool need_flow) {
    warp_concat_args(x, flow, C, "warp_concat_backward");
    need_cuda(grad_cat, "grad_cat");
    const int64_t B = flow.size(0), fh = flow.size(2), fw = flow.size(3);
    const int64_t H = mode == 0 ? fh : 4 * fh, W = mode == 0 ? fw : 4 * fw;
    TORCH_CHECK(x.size(2) == H && x.size(3) == W && grad_cat.dim() == 4 && grad_cat.size(0) == B &&
                grad_cat.size(2) == H && grad_cat.size(3) == W, "warp_concat_backward: shapes x ", x.sizes(), ", flow ",
                flow.sizes(), ", grad_cat ", grad_cat.sizes(), " do not match");
    at::Tensor gx, gf;
    int rc;
    {
        c10::cuda::CUDAGuard guard(flow.device());
        at::Tensor xx = f32(x), fl = f32c(flow), gc = f32c(grad_cat);
        gx = need_x ? at::empty({B, 2 * C, H, W}, fl.options()) : none_like(fl);
        gf = need_flow ? at::empty_like(fl) : none_like(fl);
        const size_t wsb = fn2b200_warp_concat_backward_up_workspace(B, C, H, W, mode, need_x ? 1 : 0);
        at::Tensor ws = scratch(wsb, fl);
        rc = fn2b200_warp_concat_backward_up(fptr(xx), strides4(xx).data(), C, fptr(fl), fh, fw, mode, (float)flow_mul,
                                             fptr(gc), gc.size(1), l.ch_x, l.n_x, l.ch_warped, l.ch_flow, (float)flow_div,
                                             l.ch_flow_norm, l.ch_diff_norm, fptr(gx), fptr(gf), ptr(ws), wsb, B, H, W,
                                             stream_of(fl));
    }
    check(rc, "warp_concat_backward");
    return {gx, gf};
}

std::tuple<at::Tensor, at::Tensor> warp_concat_backward(const at::Tensor &x, const at::Tensor &flow,
                                                        const at::Tensor &grad_cat, int64_t C, int64_t upsample_mode,
                                                        double flow_mul, double flow_div, int64_t ch_x, int64_t n_x,
                                                        int64_t ch_warped, int64_t ch_flow, int64_t ch_flow_norm,
                                                        int64_t ch_diff_norm, bool need_x, bool need_flow) {
    return warp_concat_backward_impl(x, flow, grad_cat, C, upsample_mode, flow_mul, flow_div,
                                     {ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm}, need_x, need_flow);
}

// concat3 of models.py:179: (img0 | sd flow | s2 flow | |sd flow| | |s2 flow| | sd diff norm | s2 diff norm), each flow
// the nearest x4 upsample of its quarter-resolution flow2 (sd: / div_flow, models.py:167; s2: * div_flow, :154)
constexpr WarpLayout FUSION_SD{0, 3, -1, 3, 7, 9}, FUSION_S2{-1, 0, -1, 5, 8, 10};
constexpr int64_t FUSION_CHANNELS = 11, NEAREST = 2;

at::Tensor fusion_concat(const at::Tensor &x, const at::Tensor &sd_flow2, const at::Tensor &s2_flow2, double div_flow) {
    warp_concat_args(x, sd_flow2, 3, "fusion_concat");
    warp_concat_args(x, s2_flow2, 3, "fusion_concat");
    c10::cuda::CUDAGuard guard(x.device());
    at::Tensor cat = at::empty({x.size(0), FUSION_CHANNELS, x.size(2), x.size(3)}, x.options().dtype(at::kFloat));
    warp_concat_into(cat, x, sd_flow2, 3, NEAREST, 1.0 / div_flow, 1.0, FUSION_SD);
    warp_concat_into(cat, x, s2_flow2, 3, NEAREST, div_flow, 1.0, FUSION_S2);
    return cat;
}

// two warp_concat backward passes, each reading its own channels of grad_cat; the x gradients summed
std::tuple<at::Tensor, at::Tensor, at::Tensor> fusion_concat_backward(const at::Tensor &x, const at::Tensor &sd_flow2,
                                                                      const at::Tensor &s2_flow2, const at::Tensor &grad_cat,
                                                                      double div_flow, bool need_x, bool need_sd,
                                                                      bool need_s2) {
    at::Tensor gx = none_like(x), g_sd = none_like(x), g_s2 = none_like(x), gx2;
    if (need_x || need_sd)
        std::tie(gx, g_sd) = warp_concat_backward_impl(x, sd_flow2, grad_cat, 3, NEAREST, 1.0 / div_flow, 1.0, FUSION_SD,
                                                       need_x, need_sd);
    if (need_x || need_s2) {
        std::tie(gx2, g_s2) = warp_concat_backward_impl(x, s2_flow2, grad_cat, 3, NEAREST, div_flow, 1.0, FUSION_S2,
                                                        need_x, need_s2);
        if (need_x) gx.add_(gx2);
    }
    return {gx, g_sd, g_s2};
}

}  // namespace

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
    m.impl("correlation_forward", &correlation_forward);
    m.impl("correlation_backward", &correlation_backward);
    m.impl("correlation_forward_cat", &correlation_forward_cat);
    m.impl("correlation_backward_cat", &correlation_backward_cat);
    m.impl("resample2d_forward", &resample2d_forward);
    m.impl("resample2d_backward", &resample2d_backward);
    m.impl("channelnorm_forward", &channelnorm_forward);
    m.impl("channelnorm_backward", &channelnorm_backward);
    m.impl("warp_concat_forward", &warp_concat_forward);
    m.impl("warp_concat_backward", &warp_concat_backward);
    m.impl("fusion_concat", &fusion_concat);
    m.impl("fusion_concat_backward", &fusion_concat_backward);
}

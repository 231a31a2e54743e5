// ext_common.h -- the host side of every op, shared by the operator library (fn2b200_ops.cc: torch.ops.fn2b200.* and
// the functions flownet2_b200.functional calls) and by the reference-named extension modules correlation_cuda /
// resample2d_cuda / channelnorm_cuda.  One function per op and direction does everything between "tensors arrive" and
// "status checked": device and shape checks, the conversion to fp32 / contiguous, the checks on caller-supplied outputs,
// the device guard and current stream, workspace sizing and allocation, the C-ABI call and the exception carrying the
// library's message.  No arithmetic lives here; everything is forwarded to libfn2b200.so (include/fn2b200.h).
#pragma once
#include <torch/extension.h>

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include "fn2b200.h"

namespace fn2ext {

using Opt = std::optional<at::Tensor>;
using Grads = std::tuple<at::Tensor, at::Tensor>;

inline void check(int rc, const char *what) {
    // the reference raises AT_ERROR("CUDA call failed") (correlation_cuda.cc:81-83); we add the library's message
    TORCH_CHECK(rc == 0, what, " failed (status ", rc, "): ", fn2b200_last_error());
}
inline void need_cuda(const at::Tensor &t, const char *name) {
    TORCH_CHECK(t.is_cuda(), "flownet2-pytorch_b200 runs on CUDA tensors only (", name, " is a ", t.device().type(),
                " tensor); there is no CPU fallback -- the reference has none either (correlation.py:4)");
}
inline void need_cuda(const Opt &t, const char *name) {
    if (t) need_cuda(*t, name);
}
// the reference's extension modules take float32 only
inline void need_cuda_f32(const at::Tensor &t, const char *name) {
    need_cuda(t, name);
    TORCH_CHECK(t.scalar_type() == at::kFloat, name, " must be float32 (got ", t.scalar_type(), ")");
}
inline void *ptr(const at::Tensor &t) { return t.defined() && t.numel() ? t.data_ptr() : nullptr; }
inline float *fptr(const at::Tensor &t) { return static_cast<float *>(ptr(t)); }
inline at::Tensor f32(const at::Tensor &t) { return t.to(at::kFloat); }                  // strided views kept as they are
inline at::Tensor f32c(const at::Tensor &t) { return t.to(at::kFloat).contiguous(); }
inline std::array<int64_t, 4> strides4(const at::Tensor &t) { return {t.stride(0), t.stride(1), t.stride(2), t.stride(3)}; }
inline void *stream_of(const at::Tensor &t) { return at::cuda::getCurrentCUDAStream(t.get_device()).stream(); }
inline at::Tensor bytes(size_t n, const at::Tensor &like) { return at::empty({(int64_t)n}, like.options().dtype(at::kByte)); }
// the C ABI's dtype code of a 16-bit tensor (1 = fp16, 2 = bf16), 0 for anything else
inline int dtype16(const at::Tensor &t) { return t.scalar_type() == at::kHalf ? 1 : (t.scalar_type() == at::kBFloat16 ? 2 : 0); }

// `out` when the caller supplied one, else a new tensor.  A supplied output reaches the C ABI as a raw pointer: anything
// the kernels would overrun or misread (wrong shape, dtype or device, a strided view) is refused.
inline at::Tensor output(const Opt &out, at::IntArrayRef shape, at::ScalarType dtype, const at::Tensor &like, const char *who,
                         const char *name) {
    if (!out) return at::empty(shape, like.options().dtype(dtype));
    const at::Tensor &t = *out;
    TORCH_CHECK(t.scalar_type() == dtype && t.is_contiguous() && t.device() == like.device() && t.sizes() == shape, who,
                ": ", name, " must be a contiguous ", dtype, " tensor of shape ", shape, " on ", like.device(), " (got ",
                t.scalar_type(), " ", t.sizes(), " on ", t.device(), ", contiguous=", t.is_contiguous(), ")");
    return t;
}

// ---- correlation -------------------------------------------------------------------------------------------------

struct CorrShape { int B, C, H, W, D, oH, oW; };

// The input checks of every correlation call and the output geometry (fn2b200_correlation_out_shape's float ceil).
inline CorrShape corr_shape(const at::Tensor &input1, const at::Tensor &input2, int64_t pad, int64_t k, int64_t md,
                            int64_t s1, int64_t s2) {
    TORCH_CHECK(input1.dim() == 4 && input1.sizes() == input2.sizes(),
                "correlation: input1/input2 must be 4-D with equal shapes, got ", input1.sizes(), " and ", input2.sizes());
    CorrShape s{(int)input1.size(0), (int)input1.size(1), (int)input1.size(2), (int)input1.size(3), 0, 0, 0};
    check(fn2b200_correlation_out_shape(s.C, s.H, s.W, pad, k, md, s1, s2, &s.D, &s.oH, &s.oW), "correlation_out_shape");
    TORCH_CHECK(s.oH > 0 && s.oW > 0, "correlation: empty output (", s.oH, " x ", s.oW, ") for input ", s.H, "x", s.W,
                ", pad_size=", pad, ", max_displacement=", md, ", kernel_size=", k);
    return s;
}

// cat = false: the plain correlation into out [B, D, oH, oW] (allocated when absent); ch_offset 0, leaky_slope 1.
// cat = true: LeakyReLU(leaky_slope)(correlation) into channels [ch_offset, ch_offset + D) of out [B, channels, oH, oW];
// its other channels are left alone.  Returns (out, workspace): the tensor-core path's bf16 hi/lo split of both inputs
// (the analogue of the reference's rbot1/rbot2, correlation.py:20-21), empty when the FP32-FMA kernels run.
inline std::tuple<at::Tensor, at::Tensor> correlation_forward(const at::Tensor &input1, const at::Tensor &input2,
                                                              const Opt &out, bool cat, int64_t ch_offset,
                                                              double leaky_slope, int64_t pad, int64_t k, int64_t md,
                                                              int64_t s1, int64_t s2, int64_t mul) {
    const char *who = cat ? "correlation_forward_cat" : "correlation_forward";
    need_cuda(input1, "input1"); need_cuda(input2, "input2"); need_cuda(out, "output");
    const CorrShape s = corr_shape(input1, input2, pad, k, md, s1, s2);
    TORCH_CHECK(!cat || (out && out->dim() == 4), who, ": the concat output must be a 4-D tensor");
    c10::cuda::CUDAGuard guard(input1.device());
    at::Tensor a = f32c(input1), b = f32c(input2);
    at::Tensor o = output(out, {s.B, cat ? out->size(1) : s.D, s.oH, s.oW}, at::kFloat, a, who, "output");
    const size_t wsb = fn2b200_correlation_forward_workspace(s.B, s.C, s.H, s.W, pad, k, md, s1, s2);
    at::Tensor ws = bytes(wsb, a);
    check(fn2b200_correlation_forward_cat(fptr(a), fptr(b), fptr(o), o.size(1), ch_offset, (float)leaky_slope, s.B, s.C,
                                          s.H, s.W, pad, k, md, s1, s2, mul, ptr(ws), wsb, stream_of(a)),
          who);
    return {o, ws};
}

// The input gradients (need1 / need2; an undefined tensor for one not asked for) of the plain correlation (cat = false,
// grad [B, D, oH, oW]), or of cat[:, ch_offset : ch_offset + D] = LeakyReLU(leaky_slope)(correlation) read straight
// from the concat's gradient grad [B, channels, oH, oW] (cat = true), LeakyReLU's derivative taken from act, the buffer
// the forward wrote (may be absent when leaky_slope == 1).  `workspace` is the forward's, still holding the split of
// these very inputs, or absent: the tensor-core backward skips the split pass when it is large enough.
inline Grads correlation_backward(const at::Tensor &input1, const at::Tensor &input2, const at::Tensor &grad, bool cat,
                                  const Opt &act, int64_t ch_offset, double leaky_slope, const Opt &workspace, int64_t pad,
                                  int64_t k, int64_t md, int64_t s1, int64_t s2, int64_t mul, bool need1, bool need2,
                                  const Opt &out1, const Opt &out2) {
    const char *who = cat ? "correlation_backward_cat" : "correlation_backward";
    need_cuda(input1, "input1"); need_cuda(input2, "input2"); need_cuda(grad, "grad_output"); need_cuda(act, "cat");
    need_cuda(out1, "grad_input1"); need_cuda(out2, "grad_input2");
    const CorrShape s = corr_shape(input1, input2, pad, k, md, s1, s2);
    if (cat) {
        TORCH_CHECK(grad.dim() == 4 && grad.size(0) == s.B && grad.size(2) == s.oH && grad.size(3) == s.oW, who,
                    ": grad_cat shape ", grad.sizes(), " does not match [", s.B, ", channels, ", s.oH, ", ", s.oW, "]");
    } else {
        TORCH_CHECK(grad.sizes() == at::IntArrayRef({s.B, s.D, s.oH, s.oW}), who, ": grad_output shape ", grad.sizes(),
                    " != expected [", s.B, ", ", s.D, ", ", s.oH, ", ", s.oW, "] (pad_size=", pad, ", kernel_size=", k,
                    ", max_displacement=", md, ", stride1=", s1, ", stride2=", s2, ")");
    }
    c10::cuda::CUDAGuard guard(input1.device());
    at::Tensor a = f32c(input1), b = f32c(input2), g = f32c(grad);
    if (act) output(act, g.sizes(), at::kFloat, a, who, "cat");
    at::Tensor g1 = need1 ? output(out1, a.sizes(), at::kFloat, a, who, "grad_input1") : at::Tensor();
    at::Tensor g2 = need2 ? output(out2, b.sizes(), at::kFloat, a, who, "grad_input2") : at::Tensor();
    const size_t wsb = fn2b200_correlation_backward_workspace(s.B, s.C, s.H, s.W, pad, k, md, s1, s2);
    const bool has_split = wsb && workspace && workspace->scalar_type() == at::kByte &&
                           workspace->device() == a.device() && (size_t)workspace->numel() >= wsb;
    at::Tensor ws = has_split ? *workspace : bytes(wsb, a);
    check(fn2b200_correlation_backward_cat(fptr(a), fptr(b), fptr(g), act ? fptr(*act) : nullptr, g.size(1), ch_offset,
                                           (float)leaky_slope, fptr(g1), fptr(g2), s.B, s.C, s.H, s.W, pad, k, md, s1, s2,
                                           mul, ptr(ws), wsb, has_split, stream_of(a)),
          who);
    return {g1, g2};
}

// ---- Resample2d --------------------------------------------------------------------------------------------------

// upsample_mode 0: Resample2d()(input1, input2) -> [B, C, h, w] on the flow's grid; the image may be larger than the
// flow and may be a strided view.  1 / 2: Resample2d()(input1, nn.Upsample(scale_factor=4, mode=bilinear / nearest)(
// input2 * flow_mul)) -> [B, C, H, W] on the image's grid, the quarter-resolution flow interpolated per pixel.
inline at::Tensor resample2d_forward(const at::Tensor &input1, const at::Tensor &input2, const Opt &out,
                                     int64_t kernel_size, bool bilinear, int64_t upsample_mode, double flow_mul) {
    const char *who = upsample_mode ? "resample2d_forward_up" : "resample2d_forward";
    need_cuda(input1, "input1"); need_cuda(input2, "input2"); need_cuda(out, "output");
    TORCH_CHECK(input1.dim() == 4 && input2.dim() == 4 && input2.size(1) == 2,
                who, ": expected image [B,C,H,W] and flow [B,2,h,w], got ", input1.sizes(), " and ", input2.sizes());
    TORCH_CHECK(input1.size(0) >= input2.size(0), who, ": image batch ", input1.size(0), " smaller than flow batch ",
                input2.size(0));
    c10::cuda::CUDAGuard guard(input2.device());
    at::Tensor img = f32(input1), flow = f32c(input2);
    const int B = flow.size(0), C = img.size(1), iH = img.size(2), iW = img.size(3), fh = flow.size(2), fw = flow.size(3);
    const int H = upsample_mode ? iH : fh, W = upsample_mode ? iW : fw;
    at::Tensor o = output(out, {B, C, H, W}, at::kFloat, flow, who, "output");
    const auto is = strides4(img);
    check(upsample_mode ? fn2b200_resample2d_forward_up(fptr(img), is.data(), fptr(flow), fh, fw, upsample_mode,
                                                        (float)flow_mul, fptr(o), B, C, H, W, stream_of(flow))
                        : fn2b200_resample2d_forward(fptr(img), is.data(), fptr(flow), fptr(o), B, C, iH, iW, H, W,
                                                     kernel_size, bilinear ? 1 : 0, stream_of(flow)),
          who);
    return o;
}

// The gradients (need1 / need2) of resample2d_forward with upsample_mode 0.  zero_grad_input1 = false accumulates
// into a caller-zeroed grad_input1 (resample2d.py:31).  Image rows beyond the flow batch get no gradient: they are zero.
inline Grads resample2d_backward(const at::Tensor &input1, const at::Tensor &input2, const at::Tensor &grad,
                                 int64_t kernel_size, bool bilinear, bool need1, bool need2, const Opt &out1,
                                 const Opt &out2, bool zero_grad_input1) {
    const char *who = "resample2d_backward";
    need_cuda(input1, "input1"); need_cuda(input2, "input2"); need_cuda(grad, "grad_output");
    need_cuda(out1, "grad_input1"); need_cuda(out2, "grad_input2");
    TORCH_CHECK(input1.dim() == 4 && input2.dim() == 4 && input2.size(1) == 2,
                who, ": expected image [B,C,H,W] and flow [B,2,h,w], got ", input1.sizes(), " and ", input2.sizes());
    const int64_t B = input2.size(0), C = input1.size(1), H = input2.size(2), W = input2.size(3);
    TORCH_CHECK(input1.size(0) >= B, who, ": image batch ", input1.size(0), " smaller than flow batch ", B);
    TORCH_CHECK(grad.sizes() == at::IntArrayRef({B, C, H, W}), who, ": grad_output shape ", grad.sizes(),
                " != expected [", B, ", ", C, ", ", H, ", ", W, "]");
    c10::cuda::CUDAGuard guard(input2.device());
    at::Tensor img = f32(input1), flow = f32c(input2), g = f32c(grad);
    at::Tensor g1 = need1 ? output(out1, img.sizes(), at::kFloat, flow, who, "grad_input1") : at::Tensor();
    if (need1 && img.size(0) != B) g1.zero_();
    at::Tensor g2 = need2 ? output(out2, flow.sizes(), at::kFloat, flow, who, "grad_input2") : at::Tensor();
    const auto is = strides4(img);
    // pixel-interleaved accumulator of the image gradient (the library zero-fills it on the stream)
    const size_t wsb = need1 ? fn2b200_resample2d_backward_workspace(is.data(), B, C, img.size(2), img.size(3), H, W) : 0;
    at::Tensor ws = bytes(wsb, flow);
    check(fn2b200_resample2d_backward_ws(fptr(img), is.data(), fptr(flow), fptr(g), fptr(g1), fptr(g2), B, C, img.size(2),
                                         img.size(3), H, W, kernel_size, bilinear ? 1 : 0, zero_grad_input1 ? 1 : 0,
                                         ptr(ws), wsb, stream_of(flow)),
          who);
    return {g1, g2};
}

// ---- ChannelNorm (fp32, and fp16 / bf16 storage natively) ---------------------------------------------------------

// fp16 / bf16 inputs run natively (the reference dispatches its kernels on half too); anything else as fp32.
inline at::Tensor channelnorm_forward(const at::Tensor &input1, const Opt &out, int64_t norm_deg) {
    const char *who = "channelnorm_forward";
    need_cuda(input1, "input1"); need_cuda(out, "output");
    TORCH_CHECK(input1.dim() == 4, who, ": expected a 4-D tensor, got ", input1.sizes());
    c10::cuda::CUDAGuard guard(input1.device());
    const int dt = dtype16(input1);
    at::Tensor a = dt ? input1.contiguous() : f32c(input1);
    const int B = a.size(0), C = a.size(1), H = a.size(2), W = a.size(3);
    at::Tensor o = output(out, {B, 1, H, W}, a.scalar_type(), a, who, "output");
    check(dt ? fn2b200_channelnorm_forward_16(ptr(a), ptr(o), B, C, H, W, norm_deg, dt, stream_of(a))
             : fn2b200_channelnorm_forward(fptr(a), fptr(o), B, C, H, W, norm_deg, stream_of(a)),
          who);
    return o;
}

// Natively 16-bit when input1, output and grad_output share an fp16 / bf16 dtype; fp32 otherwise.
inline at::Tensor channelnorm_backward(const at::Tensor &input1, const at::Tensor &output_, const at::Tensor &grad,
                                       const Opt &out, int64_t norm_deg) {
    const char *who = "channelnorm_backward";
    need_cuda(input1, "input1"); need_cuda(output_, "output"); need_cuda(grad, "grad_output");
    need_cuda(out, "grad_input1");
    TORCH_CHECK(input1.dim() == 4 && output_.dim() == 4 && grad.sizes() == output_.sizes() &&
                output_.size(0) == input1.size(0) && output_.size(1) == 1 && output_.size(2) == input1.size(2) &&
                output_.size(3) == input1.size(3), who, ": shapes input1 ", input1.sizes(), ", output ", output_.sizes(),
                ", grad_output ", grad.sizes(), " do not match");
    c10::cuda::CUDAGuard guard(input1.device());
    const int dt = output_.scalar_type() == input1.scalar_type() && grad.scalar_type() == input1.scalar_type()
                   ? dtype16(input1) : 0;
    at::Tensor a = dt ? input1.contiguous() : f32c(input1), o = dt ? output_.contiguous() : f32c(output_),
               g = dt ? grad.contiguous() : f32c(grad);
    const int B = a.size(0), C = a.size(1), H = a.size(2), W = a.size(3);
    at::Tensor gi = output(out, a.sizes(), a.scalar_type(), a, who, "grad_input1");
    check(dt ? fn2b200_channelnorm_backward_16(ptr(a), ptr(o), ptr(g), ptr(gi), B, C, H, W, norm_deg, dt, stream_of(a))
             : fn2b200_channelnorm_backward(fptr(a), fptr(o), fptr(g), fptr(gi), B, C, H, W, norm_deg, stream_of(a)),
          who);
    return gi;
}

// ---- warp -> diff -> channel-norm -> concat (include/fn2b200.h: fn2b200_warp_concat_forward) ------------------------

struct WarpLayout { int64_t ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm; };

// x [>= B, >= 2C, H, W] (may be a strided view) and flow [B, 2, h, w] (h, w = H, W, or H/4, W/4 with an upsample).
inline void warp_concat_inputs(const at::Tensor &x, const at::Tensor &flow, int64_t C, const char *who) {
    TORCH_CHECK(x.dim() == 4 && flow.dim() == 4 && flow.size(1) == 2 && x.size(1) >= 2 * C && x.size(0) >= flow.size(0),
                who, ": expected x [B,>=2C,H,W] and flow [B,2,h,w], got ", x.sizes(), " and ", flow.sizes());
}

// The products the layout names, written into out [B, cat_channels, H, W] (allocated when absent); channels no product
// covers keep what out held.
inline at::Tensor warp_concat_forward(const at::Tensor &x, const at::Tensor &flow, const Opt &out, int64_t C,
                                      int64_t upsample_mode, double flow_mul, double flow_div, int64_t cat_channels,
                                      const WarpLayout &l) {
    const char *who = "warp_concat_forward";
    need_cuda(x, "x"); need_cuda(flow, "flow"); need_cuda(out, "output");
    warp_concat_inputs(x, flow, C, who);
    TORCH_CHECK(!out || out->dim() == 4, who, ": output must be a 4-D tensor, got ", out->sizes());
    c10::cuda::CUDAGuard guard(flow.device());
    at::Tensor xx = f32(x), fl = f32c(flow);
    const int B = fl.size(0), H = xx.size(2), W = xx.size(3);
    at::Tensor cat = output(out, {B, out ? out->size(1) : cat_channels, H, W}, at::kFloat, fl, who, "output");
    check(fn2b200_warp_concat_forward(fptr(xx), strides4(xx).data(), C, fptr(fl), fl.size(2), fl.size(3), upsample_mode,
                                      (float)flow_mul, fptr(cat), cat.size(1), l.ch_x, l.n_x, l.ch_warped, l.ch_flow,
                                      (float)flow_div, l.ch_flow_norm, l.ch_diff_norm, B, H, W, stream_of(fl)),
          who);
    return cat;
}

// Backward of warp_concat_forward with the same layout: (grad_x [B, 2C, H, W], grad_flow shaped like flow), each an
// undefined tensor when not asked for (need_x / need_flow).
inline Grads warp_concat_backward(const at::Tensor &x, const at::Tensor &flow, const at::Tensor &grad_cat, int64_t C,
                                  int64_t upsample_mode, double flow_mul, double flow_div, const WarpLayout &l, bool need_x,
                                  bool need_flow) {
    const char *who = "warp_concat_backward";
    need_cuda(x, "x"); need_cuda(flow, "flow"); need_cuda(grad_cat, "grad_cat");
    warp_concat_inputs(x, flow, C, who);
    const int64_t B = flow.size(0), fh = flow.size(2), fw = flow.size(3);
    const int64_t H = upsample_mode == 0 ? fh : 4 * fh, W = upsample_mode == 0 ? fw : 4 * fw;
    TORCH_CHECK(x.size(2) == H && x.size(3) == W && grad_cat.dim() == 4 && grad_cat.size(0) == B &&
                grad_cat.size(2) == H && grad_cat.size(3) == W, who, ": shapes x ", x.sizes(), ", flow ", flow.sizes(),
                ", grad_cat ", grad_cat.sizes(), " do not match");
    c10::cuda::CUDAGuard guard(flow.device());
    at::Tensor xx = f32(x), fl = f32c(flow), gc = f32c(grad_cat);
    at::Tensor gx = need_x ? at::empty({B, 2 * C, H, W}, fl.options()) : at::Tensor();
    at::Tensor gf = need_flow ? at::empty_like(fl) : at::Tensor();
    const size_t wsb = fn2b200_warp_concat_backward_up_workspace(B, C, H, W, upsample_mode, need_x ? 1 : 0);
    at::Tensor ws = bytes(std::max<size_t>(wsb, 16), fl);           // 16-byte aligned even when nothing is needed
    check(fn2b200_warp_concat_backward_up(fptr(xx), strides4(xx).data(), C, fptr(fl), fh, fw, upsample_mode,
                                          (float)flow_mul, fptr(gc), gc.size(1), l.ch_x, l.n_x, l.ch_warped, l.ch_flow,
                                          (float)flow_div, l.ch_flow_norm, l.ch_diff_norm, fptr(gx), fptr(gf), ptr(ws),
                                          wsb, B, H, W, stream_of(fl)),
          who);
    return {gx, gf};
}

}  // namespace fn2ext

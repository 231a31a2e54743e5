"""Tensor-level entry points: torch tensors in, C-ABI calls out (device memory + stream plumbing).

These are the functions the autograd wrappers and the ``*_cuda`` shim modules share.  PyTorch is
used for allocation, the current device and the current stream only; all arithmetic happens in
libfn2b200's hand-written sm_90a kernels.
"""
import ctypes

import torch

from ._lib import LIB, check

_I64x4 = ctypes.c_int64 * 4


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "flownet2-pytorch_b200 runs on CUDA tensors only (got a %s tensor); there is no CPU "
                "fallback -- the reference has none either (correlation.py:4)" % t.device.type)


def _f32c(t):
    """fp32 + contiguous (superset of the reference, which assumes both: SURVEY C-2)."""
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def _check_out(out, shape, device, who, dtype=torch.float32):
    """Caller-supplied outputs go to the C ABI as raw pointers: refuse anything the kernels would overrun or
    misinterpret (ADVICE r1: fp16 `input1.new()` outputs under the *_cuda shims, sliced views, wrong device)."""
    if out.dtype != dtype or not out.is_contiguous() or out.device != device or tuple(out.shape) != tuple(shape):
        raise RuntimeError("%s: out= must be a contiguous %s tensor of shape %s on %s (got %s %s on %s, contiguous=%s)"
                           % (who, dtype, tuple(shape), device, out.dtype, tuple(out.shape), out.device, out.is_contiguous()))
    return out


def _stream(t):
    return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None and t.numel() > 0 else ctypes.c_void_p(0)


def correlation_out_shape(C, H, W, pad_size, kernel_size, max_displacement, stride1, stride2):
    D, oH, oW = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    check(LIB.fn2b200_correlation_out_shape(C, H, W, pad_size, kernel_size, max_displacement, stride1,
                                            stride2, ctypes.byref(D), ctypes.byref(oH), ctypes.byref(oW)),
          "correlation_out_shape")
    return D.value, oH.value, oW.value


class CorrWorkspace(object):
    """Scratch of the tensor-core correlation path (bf16 hi/lo copies of input1/input2).  Returned by
    ``correlation_forward(..., return_workspace=True)`` and accepted by ``correlation_backward`` so the
    backward can skip the split pass when it runs on the SAME inputs (what autograd does)."""
    __slots__ = ("buf", "key")

    def __init__(self, buf, key):
        self.buf, self.key = buf, key


def _ws_key(a, b, prm):
    return (a.data_ptr(), b.data_ptr(), a._version, b._version, tuple(a.shape)) + tuple(prm)


def _corr_inputs(input1, input2, prm, *others):
    """(input1, input2) as contiguous fp32 and the correlation's (D, oH, oW); every tensor must be on CUDA."""
    _require_cuda(input1, input2, *others)
    if input1.dim() != 4 or input1.shape != input2.shape:
        raise ValueError("correlation: input1/input2 must be 4-D with equal shapes, got %s and %s"
                         % (tuple(input1.shape), tuple(input2.shape)))
    a, b = _f32c(input1), _f32c(input2)
    return a, b, correlation_out_shape(a.size(1), a.size(2), a.size(3), *prm)


def _corr_forward(a, b, cat, ch_offset, leaky_slope, prm, corr_multiply, who):
    """LeakyReLU(leaky_slope)(correlation) into cat[:, ch_offset : ch_offset + D] with one
    fn2b200_correlation_forward_cat call.  Returns the tensor-core workspace as a CorrWorkspace, or None."""
    B, C, H, W = a.shape
    with torch.cuda.device_of(a):
        ws_bytes = int(LIB.fn2b200_correlation_forward_workspace(B, C, H, W, *prm))
        # scratch for the tensor-core path's bf16 hi/lo operands (the analogue of the reference's
        # rbot1/rbot2, correlation.py:20-21); the caching allocator keeps it stream-ordered
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=a.device) if ws_bytes else None
        check(LIB.fn2b200_correlation_forward_cat(_ptr(a), _ptr(b), _ptr(cat), cat.size(1), int(ch_offset), float(leaky_slope),
                                                  B, C, H, W, *prm, int(corr_multiply), _ptr(ws), ws_bytes, _stream(a)), who)
    return CorrWorkspace(ws, _ws_key(a, b, prm)) if ws is not None else None


def _corr_backward(a, b, g, cat, ch_offset, leaky_slope, prm, corr_multiply, g1, g2, workspace, who):
    """g1, g2 (either may be None) from one fn2b200_correlation_backward_cat call, the correlation's gradient being
    g[:, ch_offset : ch_offset + D].  The forward's workspace is reused when its key still matches the inputs (same
    tensors, not modified in place since): the tensor-core backward then skips the split pass."""
    B, C, H, W = a.shape
    with torch.cuda.device_of(a):
        ws_bytes = int(LIB.fn2b200_correlation_backward_workspace(B, C, H, W, *prm))
        have = int(bool(ws_bytes) and workspace is not None and workspace.buf.numel() >= ws_bytes
                   and workspace.buf.device == a.device and workspace.key == _ws_key(a, b, prm))
        ws = workspace.buf if have else (torch.empty(ws_bytes, dtype=torch.uint8, device=a.device) if ws_bytes else None)
        check(LIB.fn2b200_correlation_backward_cat(_ptr(a), _ptr(b), _ptr(g), _ptr(cat), g.size(1), int(ch_offset),
                                                   float(leaky_slope), _ptr(g1), _ptr(g2), B, C, H, W, *prm,
                                                   int(corr_multiply), _ptr(ws), ws_bytes, have, _stream(a)), who)
    return g1, g2


def correlation_forward(input1, input2, pad_size, kernel_size, max_displacement, stride1, stride2,
                        corr_multiply=1, out=None, return_workspace=False):
    prm = (pad_size, kernel_size, max_displacement, stride1, stride2)
    a, b, (D, oH, oW) = _corr_inputs(input1, input2, prm)
    if oH <= 0 or oW <= 0:
        raise ValueError("correlation: empty output (%d x %d) for input %dx%d, pad_size=%d, max_displacement=%d, "
                         "kernel_size=%d" % (oH, oW, a.size(2), a.size(3), pad_size, max_displacement, kernel_size))
    shape = (a.size(0), D, oH, oW)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=a.device)
    else:
        _check_out(out, shape, a.device, "correlation_forward")
    ws = _corr_forward(a, b, out, 0, 1.0, prm, corr_multiply, "correlation_forward")
    return (out, ws) if return_workspace else out


def correlation_forward_cat(input1, input2, cat, ch_offset, leaky_slope, pad_size, kernel_size, max_displacement, stride1,
                            stride2, corr_multiply=1, return_workspace=False):
    """LeakyReLU(leaky_slope)(Correlation(...)(input1, input2)) written into cat[:, ch_offset : ch_offset + D] in place
    (FlowNetC.py:86-92: `torch.cat((out_conv_redir, corr_activation(corr)), 1)` without the activation pass and without
    the copy).  cat: contiguous fp32 [B, channels, oH, oW]; its other channels are left alone.  Returns cat, or
    (cat, CorrWorkspace or None) with return_workspace=True, for correlation_backward_cat."""
    prm = (pad_size, kernel_size, max_displacement, stride1, stride2)
    a, b, (D, oH, oW) = _corr_inputs(input1, input2, prm, cat)
    if cat.dim() != 4:
        raise ValueError("correlation_forward_cat: cat must be 4-D")
    _check_out(cat, (a.size(0), cat.size(1), oH, oW), a.device, "correlation_forward_cat")
    ws = _corr_forward(a, b, cat, ch_offset, leaky_slope, prm, corr_multiply, "correlation_forward_cat")
    return (cat, ws) if return_workspace else cat


def correlation_backward_cat(input1, input2, grad_cat, cat, ch_offset, leaky_slope, pad_size, kernel_size,
                             max_displacement, stride1, stride2, corr_multiply=1, need1=True, need2=True, workspace=None):
    """Backward of correlation_forward_cat: the input gradients of
    cat[:, ch_offset : ch_offset + D] = LeakyReLU(leaky_slope)(Correlation(...)(input1, input2)), read straight from
    grad_cat (the gradient of the whole concat) with LeakyReLU's derivative taken from `cat`, the buffer the forward
    wrote (may be None when leaky_slope == 1).  One kernel launch on the tensor-core path when `workspace` is what
    correlation_forward_cat(..., return_workspace=True) returned for the same inputs.  Returns (grad1, grad2)."""
    prm = (pad_size, kernel_size, max_displacement, stride1, stride2)
    a, b, (D, oH, oW) = _corr_inputs(input1, input2, prm, grad_cat, cat)
    g = _f32c(grad_cat)
    if g.dim() != 4 or (g.size(0), g.size(2), g.size(3)) != (a.size(0), oH, oW):
        raise ValueError("correlation_backward_cat: grad_cat shape %s does not match [%d, channels, %d, %d]"
                         % (tuple(g.shape), a.size(0), oH, oW))
    if cat is not None:
        _check_out(cat, g.shape, a.device, "correlation_backward_cat (cat)")
    g1 = torch.empty_like(a) if need1 else None
    g2 = torch.empty_like(b) if need2 else None
    return _corr_backward(a, b, g, cat, ch_offset, leaky_slope, prm, corr_multiply, g1, g2, workspace,
                          "correlation_backward_cat")


def correlation_backward(input1, input2, grad_output, pad_size, kernel_size, max_displacement, stride1,
                         stride2, corr_multiply=1, need1=True, need2=True, out1=None, out2=None, workspace=None):
    prm = (pad_size, kernel_size, max_displacement, stride1, stride2)
    a, b, (D, oH, oW) = _corr_inputs(input1, input2, prm, grad_output)
    g = _f32c(grad_output)
    if tuple(g.shape) != (a.size(0), D, oH, oW):
        raise ValueError("correlation_backward: grad_output shape %s != expected %s"
                         % (tuple(g.shape), (a.size(0), D, oH, oW)))
    for o_ in (out1, out2):
        if o_ is not None:
            _check_out(o_, a.shape, a.device, "correlation_backward")
    g1 = (out1 if out1 is not None else torch.empty_like(a)) if need1 else None
    g2 = (out2 if out2 is not None else torch.empty_like(b)) if need2 else None
    return _corr_backward(a, b, g, None, 0, 1.0, prm, corr_multiply, g1, g2, workspace, "correlation_backward")


def _img_strides(img):
    return _I64x4(*img.stride())


def resample2d_forward(input1, input2, kernel_size=1, bilinear=True, out=None):
    _require_cuda(input1, input2)
    if input1.dim() != 4 or input2.dim() != 4 or input2.size(1) != 2:
        raise ValueError("resample2d: expected image [B,C,H,W] and flow [B,2,H,W], got %s and %s"
                         % (tuple(input1.shape), tuple(input2.shape)))
    img = input1 if input1.dtype == torch.float32 else input1.float()   # strided views accepted as-is
    flow = _f32c(input2)
    _, C, iH, iW = img.shape
    B, _, H, W = flow.shape
    if img.size(0) < B:
        raise ValueError("resample2d: image batch %d smaller than flow batch %d" % (img.size(0), B))
    with torch.cuda.device_of(flow):
        if out is None:
            out = torch.empty((B, C, H, W), dtype=torch.float32, device=flow.device)
        else:
            _check_out(out, (B, C, H, W), flow.device, "resample2d_forward")
        check(LIB.fn2b200_resample2d_forward(_ptr(img), _img_strides(img), _ptr(flow), _ptr(out), B, C, iH, iW,
                                             H, W, int(kernel_size), int(bool(bilinear)), _stream(flow)),
              "resample2d_forward")
    return out


def resample2d_backward(input1, input2, grad_output, kernel_size=1, bilinear=True, need1=True, need2=True,
                        out1=None, out2=None, zero_out1=True):
    _require_cuda(input1, input2, grad_output)
    img = input1 if input1.dtype == torch.float32 else input1.float()
    flow, g = _f32c(input2), _f32c(grad_output)
    _, C, iH, iW = img.shape
    B, _, H, W = flow.shape
    if tuple(g.shape) != (B, C, H, W):
        raise ValueError("resample2d_backward: grad_output shape %s != expected %s" % (tuple(g.shape), (B, C, H, W)))
    with torch.cuda.device_of(flow):
        g1 = None
        if need1:
            if out1 is not None:
                _check_out(out1, img.shape, flow.device, "resample2d_backward")
            g1 = out1 if out1 is not None else torch.empty(tuple(img.shape), dtype=torch.float32, device=flow.device)
            if img.size(0) != B:      # rows the flow batch does not touch stay zero
                g1.zero_()
        if out2 is not None:
            _check_out(out2, flow.shape, flow.device, "resample2d_backward")
        g2 = (out2 if out2 is not None else torch.empty_like(flow)) if need2 else None
        strides = _img_strides(img)
        ws_bytes = int(LIB.fn2b200_resample2d_backward_workspace(strides, B, C, iH, iW, H, W)) if g1 is not None else 0
        # pixel-interleaved accumulator of the image gradient (the library zero-fills it on the stream)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=flow.device) if ws_bytes else None
        check(LIB.fn2b200_resample2d_backward_ws(_ptr(img), strides, _ptr(flow), _ptr(g), _ptr(g1), _ptr(g2),
                                                 B, C, iH, iW, H, W, int(kernel_size), int(bool(bilinear)),
                                                 int(bool(zero_out1)), _ptr(ws), ws_bytes, _stream(flow)),
              "resample2d_backward")
    return g1, g2


UPSAMPLE_MODES = {None: 0, "none": 0, 0: 0, "bilinear": 1, 1: 1, "nearest": 2, 2: 2}


def resample2d_forward_up(input1, flow_lr, upsample="bilinear", flow_mul=1.0, out=None):
    """Resample2d()(input1, nn.Upsample(scale_factor=4, mode=upsample)(flow_lr * flow_mul)) without materialising the
    full-resolution flow (models.py:130-133): the kernel interpolates the quarter-resolution flow per pixel."""
    _require_cuda(input1, flow_lr)
    if input1.dim() != 4 or flow_lr.dim() != 4 or flow_lr.size(1) != 2:
        raise ValueError("resample2d_forward_up: expected image [B,C,H,W] and flow [B,2,H/4,W/4], got %s and %s"
                         % (tuple(input1.shape), tuple(flow_lr.shape)))
    img = input1 if input1.dtype == torch.float32 else input1.float()
    flow = _f32c(flow_lr)
    mode = UPSAMPLE_MODES[upsample]
    B, _, fh, fw = flow.shape
    _, C, H, W = img.shape
    with torch.cuda.device_of(flow):
        if out is None:
            out = torch.empty((B, C, H, W), dtype=torch.float32, device=flow.device)
        else:
            _check_out(out, (B, C, H, W), flow.device, "resample2d_forward_up")
        check(LIB.fn2b200_resample2d_forward_up(_ptr(img), _img_strides(img), _ptr(flow), fh, fw, mode, float(flow_mul),
                                                _ptr(out), B, C, H, W, _stream(flow)), "resample2d_forward_up")
    return out


def warp_concat_forward(x, flow, C=3, upsample=None, flow_mul=1.0, flow_div=1.0, out=None, cat_channels=None, ch_x=0,
                        n_x=None, ch_warped=None, ch_flow=None, ch_flow_norm=-1, ch_diff_norm=None):
    """One kernel for the chain models.py:130-138 spells out with five modules and a torch.cat:

        flow_up = upsample(flow * flow_mul)            (upsample in {None, "bilinear", "nearest"}; None: flow is full-res)
        warped  = Resample2d()(x[:, C:2C], flow_up);   diff_norm = ChannelNorm()(x[:, :C] - warped)
        out[:, ch_x:ch_x+n_x] = x[:, :n_x];  out[:, ch_warped:+C] = warped;  out[:, ch_flow:+2] = flow_up / flow_div
        out[:, ch_flow_norm] = ChannelNorm()(flow_up);  out[:, ch_diff_norm] = diff_norm

    Defaults = models.py:138's 12-channel `concat1` (x | warped | flow / div_flow | diff norm).  A negative ch_* skips
    that product; channels nobody writes keep whatever `out` held.  x may be a strided view (unit stride along W)."""
    _require_cuda(x, flow)
    if x.dim() != 4 or flow.dim() != 4 or flow.size(1) != 2 or x.size(1) < 2 * C:
        raise ValueError("warp_concat_forward: expected x [B,>=2C,H,W] and flow [B,2,h,w], got %s and %s"
                         % (tuple(x.shape), tuple(flow.shape)))
    xx = x if x.dtype == torch.float32 else x.float()
    fl = _f32c(flow)
    mode = UPSAMPLE_MODES[upsample]
    B, _, fh, fw = fl.shape
    H, W = xx.shape[2], xx.shape[3]
    n_x = 2 * C if n_x is None else n_x
    ch_warped = 2 * C if ch_warped is None else ch_warped
    ch_flow = 3 * C if ch_flow is None else ch_flow
    ch_diff_norm = 3 * C + 2 if ch_diff_norm is None else ch_diff_norm
    with torch.cuda.device_of(fl):
        if out is None:
            cat_channels = 3 * C + 3 if cat_channels is None else cat_channels
            out = torch.empty((B, cat_channels, H, W), dtype=torch.float32, device=fl.device)
        else:
            cat_channels = out.size(1)
            _check_out(out, (B, cat_channels, H, W), fl.device, "warp_concat_forward")
        check(LIB.fn2b200_warp_concat_forward(_ptr(xx), _img_strides(xx), C, _ptr(fl), fh, fw, mode, float(flow_mul), _ptr(out),
                                              cat_channels, ch_x, n_x, ch_warped, ch_flow, float(flow_div), ch_flow_norm,
                                              ch_diff_norm, B, H, W, _stream(fl)), "warp_concat_forward")
    return out


def warp_concat_backward(x, flow, grad_cat, C=3, flow_div=1.0, ch_x=0, n_x=None, ch_warped=None, ch_flow=None,
                         ch_flow_norm=-1, ch_diff_norm=None):
    """Backward of warp_concat_forward(x, flow, upsample=None, ...): returns (grad_x [B,2C,H,W], grad_flow [B,2,H,W]).
    The layout arguments must be the forward's; C <= 3."""
    _require_cuda(x, flow, grad_cat)
    xx = x if x.dtype == torch.float32 else x.float()
    fl, gc = _f32c(flow), _f32c(grad_cat)
    B, _, H, W = fl.shape
    if tuple(xx.shape[2:]) != (H, W) or xx.size(1) < 2 * C or tuple(gc.shape[2:]) != (H, W) or gc.size(0) != B:
        raise ValueError("warp_concat_backward: shapes x %s, flow %s, grad_cat %s do not match" % (tuple(xx.shape), tuple(fl.shape), tuple(gc.shape)))
    n_x = 2 * C if n_x is None else n_x
    ch_warped = 2 * C if ch_warped is None else ch_warped
    ch_flow = 3 * C if ch_flow is None else ch_flow
    ch_diff_norm = 3 * C + 2 if ch_diff_norm is None else ch_diff_norm
    with torch.cuda.device_of(fl):
        gx = torch.empty((B, 2 * C, H, W), dtype=torch.float32, device=fl.device)
        gf = torch.empty_like(fl)
        ws_bytes = int(LIB.fn2b200_warp_concat_backward_workspace(B, C, H, W))
        ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=fl.device)
        check(LIB.fn2b200_warp_concat_backward(_ptr(xx), _img_strides(xx), C, _ptr(fl), _ptr(gc), gc.size(1), ch_x, n_x, ch_warped,
                                               ch_flow, float(flow_div), ch_flow_norm, ch_diff_norm, _ptr(gx), _ptr(gf), _ptr(ws),
                                               ws_bytes, B, H, W, _stream(fl)), "warp_concat_backward")
    return gx, gf


_DT16 = {torch.float16: 1, torch.bfloat16: 2}


def channelnorm_forward(input1, norm_deg=2, out=None):
    _require_cuda(input1)
    if input1.dim() != 4:
        raise ValueError("channelnorm: expected a 4-D tensor, got %s" % (tuple(input1.shape),))
    if input1.dtype in _DT16:        # native 16-bit kernels (the reference dispatches K8/K9 on half too)
        a = input1 if input1.is_contiguous() else input1.contiguous()
        B, C, H, W = a.shape
        with torch.cuda.device_of(a):
            if out is None:
                out = torch.empty((B, 1, H, W), dtype=a.dtype, device=a.device)
            else:
                _check_out(out, (B, 1, H, W), a.device, "channelnorm_forward", a.dtype)
            check(LIB.fn2b200_channelnorm_forward_16(_ptr(a), _ptr(out), B, C, H, W, int(norm_deg), _DT16[a.dtype],
                                                     _stream(a)), "channelnorm_forward")
        return out
    a = _f32c(input1)
    B, C, H, W = a.shape
    with torch.cuda.device_of(a):
        if out is None:
            out = torch.empty((B, 1, H, W), dtype=torch.float32, device=a.device)
        else:
            _check_out(out, (B, 1, H, W), a.device, "channelnorm_forward")
        check(LIB.fn2b200_channelnorm_forward(_ptr(a), _ptr(out), B, C, H, W, int(norm_deg), _stream(a)),
              "channelnorm_forward")
    return out


def channelnorm_backward(input1, output, grad_output, norm_deg=2, out=None):
    _require_cuda(input1, output, grad_output)
    if input1.dtype in _DT16 and output.dtype == input1.dtype and grad_output.dtype == input1.dtype:
        a, o, g = (t if t.is_contiguous() else t.contiguous() for t in (input1, output, grad_output))
        B, C, H, W = a.shape
        with torch.cuda.device_of(a):
            if out is None:
                out = torch.empty_like(a)
            else:
                _check_out(out, a.shape, a.device, "channelnorm_backward", a.dtype)
            check(LIB.fn2b200_channelnorm_backward_16(_ptr(a), _ptr(o), _ptr(g), _ptr(out), B, C, H, W, int(norm_deg),
                                                      _DT16[a.dtype], _stream(a)), "channelnorm_backward")
        return out
    a, o, g = _f32c(input1), _f32c(output), _f32c(grad_output)
    B, C, H, W = a.shape
    with torch.cuda.device_of(a):
        if out is None:
            out = torch.empty_like(a)
        else:
            _check_out(out, a.shape, a.device, "channelnorm_backward")
        check(LIB.fn2b200_channelnorm_backward(_ptr(a), _ptr(o), _ptr(g), _ptr(out), B, C, H, W, int(norm_deg),
                                               _stream(a)),
              "channelnorm_backward")
    return out


def launch_count():
    """Kernel launches issued by libfn2b200 in this PROCESS so far (one atomic counter, all threads)."""
    return int(LIB.fn2b200_launch_count())

"""Correlation (cost-volume) layer -- drop-in for networks/correlation_package/correlation.py.

Same class names, constructor arguments, ``Function.apply`` argument order and defaults as the
reference (correlation.py:8-60); the arithmetic runs in libfn2b200's sm_90a kernels.
"""
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable
from torch.nn.modules.module import Module

from . import functional as F2


class CorrelationFunction(Function):
    """reference: correlation.py:6-43 (note its Function-level defaults pad=3,k=3,md=20, :9)."""

    @staticmethod
    def forward(ctx, input1, input2, pad_size=3, kernel_size=3, max_displacement=20, stride1=1, stride2=2,
                corr_multiply=1):
        ctx.save_for_backward(input1, input2)
        ctx.pad_size = pad_size
        ctx.kernel_size = kernel_size
        ctx.max_displacement = max_displacement
        ctx.stride1 = stride1
        ctx.stride2 = stride2
        ctx.corr_multiply = corr_multiply
        # grad mode is always OFF inside Function.forward (autograd disables it), so is_grad_enabled() cannot be the
        # test; needs_input_grad says whether a backward can follow (under no_grad the ctx -- and the workspace with
        # it -- is dropped as soon as forward returns, so keeping it there costs nothing).
        keep = bool(ctx.needs_input_grad[0] or ctx.needs_input_grad[1])
        out, ws = F2.correlation_forward(input1, input2, pad_size, kernel_size, max_displacement, stride1, stride2,
                                         corr_multiply, return_workspace=True)
        # tensor-core path: keep the bf16 hi/lo copies of the inputs for backward (the reference keeps
        # nothing but recomputes its padded copies, correlation_cuda_kernel.cu:495-517); freed with ctx
        ctx.workspace = ws if keep else None
        return out if input1.dtype == torch.float32 else out.to(input1.dtype)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        input1, input2 = ctx.saved_tensors
        need1, need2 = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        g1, g2 = F2.correlation_backward(input1, input2, grad_output, ctx.pad_size, ctx.kernel_size,
                                         ctx.max_displacement, ctx.stride1, ctx.stride2, ctx.corr_multiply,
                                         need1=need1, need2=need2, workspace=getattr(ctx, "workspace", None))
        ctx.workspace = None
        if g1 is not None and g1.dtype != input1.dtype:
            g1 = g1.to(input1.dtype)
        if g2 is not None and g2.dtype != input2.dtype:
            g2 = g2.to(input2.dtype)
        return g1, g2, None, None, None, None, None, None


class Correlation(Module):
    """reference: correlation.py:46-60 -- Correlation(pad_size, kernel_size, max_displacement, stride1,
    stride2, corr_multiply); no parameters or buffers, so no state_dict keys."""

    def __init__(self, pad_size=0, kernel_size=0, max_displacement=0, stride1=1, stride2=2, corr_multiply=1):
        super(Correlation, self).__init__()
        self.pad_size = pad_size
        self.kernel_size = kernel_size
        self.max_displacement = max_displacement
        self.stride1 = stride1
        self.stride2 = stride2
        self.corr_multiply = corr_multiply

    def forward(self, input1, input2):
        return CorrelationFunction.apply(input1, input2, self.pad_size, self.kernel_size, self.max_displacement,
                                         self.stride1, self.stride2, self.corr_multiply)

    def extra_repr(self):
        return "pad_size=%d, kernel_size=%d, max_displacement=%d, stride1=%d, stride2=%d, corr_multiply=%d" % (
            self.pad_size, self.kernel_size, self.max_displacement, self.stride1, self.stride2, self.corr_multiply)

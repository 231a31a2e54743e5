"""Correlation (cost-volume) layer -- drop-in for networks/correlation_package/correlation.py.

Same class names, constructor arguments, ``Function.apply`` argument order and defaults as the
reference (correlation.py:8-60); the arithmetic runs in libfn2b200's sm_90a kernels.
"""
import torch
from torch.nn.modules.module import Module

from . import functional as F2
from .ops import fn2b200


def correlation(input1, input2, pad_size=3, kernel_size=3, max_displacement=20, stride1=1, stride2=2, corr_multiply=1):
    """torch.ops.fn2b200.correlation_forward (differentiable; the output in input1's dtype).  Its tensor-core workspace
    goes to the backward through autograd and is dropped here when no gradient is recorded."""
    F2._require_cuda(input1, input2)
    out = fn2b200.correlation_forward(input1, input2, pad_size, kernel_size, max_displacement, stride1, stride2,
                                      corr_multiply)[0]
    return out if input1.dtype == torch.float32 else out.to(input1.dtype)


class CorrelationFunction(object):
    """reference: correlation.py:6-43 (note its Function-level defaults pad=3,k=3,md=20, :9).  The reference's
    ``CorrelationFunction.apply(input1, input2, ...)`` call, forwarded to the operator (``correlation``)."""
    apply = forward = staticmethod(correlation)


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
        return correlation(input1, input2, self.pad_size, self.kernel_size, self.max_displacement, self.stride1,
                           self.stride2, self.corr_multiply)

    def extra_repr(self):
        return "pad_size=%d, kernel_size=%d, max_displacement=%d, stride1=%d, stride2=%d, corr_multiply=%d" % (
            self.pad_size, self.kernel_size, self.max_displacement, self.stride1, self.stride2, self.corr_multiply)

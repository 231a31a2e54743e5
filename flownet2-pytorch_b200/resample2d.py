"""Resample2d (flow warp) layer -- drop-in for networks/resample2d_package/resample2d.py.

Differences that are strict supersets of the reference (resample2d.py:7-49): the image may be a
non-contiguous view (no ``.contiguous()`` copy, :48), outputs are not zero-filled before being
overwritten (:18), and the image-gradient buffer is zeroed inside the C-ABI call on the same stream.
"""
import torch
from torch.nn.modules.module import Module

from . import functional as F2
from .ops import fn2b200


def resample2d(input1, input2, kernel_size=1, bilinear=True):
    """torch.ops.fn2b200.resample2d_forward (differentiable; the output in input1's dtype)."""
    F2._require_cuda(input1, input2)
    out = fn2b200.resample2d_forward(input1, input2, kernel_size, bilinear)
    return out if input1.dtype == torch.float32 else out.to(input1.dtype)


class Resample2dFunction(object):
    """reference: resample2d.py:7-38 -- ``Resample2dFunction.apply(input1, input2, kernel_size, bilinear)``, forwarded to
    the operator (``resample2d``)."""
    apply = forward = staticmethod(resample2d)


class Resample2d(Module):
    """reference: resample2d.py:40-49 -- Resample2d(kernel_size=1, bilinear=True)."""

    def __init__(self, kernel_size=1, bilinear=True):
        super(Resample2d, self).__init__()
        self.kernel_size = kernel_size
        self.bilinear = bilinear

    def forward(self, input1, input2):
        return resample2d(input1, input2, self.kernel_size, self.bilinear)

    def extra_repr(self):
        return "kernel_size=%d, bilinear=%s" % (self.kernel_size, self.bilinear)

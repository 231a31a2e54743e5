"""ChannelNorm layer -- drop-in for networks/channelnorm_package/channelnorm.py (:5-38).

``norm_deg`` is stored and passed through but, as in the reference kernels, always L2.
"""
import torch
from torch.nn.modules.module import Module

from . import functional as F2
from .ops import fn2b200


def channelnorm(input1, norm_deg=2):
    """torch.ops.fn2b200.channelnorm_forward (differentiable; fp16 / bf16 run natively, other dtypes through fp32 and
    back)."""
    F2._require_cuda(input1)
    out = fn2b200.channelnorm_forward(input1, norm_deg)
    return out if out.dtype == input1.dtype else out.to(input1.dtype)


class ChannelNormFunction(object):
    """reference: channelnorm.py:5-28 -- ``ChannelNormFunction.apply(input1, norm_deg)``, forwarded to the operator
    (``channelnorm``)."""
    apply = forward = staticmethod(channelnorm)


class ChannelNorm(Module):

    def __init__(self, norm_deg=2):
        super(ChannelNorm, self).__init__()
        self.norm_deg = norm_deg

    def forward(self, input1):
        return channelnorm(input1, self.norm_deg)

    def extra_repr(self):
        return "norm_deg=%d" % self.norm_deg

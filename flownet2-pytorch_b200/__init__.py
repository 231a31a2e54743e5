"""flownet2-pytorch_b200 -- H100-native (sm_90a) Correlation / Resample2d / ChannelNorm.

Import it as ``flownet2_b200`` (the directory name carries a hyphen; ``flownet2_b200.py`` at the
repo root aliases it).  Public surface = the reference's (networks/*_package/*.py):

    Correlation(pad_size, kernel_size, max_displacement, stride1, stride2, corr_multiply)
    Resample2d(kernel_size=1, bilinear=True)
    ChannelNorm(norm_deg=2)
    CorrelationFunction / Resample2dFunction / ChannelNormFunction  (torch.autograd.Function)

plus ``functional`` (tensor-level calls into the C ABI), ``compat`` (hooks for running the
unmodified reference models.py), ``fused`` (opt-in inference forwards of FlowNetC / FlowNet2C / FlowNet2 with the
upsample / warp / diff / norm / concat glue and the correlation's LeakyReLU + concat folded into our kernels),
``hostpipe.HostPipeline`` (host-resident data: H2D, kernels and D2H of consecutive steps overlapped) and ``numa``
(bind a rank's staging buffers to its GPU's NUMA node).  The CUDA library is mandatory: importing this package without
``libfn2b200.so`` raises, and CPU tensors are rejected -- there is no fallback path.
"""
from . import _lib, compat, functional, fused, hostpipe, numa, sharding  # noqa: F401
from .channelnorm import ChannelNorm, ChannelNormFunction  # noqa: F401
from .correlation import Correlation, CorrelationFunction  # noqa: F401
from .resample2d import Resample2d, Resample2dFunction  # noqa: F401

__version__ = "0.1.0"
__all__ = ["Correlation", "CorrelationFunction", "Resample2d", "Resample2dFunction", "ChannelNorm",
           "ChannelNormFunction", "functional", "compat", "fused", "hostpipe", "numa"]

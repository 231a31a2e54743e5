"""Shared helpers for the parity tests."""
import contextlib

import numpy as np


def rel_err(a, ref):
    """max|a-ref| / max|ref|  -- the 1e-4 contract of BASELINE.json's north_star (SURVEY 7, hard part 2)."""
    a = np.asarray(a, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    denom = np.abs(ref).max()
    return float(np.abs(a - ref).max() / (denom if denom > 0 else 1.0))


def assert_close(a, ref, tol=1e-4, what=""):
    a = np.asarray(a)
    ref = np.asarray(ref)
    assert a.shape == ref.shape, "%s: shape %s vs %s" % (what, a.shape, ref.shape)
    assert np.isfinite(a).all(), "%s: non-finite values" % what
    e = rel_err(a, ref)
    assert e <= tol, "%s: max|d|/max|ref| = %.3e > %.1e" % (what, e, tol)
    rms = float(np.sqrt(np.mean(np.asarray(ref, dtype=np.float64) ** 2)))
    assert np.allclose(a, ref, rtol=tol, atol=tol * max(rms, 1e-30)), "%s: allclose(rtol, atol=tol*rms) failed" % what


@contextlib.contextmanager
def cuda_profile(margin_s=0.05):
    """torch.profiler with CUDA activities, with a synchronised kernel of torch's and `margin_s` seconds of idle time
    after it starts and before it stops.  Late in a long test process the profiler has been seen to lose the record of
    the first kernel a case launched (a forward missing while its backward was recorded), and less often with the
    margins; callers still run a case whose record is incomplete once more before failing it.  The warm-up kernel's
    name is torch's, never one of the library's."""
    import time

    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()
        time.sleep(margin_s)
        yield prof
        torch.cuda.synchronize()
        time.sleep(margin_s)

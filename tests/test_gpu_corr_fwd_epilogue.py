"""The tensor-core correlation forward's cost volume, bit for bit, against digests of the stored results.

`corr_fwd_tc_kernel` stages each warp's band in shared memory and stores it one plane row at a time.  The values are
those of the kernel that stored straight from the accumulator fragment (same products, same accumulation, the same
x 1/C and LeakyReLU), so the bits must not move.  tests/golden/corr_fwd_epilogue_digests.npy holds the first 8
bytes (a little-endian uint64) of the SHA-256 of every (sample, displacement plane) of the forward and of
`forward_cat`'s 441 channels (473-channel concat, channel offset 32, LeakyReLU slope 0.1): one flat array, case by case
in the order of CASES, forward before forward_cat, [B, 441] each.  It is a .npy, not a .npz: tests/golden/*.npz are the
reference kernels' results.  Recorded from that kernel on an H100 with

    python tests/test_gpu_corr_fwd_epilogue.py --record

Inputs are seeded numpy normals copied to the device, so the digests do not depend on the device's random generator.
The cases cover C = 64, 128, 192 and 256, a partial x tile (W = 34: Wc % 16 != 0), a partial y tile (H = 22:
Hc % 8 != 0), a batch whose 192 tiles leave a partial last round on 132 SMs, and FlowNet2's [2,256,56,128].  A
mismatch names the first differing (sample, displacement plane) and, within it, the element farthest from an fp64
reference.
"""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "corr_fwd_epilogue_digests.npy")
MD, S2 = 20, 2
PRM = (MD, 1, MD, 1, S2)                  # pad, kernel_size, max_displacement, stride1, stride2
D = 441
CAT_CH, CH_OFF, SLOPE = 473, 32, 0.1
CASES = {
    "c64": (2, 64, 32, 64),
    "c128": (2, 128, 32, 64),
    "c192": (2, 192, 32, 64),
    "c256": (2, 256, 32, 64),
    "partial_x": (1, 128, 32, 34),
    "partial_y": (1, 192, 22, 64),
    "partial_round": (3, 256, 64, 128),
    "flownet2_448x1024": (2, 256, 56, 128),
}
OUTPUTS = ("forward", "forward_cat")


def _inputs(name):
    B, C, H, W = CASES[name]
    rng = np.random.default_rng(sorted(CASES).index(name) + 1)
    return [torch.from_numpy(rng.standard_normal((B, C, H, W), dtype=np.float32)).cuda() for _ in range(2)]


def _outputs(a, b):
    import flownet2_b200
    F2 = flownet2_b200.functional
    B, C, H, W = a.shape
    assert flownet2_b200._lib.LIB.fn2b200_correlation_path(C, H, W, *PRM) == 2, "not the tensor-core path"
    out = F2.correlation_forward(a, b, *PRM)
    cat = torch.zeros(B, CAT_CH, H, W, device=a.device)
    F2.correlation_forward_cat(a, b, cat, CH_OFF, SLOPE, *PRM)
    torch.cuda.synchronize()
    return {"forward": out, "forward_cat": cat[:, CH_OFF:CH_OFF + D]}


def _digests(t):
    """[B, 441] uint64: the first 8 bytes of the SHA-256 of each plane's fp32 bytes."""
    x = np.ascontiguousarray(t.cpu().numpy())
    return np.array([[np.frombuffer(hashlib.sha256(x[n, k].tobytes()).digest()[:8], "<u8")[0] for k in range(x.shape[1])]
                     for n in range(x.shape[0])], dtype="<u8")


def _golden():
    """{"case/output": [B, 441] digests} from the flat array."""
    flat, res, at = np.load(GOLDEN), {}, 0
    for name, (B, _, _, _) in CASES.items():
        for what in OUTPUTS:
            res["%s/%s" % (name, what)] = flat[at:at + B * D].reshape(B, D)
            at += B * D
    assert at == flat.size, "%s holds %d digests, CASES need %d" % (GOLDEN, flat.size, at)
    return res


@pytest.mark.parametrize("name", list(CASES))
def test_fwd_epilogue_bits(name):
    gold = _golden()
    a, b = _inputs(name)
    for what, t in _outputs(a, b).items():
        want, got = gold["%s/%s" % (name, what)], _digests(t)
        assert want.shape == got.shape
        if np.array_equal(want, got):
            continue
        n, k = (int(v) for v in np.argwhere(want != got)[0])
        import torch_ref
        ref = torch_ref.correlation64(a[n:n + 1].double(), b[n:n + 1].double(), MD, 1, MD, 1, S2)[0, k]
        if what == "forward_cat":
            ref = torch.where(ref > 0, ref, ref * SLOPE)
        d = (t[n, k].double() - ref).abs()
        y, x = np.unravel_index(int(d.argmax()), tuple(d.shape))
        pytest.fail("%s %s: %d of %d planes differ; the first is sample %d, displacement (tj, ti) = (%d, %d); there the "
                    "largest |value - fp64 ref| = %.3e is at (y, x) = (%d, %d): %.9e vs %.9e" % (
                        name, what, int((want != got).sum()), want.size, n, k // 21 - 10, k % 21 - 10, float(d.max()),
                        y, x, float(t[n, k, y, x]), float(ref[y, x])))


def record():
    parts = []
    for name in CASES:
        outs = _outputs(*_inputs(name))
        parts += [_digests(outs[what]).ravel() for what in OUTPUTS]
    np.save(GOLDEN, np.concatenate(parts).astype("<u8"))
    print("wrote %s (%d digests)" % (GOLDEN, sum(p.size for p in parts)))


if __name__ == "__main__":
    ROOT = os.path.dirname(HERE)
    for p in (ROOT, HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    if "--record" not in sys.argv:
        raise SystemExit("usage: python tests/test_gpu_corr_fwd_epilogue.py --record")
    record()

#!/usr/bin/env python3
"""Per-kernel times of the tensor-core correlation: split pass, forward and backward kernels.

    python tools/corr_tc_kernel_times.py --out DIR [--steps 20] [--warmup 5] [--tag NAME]

bench.py times the forward as one call (split pass + corr_fwd_tc_kernel); this script separates the three launches of a
training step.  At the correlation input FlowNet2 produces at 448x1024 ([8,256,56,128]) and at bench.py's cfg2
([8,256,112,256]), pad=20 k=1 md=20 s1=1 s2=2, it runs `steps` forward + backward calls of the functional API (the
forward's workspace handed to the backward, as the autograd Function does) under torch.profiler with CUDA activities and
reports, per kernel name, the launch count and the mean / min / max device time in ms.  The card's name and power limit
are read in the same run.  Writes DIR/corr_tc_kernel_times[_TAG].json and prints it.  Needs a CUDA device.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SHAPES = [(8, 256, 56, 128), (8, 256, 112, 256)]
PRM = (20, 1, 20, 1, 2)
KERNELS = ("corr_tc_split_kernel", "corr_fwd_tc_kernel", "corr_bwd_tc_kernel")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # the measurement itself does not depend on it
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown (%s)" % e}


def kernel_key(name):
    for k in KERNELS:
        if k in name:
            return k
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--tag", default="")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("corr_tc_kernel_times.py needs a CUDA device")
    import flownet2_b200
    F2 = flownet2_b200.functional
    dev = torch.device("cuda", 0)
    res = {"card": card(), "steps": args.steps, "library": os.path.abspath(flownet2_b200._lib.LIB._name), "shapes": {}}
    for shp in SHAPES:
        g = torch.Generator(device=dev).manual_seed(0)
        f1 = torch.randn(*shp, device=dev, generator=g)
        f2 = torch.randn(*shp, device=dev, generator=g)
        out = torch.empty(shp[0], 441, shp[2], shp[3], device=dev)
        gO = torch.randn(out.shape, device=dev, generator=g)
        g1, g2 = torch.empty_like(f1), torch.empty_like(f2)

        def step():
            _, ws = F2.correlation_forward(f1, f2, *PRM, 1, out=out, return_workspace=True)
            F2.correlation_backward(f1, f2, gO, *PRM, 1, out1=g1, out2=g2, workspace=ws)
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                step()
            torch.cuda.synchronize()
        times = {}
        for ev in prof.events():
            k = kernel_key(ev.name)
            if k is not None and ev.device_type == torch.autograd.DeviceType.CUDA:
                times.setdefault(k, []).append(ev.time_range.elapsed_us() / 1e3)
        res["shapes"]["x".join(map(str, shp))] = {
            k: {"launches": len(v), "mean_ms": round(sum(v) / len(v), 4), "min_ms": round(min(v), 4),
                "max_ms": round(max(v), 4)} for k, v in sorted(times.items())}
        del f1, f2, out, gO, g1, g2
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "corr_tc_kernel_times%s.json" % ("_" + args.tag if args.tag else ""))
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

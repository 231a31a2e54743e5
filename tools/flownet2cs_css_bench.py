#!/usr/bin/env python3
"""FlowNet2CS and FlowNet2CSS, module graph against the fused data flow, for inference and for a training step.

    python tools/flownet2cs_css_bench.py --out DIR [--steps 20] [--repeats 5] [--warmup 5]

The networks are the unmodified models.FlowNet2CS / FlowNet2CSS (installed under baseline/_ref by oracle/build_ref.py)
on our layers (compat.install("B2")), random xavier weights (seed 0), fp32, input U(0,255) [8,3,2,448,1024].
    module : net(x), the reference's own forward on the drop-in Correlation / Resample2d / ChannelNorm modules
    fused  : fused.fused_forward(net, x) for inference, fused.train_forward(net, x) for training
Inference runs in eval mode under no_grad; the rate is image pairs per second.  A training step runs in train mode:
the forward, then torch.autograd.grad of every parameter against a seeded weighting of the output flow.  The arms
alternate inside one process, repeat by repeat.  Reported per arm: the median over the repeats and its spread (time
per forward or per step, CUDA events over `steps` iterations), activation memory held between forward and backward
(allocated after the forward, above what was allocated before it) and the step's peak, libfn2b200 launches per
forward / per step; the output agreement between the arms (max|d| / max|ref|, deterministic cuDNN with TF32 off, one
seeded input); the card's name and power limit.  The timed runs use cuDNN's autotuner and TF32, as bench.py's FlowNet2 leg does.
Needs a CUDA device; there is no CPU fallback.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

B, H, W = 8, 448, 1024
NAMES = ("FlowNet2CS", "FlowNet2CSS")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # the measurement itself does not depend on it
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown (%s)" % e}


def _deterministic(on):
    import torch
    torch.backends.cudnn.deterministic = on
    torch.backends.cudnn.benchmark = not on
    torch.backends.cudnn.allow_tf32 = not on
    torch.backends.cuda.matmul.allow_tf32 = not on


def summary(xs):
    xs = sorted(xs)
    med = xs[len(xs) // 2]
    return {"median_ms": med, "min_ms": xs[0], "max_ms": xs[-1], "spread_pct": 100.0 * (xs[-1] - xs[0]) / med}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("flownet2cs_css_bench: no CUDA device (the measurement needs an H100; there is no CPU fallback)")
    from types import SimpleNamespace
    import flownet2_b200 as f
    from flownet2_b200 import compat, fused
    from oracle import ref as oref
    if not oref.python_tree_available():
        sys.exit("flownet2cs_css_bench: baseline/_ref/flownet2_pytorch missing (python oracle/build_ref.py)")
    compat.install("B2")
    models = oref.import_reference_models(fresh=True)
    dev = torch.device("cuda:0")
    x = (torch.rand(B, 3, 2, H, W, generator=torch.Generator().manual_seed(0)) * 255.0).to(dev)
    arms = ("module", "fused")
    results = {"card": card(), "steps": args.steps, "repeats": args.repeats, "input": [B, 3, 2, H, W], "models": []}

    def timed(fn):
        """Mean ms per call of fn over args.steps calls, CUDA events on the current stream."""
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for name in NAMES:
        torch.manual_seed(0)
        net = getattr(models, name)(SimpleNamespace(rgb_max=255.0, fp16=False)).to(dev)
        params = [p for p in net.parameters() if p.requires_grad]
        infer = {"module": lambda: net(x), "fused": lambda: fused.fused_forward(net, x)}
        train = {"module": lambda: net(x), "fused": lambda: fused.train_forward(net, x)}
        res = {"model": name}

        # agreement between the arms at fixed arithmetic, inference
        _deterministic(True)
        net.eval()
        with torch.no_grad():
            outs = {arm: infer[arm]().float() for arm in arms}
        res["output_agreement"] = float((outs["fused"] - outs["module"]).abs().max() / outs["module"].abs().max())
        del outs
        _deterministic(False)

        # inference: launches, then pairs/s
        info = {arm: {} for arm in arms}
        for arm in arms:
            with torch.no_grad():
                n0 = f.functional.launch_count()
                infer[arm]()
                info[arm]["launches_forward"] = f.functional.launch_count() - n0
                for _ in range(args.warmup):
                    infer[arm]()
        ms = {arm: [] for arm in arms}
        with torch.no_grad():
            for rep in range(args.repeats):
                for arm in (arms if rep % 2 == 0 else arms[::-1]):
                    ms[arm].append(timed(infer[arm]))
        for arm in arms:
            s = summary(ms[arm])
            info[arm].update(forward=s, pairs_per_s=B * 1000.0 / s["median_ms"])
        res["inference"] = info
        res["inference"]["fused_over_module_pairs_per_s"] = info["fused"]["pairs_per_s"] / info["module"]["pairs_per_s"]

        # training step: forward + autograd.grad of every parameter
        net.train()
        w = None

        def step(arm):
            out = train[arm]()
            return torch.autograd.grad((out * w).sum(), params)

        info = {arm: {} for arm in arms}
        for arm in arms:
            if w is None:
                w = torch.randn(train[arm]().shape, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
            step(arm)                    # cuDNN's autotuner allocates its workspaces on the first step of each shape
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            n0 = f.functional.launch_count()
            out = train[arm]()
            held = torch.cuda.memory_allocated() - base
            n1 = f.functional.launch_count()
            torch.autograd.grad((out * w).sum(), params)
            del out
            torch.cuda.synchronize()
            info[arm].update(held_fwd_to_bwd_MB=held / 1e6, peak_step_MB=(torch.cuda.max_memory_allocated() - base) / 1e6,
                             launches_fwd=n1 - n0, launches_bwd=f.functional.launch_count() - n1)
            for _ in range(args.warmup):
                step(arm)
        ms = {arm: [] for arm in arms}
        for rep in range(args.repeats):
            for arm in (arms if rep % 2 == 0 else arms[::-1]):
                ms[arm].append(timed(lambda: step(arm)))
        for arm in arms:
            info[arm]["step"] = summary(ms[arm])
        res["training"] = info
        res["training"]["fused_over_module_step"] = info["fused"]["step"]["median_ms"] / info["module"]["step"]["median_ms"]
        res["training"]["held_memory_saved_MB"] = info["module"]["held_fwd_to_bwd_MB"] - info["fused"]["held_fwd_to_bwd_MB"]
        results["models"].append(res)
        del net, params, w
        torch.cuda.empty_cache()
    compat.uninstall()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "flownet2cs_css_bench.json"), "w") as fh:
        json.dump(results, fh, indent=1)
    print(json.dumps(results))


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Training step of FlowNetC's correlation -> LeakyReLU(0.1) -> concat, unfused against fused.

    python tools/corr_cat_train_bench.py --out DIR [--steps 20] [--repeats 5] [--warmup 5]

One step = forward of `in_conv3_1 = cat(redir, LeakyReLU(0.1)(corr(f1, f2)))` (FlowNetC.py:86-92) with a seeded 32-channel
redir, then torch.autograd.grad of (redir, f1, f2) against a seeded upstream gradient.
    unfused : the drop-in Correlation module, F.leaky_relu(inplace=True), torch.cat
    fused   : fused.CorrelationCat (correlation_forward_cat + one correlation_backward_cat launch)
The two arms alternate inside one process, repeat by repeat, at the correlation input FlowNet2 produces at 448x1024
([8,256,56,128]) and at bench.py's cfg2 ([8,256,112,256]).  Reported per arm: the median step time over the repeats and
its spread, the backward-only time, memory held between forward and backward and the step's peak (above what was
allocated before the step), libfn2b200 launches per step; max|d| of the three gradients between the arms; the card's
name and power limit.  Needs a CUDA device; there is no CPU fallback.
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
NREDIR = 32


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # the measurement itself does not depend on it
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown (%s)" % e}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("corr_cat_train_bench: no CUDA device (the measurement needs an H100; there is no CPU fallback)")
    import flownet2_b200 as f
    F = torch.nn.functional
    dev = torch.device("cuda:0")
    corr = f.Correlation(*PRM, 1)
    fused = f.fused.CorrelationCat(*PRM, 1, 0.1)

    def forward(arm, redir, f1, f2):
        if arm == "fused":
            return fused(redir, f1, f2)
        return torch.cat((redir, F.leaky_relu(corr(f1, f2), 0.1, inplace=True)), 1)

    results = {"card": card(), "steps": args.steps, "repeats": args.repeats, "shapes": []}
    for shape in SHAPES:
        B, C, H, W = shape
        gen = torch.Generator(device=dev).manual_seed(0)
        f1 = torch.randn(*shape, device=dev, generator=gen).requires_grad_()
        f2 = torch.randn(*shape, device=dev, generator=gen).requires_grad_()
        redir = torch.randn(B, NREDIR, H, W, device=dev, generator=gen).requires_grad_()
        gcat = torch.randn(B, NREDIR + 441, H, W, device=dev, generator=gen)
        leaves = (redir, f1, f2)

        def step(arm, ev=None):
            out = forward(arm, *leaves)
            if ev is not None:
                ev.record()
            return torch.autograd.grad(out, leaves, gcat)

        arms = ("unfused", "fused")
        grads = {arm: step(arm) for arm in arms}
        max_diff = {name: float((grads["fused"][i] - grads["unfused"][i]).abs().max())
                    for i, name in enumerate(("redir", "f1", "f2"))}
        del grads
        info = {arm: {} for arm in arms}
        for arm in arms:
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            n0 = f.functional.launch_count()
            out = forward(arm, *leaves)
            held = torch.cuda.memory_allocated() - base
            n1 = f.functional.launch_count()
            torch.autograd.grad(out, leaves, gcat)
            del out
            torch.cuda.synchronize()
            info[arm].update(held_fwd_to_bwd_MB=held / 1e6, peak_step_MB=(torch.cuda.max_memory_allocated() - base) / 1e6,
                             launches_fwd=n1 - n0, launches_bwd=f.functional.launch_count() - n1)
            for _ in range(args.warmup):
                step(arm)
        step_ms = {arm: [] for arm in arms}
        bwd_ms = {arm: [] for arm in arms}
        for rep in range(args.repeats):
            for arm in (arms if rep % 2 == 0 else arms[::-1]):
                torch.cuda.synchronize()
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                mids = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps)]
                ends = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps)]
                t0.record()
                for i in range(args.steps):
                    step(arm, mids[i])
                    ends[i].record()
                t1.record()
                torch.cuda.synchronize()
                step_ms[arm].append(t0.elapsed_time(t1) / args.steps)
                bwd_ms[arm].append(sum(m.elapsed_time(e) for m, e in zip(mids, ends)) / args.steps)

        def summary(xs):
            xs = sorted(xs)
            med = xs[len(xs) // 2]
            return {"median_ms": med, "min_ms": xs[0], "max_ms": xs[-1], "spread_pct": 100.0 * (xs[-1] - xs[0]) / med}

        for arm in arms:
            info[arm].update(step=summary(step_ms[arm]), backward=summary(bwd_ms[arm]))
        cost_volume_MB = 4.0 * B * 441 * H * W / 1e6
        results["shapes"].append({
            "input": list(shape), "cost_volume_MB": cost_volume_MB, "max_abs_grad_diff": max_diff,
            "fused_over_unfused_step": info["fused"]["step"]["median_ms"] / info["unfused"]["step"]["median_ms"],
            "fused_over_unfused_backward": info["fused"]["backward"]["median_ms"] / info["unfused"]["backward"]["median_ms"],
            "held_memory_saved_MB": info["unfused"]["held_fwd_to_bwd_MB"] - info["fused"]["held_fwd_to_bwd_MB"],
            **info})
        del f1, f2, redir, gcat, leaves
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "corr_cat_train_bench.json"), "w") as fh:
        json.dump(results, fh, indent=1)
    print(json.dumps(results))


if __name__ == "__main__":
    main()

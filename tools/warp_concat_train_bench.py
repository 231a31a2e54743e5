#!/usr/bin/env python3
"""Training step of FlowNet2's warp groups, unfused against fused.

    python tools/warp_concat_train_bench.py --out DIR [--steps 20] [--repeats 5] [--warmup 5]

Workloads at FlowNet2's 448x1024, batch 8 (x [8,6,448,1024], quarter-resolution flows [8,2,112,256], div_flow 20):
    concat1 : cat(x, warped, up(flow2 * 20) / 20, |img0 - warped|), up = bilinear x4          (models.py:130-138)
    concat3 : the fusion stage's 11 channels from the FlowNetSD and FlowNetS2 flows, nearest x4 (models.py:153-179)
One step = the forward, then torch.autograd.grad of the leaves against a seeded upstream gradient.
    unfused : nn.Upsample -> the drop-in Resample2d -> subtraction -> ChannelNorm -> torch.cat under autograd
    fused   : fused.WarpConcat(upsample="bilinear") / fused.FusionConcat
Two cases per workload: x needs no gradient (FlowNet2 training: x is the normalised input) and x needs one.  The arms
alternate inside one process, repeat by repeat.  Reported per arm: the median step time over the repeats and its
spread, the same for the backward alone, memory held between forward and backward and the step's peak (above what was
allocated before the step), libfn2b200 launches; max|d| of the gradients between the arms; the backward's algorithmic
bytes (every tensor it must read or write, once: x, the concat-gradient channels it uses, the quarter-resolution flows
and the gradients it returns); the card's name and power limit.  Needs a CUDA device; there is no CPU fallback.
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
DIV = 20.0


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
        sys.exit("warp_concat_train_bench: no CUDA device (the measurement needs an H100; there is no CPU fallback)")
    import flownet2_b200 as f
    nn = torch.nn
    dev = torch.device("cuda:0")
    resample, cnorm = f.Resample2d(), f.ChannelNorm()
    up_bilinear = nn.Upsample(scale_factor=4, mode="bilinear")
    up_nearest = nn.Upsample(scale_factor=4, mode="nearest")
    warp_concat, fusion_concat = f.fused.WarpConcat(DIV, upsample="bilinear"), f.fused.FusionConcat(DIV)

    def concat1(arm, x, flow2):
        if arm == "fused":
            return warp_concat(x, flow2)
        up = up_bilinear(flow2 * DIV)
        warped = resample(x[:, 3:], up)
        return torch.cat((x, warped, up / DIV, cnorm(x[:, :3] - warped)), 1)

    def concat3(arm, x, sd_flow2, s2_flow2):
        if arm == "fused":
            return fusion_concat(x, sd_flow2, s2_flow2)
        s2 = up_nearest(s2_flow2 * DIV)
        d_s2 = cnorm(x[:, :3] - resample(x[:, 3:], s2))
        sd = up_nearest(sd_flow2 / DIV)
        d_sd = cnorm(x[:, :3] - resample(x[:, 3:], sd))
        return torch.cat((x[:, :3], sd, s2, cnorm(sd), cnorm(s2), d_sd, d_s2), 1)

    plane, qplane = 4 * B * H * W, 4 * B * (H // 4) * (W // 4)
    workloads = [
        # name, forward, number of flows, concat channels, concat-gradient planes read (without / with grad_x)
        ("concat1", concat1, 1, 12, (6, 12)),
        ("concat3", concat3, 2, 11, (8, 11)),
    ]
    results = {"card": card(), "steps": args.steps, "repeats": args.repeats, "shape": [B, 6, H, W], "workloads": []}
    for name, forward, nflows, nch, gplanes in workloads:
        for need_x in (False, True):
            gen = torch.Generator(device=dev).manual_seed(0)
            x = (torch.rand(B, 6, H, W, device=dev, generator=gen) - 0.5).requires_grad_(need_x)
            flows = [(torch.randn(B, 2, H // 4, W // 4, device=dev, generator=gen) * 0.3).requires_grad_()
                     for _ in range(nflows)]
            gcat = torch.randn(B, nch, H, W, device=dev, generator=gen)
            leaves = ([x] if need_x else []) + flows

            def step(arm, ev=None):
                out = forward(arm, x, *flows)
                if ev is not None:
                    ev.record()
                return torch.autograd.grad(out, leaves, gcat)

            arms = ("unfused", "fused")
            grads = {arm: step(arm) for arm in arms}
            names = (["x"] if need_x else []) + ["flow2_%d" % i for i in range(nflows)]
            max_diff = {n: float((grads["fused"][i] - grads["unfused"][i]).abs().max()) for i, n in enumerate(names)}
            max_ref = {n: float(grads["unfused"][i].abs().max()) for i, n in enumerate(names)}
            del grads
            info = {arm: {} for arm in arms}
            for arm in arms:
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                n0 = f.functional.launch_count()
                out = forward(arm, x, *flows)
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
            alg = plane * (6 + gplanes[need_x] + (6 if need_x else 0)) + qplane * 2 * 2 * nflows
            results["workloads"].append({
                "workload": name, "x_requires_grad": need_x, "max_abs_grad_diff": max_diff, "max_abs_grad_ref": max_ref,
                "algorithmic_bytes_backward": alg,
                "fused_backward_GBps": alg / (info["fused"]["backward"]["median_ms"] * 1e6),
                "fused_over_unfused_step": info["fused"]["step"]["median_ms"] / info["unfused"]["step"]["median_ms"],
                "fused_over_unfused_backward": info["fused"]["backward"]["median_ms"] / info["unfused"]["backward"]["median_ms"],
                "held_memory_saved_MB": info["unfused"]["held_fwd_to_bwd_MB"] - info["fused"]["held_fwd_to_bwd_MB"],
                **info})
            del x, flows, gcat, leaves
            torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "warp_concat_train_bench.json"), "w") as fh:
        json.dump(results, fh, indent=1)
    print(json.dumps(results))


if __name__ == "__main__":
    main()

"""Per-kernel time of the bench.py training step under torch.profiler (CUDA activities), in a run of its own.

    python scripts/profile_step.py --out DIR [--steps 10] [--warmup 5]

Prints, per step, the summed duration of the saving and non-saving mlp_fwd, mlp_bwd and mlp_wgrad kernels, and each
level's backward span (first mlp_bwd start to last mlp_wgrad end of the level) and its data-gradient idle time (how far
the last mlp_wgrad end falls behind the mlp_bwd end: the SMs that ran mlp_bwd wait that long for the weight gradient;
negative when the weight gradient finishes first).  bench.py's kernel_ms_per_step puts
events between mlp_bwd and mlp_wgrad, which serialises them; the trace here shows them running together.  Writes
summary.json (with the card name and power limit) and the Chrome trace under the output directory.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (workload constants)
from plenoctree_b200.nerf import train as T  # noqa: E402
from plenoctree_b200.nerf.models import NerfModel, Rays  # noqa: E402
from plenoctree_b200.nerf.utils import random_rays_np  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def kernel_class(name):
    if "mlp_fwd_kernel" in name:
        return "mlp_fwd (saving)" if ("Lb1E" in name or ", true>" in name) else "mlp_fwd (non-saving)"
    for k in ("mlp_bwd", "mlp_wgrad"):
        if k in name:
            return k
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", required=True, help="directory for summary.json and the Chrome trace")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profile_step.py needs a GPU"
    dev = torch.device("cuda", 0)
    model = NerfModel(sh_deg=bench.SH_DEG, num_coarse_samples=bench.NC, num_fine_samples=bench.NF, near=2.0, far=6.0,
                      white_bkgd=True, max_rays=bench.RAYS, sparsity_npoints=bench.NSP, device=dev)
    model.init_params(20200823)
    state = T.TrainState(model)
    n = args.steps + args.warmup
    o, d, vd, px = random_rays_np(n * bench.RAYS, 20200823)
    pool = torch.from_numpy(np.concatenate([o, d, vd, px], axis=1)).to(dev)

    def step(i):
        b = pool[i * bench.RAYS:(i + 1) * bench.RAYS]
        T.train_step(model, state, {"rays": Rays(b[:, 0:3], b[:, 3:6], b[:, 6:9]), "pixels": b[:, 9:12]}, 5e-4)

    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for i in range(args.warmup, n):
            step(i)
        torch.cuda.synchronize()
    os.makedirs(args.out, exist_ok=True)
    prof.export_chrome_trace(os.path.join(args.out, "trace.pt.trace.json"))

    kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                  key=lambda e: e.time_range.start)
    per = {}
    spans = []          # [mlp_bwd start, mlp_bwd end, last mlp_wgrad end] in launch order: two levels per step
    cur = None
    for e in kern:
        c = kernel_class(e.name)
        if c is None:
            continue
        per[c] = per.get(c, 0.0) + (e.time_range.end - e.time_range.start) / 1e3
        if c == "mlp_bwd":
            cur = [e.time_range.start, e.time_range.end, e.time_range.end]
            spans.append(cur)
        elif c == "mlp_wgrad" and cur is not None:
            cur[2] = max(cur[2], e.time_range.end)
    K = args.steps
    per_step = {k: v / K for k, v in sorted(per.items())}
    levels, idle = {}, {}
    for i, (s, b, t) in enumerate(spans):
        levels.setdefault(f"level {i % 2} backward span", []).append((t - s) / 1e3)
        idle.setdefault(f"level {i % 2} dgrad idle", []).append((t - b) / 1e3)

    def stats(d):
        return {k: {"min": min(v), "median": float(np.median(v)), "max": max(v)} for k, v in d.items()}

    res = {"card": card(), "steps": K, "kernel_ms_per_step": per_step,
           "backward_span_ms": stats(levels), "dgrad_idle_ms": stats(idle)}
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

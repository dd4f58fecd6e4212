"""Per-kernel time of the bench.py training step under torch.profiler (CUDA activities), in a run of its own.

    python scripts/profile_step.py --out DIR [--steps 10] [--warmup 5]

Prints, per step, the summed duration of the saving and non-saving mlp_fwd, mlp_bwd and mlp_wgrad kernels, and each
level's backward span (first mlp_bwd start to last mlp_wgrad end of the level) and its data-gradient idle time (how far
the last mlp_wgrad end falls behind the mlp_bwd end: the SMs that ran mlp_bwd wait that long for the weight gradient;
negative when the weight gradient finishes first).  bench.py's kernel_ms_per_step puts
events between mlp_bwd and mlp_wgrad, which serialises them; the trace here shows them running together.  Writes
summary.json (with the card name and power limit) and the Chrome trace under the output directory.

Beside the times it prints the HBM byte model of the step (hbm_bytes: the tile images each kernel class writes and
reads, from the workspace layout in layouts.py), the achieved GB/s of each kernel class and backward span, and the
least time each kernel could take from its HBM bytes (at --hbm-gbps, e.g. the copy rate scripts/hbm_probe.py measures
in the same session; default: the data-sheet 3350 GB/s) and from its algorithmic FLOPs (at --tflops, default the
data-sheet 989 dense fp16 TFLOP/s): the larger of the two names the bound the kernel is closer to.
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
from plenoctree_b200 import layouts as L  # noqa: E402
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


def hbm_bytes(cfg, n_rays, discard=True):
    """HBM bytes per training step by kernel class and per level's backward, from the workspace layout.
    Saving forward: writes h_0..h_7, the posenc tile and the ReLU masks.  Data gradient: reads the masks and writes
    dZ_0..dZ_7 and dO, unless the weight gradient discards them from L2 (train_step does: nerf/train.py), in which
    case they never reach HBM.  Weight gradient: reads h_0..h_7 and posenc (once: both row halves of a layer read
    the same h tile, the second from L2) and dZ / dO from L2 right after they were stored.  Weights, rays and the
    per-sample arrays (< 1 % of the bytes) are left out.  The write-back of a dirty line happens when L2 evicts it,
    so the data gradient's write bytes land somewhere in its level's backward span, not necessarily in its kernel."""
    K = L.K_of(int(cfg.sh_deg))
    do_bytes = (L.heads_width(K) + 63) // 64 * L.A_CHUNK_BYTES
    per, levels = {"mlp_fwd (saving)": 0, "mlp_bwd": 0, "mlp_wgrad": 0}, []
    for v in L.train_workspace_views(cfg, n_rays, True)["levels"]:
        t = v["tiles"]
        h_e = t * (L.NUM_TRUNK * L.A_TILE_BYTES + L.E_TILE_BYTES)
        mask = L.NUM_TRUNK * v["rows"] * 8 * 4
        dz_do = 0 if discard else t * (L.NUM_TRUNK * L.A_TILE_BYTES + do_bytes)
        per["mlp_fwd (saving)"] += h_e + mask
        per["mlp_bwd"] += mask + dz_do
        per["mlp_wgrad"] += h_e
        levels.append(mask + dz_do + h_e)
    return per, levels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", required=True, help="directory for summary.json and the Chrome trace")
    ap.add_argument("--hbm-gbps", type=float, default=3350.0, help="HBM bandwidth ceiling for the bound")
    ap.add_argument("--tflops", type=float, default=989.0, help="tensor-core ceiling for the bound")
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

    nbytes, span_bytes = hbm_bytes(model.cfg, bench.RAYS)
    flops = {"mlp_fwd (saving)": bench.F_FWD, "mlp_bwd": bench.F_DGRAD, "mlp_wgrad": bench.F_WGRAD}
    rows = sum(v["M"] for v in L.train_workspace_views(model.cfg, bench.RAYS, True)["levels"])
    hbm = {}
    for k, b in nbytes.items():
        ms = per_step.get(k)
        t_bytes, t_flops = b / (args.hbm_gbps * 1e6), rows * flops[k] / (args.tflops * 1e9)   # ms
        hbm[k] = {"bytes": b, "gbps": b / (ms * 1e6) if ms else None, "min_ms_bytes": t_bytes,
                  "min_ms_flops": t_flops, "closer_to": "HBM bytes" if t_bytes > t_flops else "tensor FLOPs"}
    for i, b in enumerate(span_bytes):
        med = float(np.median(levels[f"level {i} backward span"]))
        hbm[f"level {i} backward span"] = {"bytes": b, "gbps": b / (med * 1e6)}
    res = {"card": card(), "steps": K, "kernel_ms_per_step": per_step,
           "backward_span_ms": stats(levels), "dgrad_idle_ms": stats(idle),
           "hbm": hbm, "hbm_gbps_ceiling": args.hbm_gbps, "tflops_ceiling": args.tflops}
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

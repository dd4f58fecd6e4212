"""octree.optimization's per-image step with SGD momentum, 1 GPU: the c5_octree_opt workload of bench_extras.py
(256^3-equivalent SH16 tree, 800x800 images), one fused train pass (render + clamp-MSE gradient + scatter) and the
update, for momentum 0 (octree_sgd_kernel), 0.9 and 0.9 + Nesterov (octree_sgd_momentum_kernel).  The three run
alternately in one process, on three copies of the tree, over three rounds.

Per image: step time (CUDA events around train pass + update) and update time (events around the update alone).
Update bandwidth uses the byte model of DESIGN.md §6: plain 4 B per element (read g) + 12 B per element with g != 0
(read / write data, zero g); momentum 8 B per element (read g, b) + 12 B per element with g or b != 0 (read / write
data, write b) + 4 B per element with g != 0 (zero g).  The counts come from one untimed image per mode and round.
Prints one JSON line, with the card's name and power limit read in the same run.

  python scripts/bench_octree_momentum.py [--depth 7] [--images 12] [--rounds 3] [--hw 800]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

from bench_octree import build_tree  # noqa: E402
from plenoctree_b200.nerf.rays import pose_spherical  # noqa: E402
from plenoctree_b200.octree import VolumeRenderer  # noqa: E402

MODES = {"momentum_0": (0.0, False), "momentum_0.9": (0.9, False), "nesterov_0.9": (0.9, True)}


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:   # noqa: BLE001
        info["power_limit"] = f"unavailable ({e!r})"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=7)
    ap.add_argument("--images", type=int, default=12)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--hw", type=int, default=800)
    ap.add_argument("--lr", type=float, default=1e-3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    base, n_occ, _ = build_tree(args.depth, dev)
    H = W = args.hw
    focal = 0.5 * W / math.tan(0.5 * 0.6911112070083618)
    rs = np.random.RandomState(20200823)
    poses = [pose_spherical(rs.uniform(-180, 180), rs.uniform(-90, 0), 4.0) for _ in range(8)]
    with torch.no_grad():
        r0 = VolumeRenderer(base, step_size=1e-4)
        gts = [(r0.render_persp(p, W, H, focal) + 0.05 * torch.randn((H, W, 3), device=dev)).clamp_(0, 1) for p in poses]
    trees = {k: base.clone() for k in MODES}
    rend = {k: VolumeRenderer(t, step_size=1e-4) for k, t in trees.items()}
    n = base.n_internal * base.N ** 3 * base.data_dim
    sq = torch.zeros(1, dtype=torch.float64, device=dev)
    img = {k: 0 for k in MODES}

    def image(k, ev=None):
        mu, nest = MODES[k]
        rend[k].train_persp(poses[img[k] % 8], gts[img[k] % 8], W, H, focal, sq_err=sq)
        img[k] += 1
        if ev is not None:
            ev[0].record()
        trees[k].sgd_step(args.lr, mu, nest)
        if ev is not None:
            ev[1].record()

    for k in MODES:                                   # warm-up; the momentum buffers fill
        for _ in range(3):
            image(k)
    res = {k: {"ms_per_image": [], "ms_update": [], "bytes_update": []} for k in MODES}
    for _ in range(args.rounds):
        for k in MODES:
            mu, _ = MODES[k]
            # the bytes this mode's update moves, from one untimed image
            t = trees[k]
            rend[k].train_persp(poses[img[k] % 8], gts[img[k] % 8], W, H, focal, sq_err=sq)
            img[k] += 1
            g = t.grad_buffer().reshape(-1)[:n]
            nz_g = int((g != 0).sum())
            if mu == 0.0:
                nbytes = 4 * n + 12 * nz_g
            else:
                b = t._sgd_buf.reshape(-1)[:n]
                nbytes = 8 * n + 12 * int(((g != 0) | (b != 0)).sum()) + 4 * nz_g
            t.sgd_step(args.lr, *MODES[k])
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                   for _ in range(args.images)]
            a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            for i in range(args.images):
                image(k, evs[i])
            z.record()
            torch.cuda.synchronize()
            res[k]["ms_per_image"].append(a.elapsed_time(z) / args.images)
            res[k]["ms_update"].append(float(np.mean([e[0].elapsed_time(e[1]) for e in evs])))
            res[k]["bytes_update"].append(nbytes)
    out = {"metric": "octree.optimization per-image step with SGD momentum (c5_octree_opt: 256^3-equivalent SH16, "
                     f"{H}x{W})", "card": card(), "nodes": int(base.n_internal), "elements": int(n),
           "occupied_voxels": int(n_occ), "images_per_round": args.images, "rounds": args.rounds}
    for k, v in res.items():
        gbs = [b / 1e9 / (ms / 1e3) for b, ms in zip(v["bytes_update"], v["ms_update"])]
        out[k] = {"ms_per_image": [round(x, 4) for x in v["ms_per_image"]],
                  "ms_update": [round(x, 4) for x in v["ms_update"]],
                  "update_gb": [round(b / 1e9, 4) for b in v["bytes_update"]],
                  "update_gb_per_s": [round(x, 1) for x in gbs]}
    plain = np.mean(res["momentum_0"]["bytes_update"])
    for k in MODES:
        out[k]["bytes_ratio_to_plain"] = round(float(np.mean(res[k]["bytes_update"]) / plain), 3)
        out[k]["update_time_ratio_to_plain"] = round(float(np.mean(res[k]["ms_update"]) /
                                                           np.mean(res["momentum_0"]["ms_update"])), 3)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

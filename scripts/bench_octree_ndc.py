"""NDC (forward-facing) against world-space rays on the PlenOctree path, 1 GPU, one process, one tree: the 800x800-class
render_persp frame (fast and full quality), the fused training pass, and extraction's grid-weight render, each timed
with CUDA events in NDC mode and in world mode alternately over --rounds rounds.  The tree is scripts/bench_octree.py's
(depth 8, SH16, radius 1.3 about the origin, so it covers the NDC cube [-1, 1]^3 too).  World-mode cameras orbit the
tree (radius 4); NDC-mode cameras are forward-facing poses near the origin looking down -z.  NDC render_persp builds
its rays with pob_ndc_rays (36 B written and read back per ray and array) before the explicit-ray march; the
training pass and the grid weights transform each ray in the kernel.  World and NDC modes march different cameras, so
their gap is not the transform's cost; that cost is measured on the NDC cameras alone: pob_ndc_rays by itself
(ndc_rays_ms) and the explicit-ray march of the same rays computed beforehand (forward_precomputed_*_ms), which is
what NDC render_persp runs after pob_ndc_rays.  Prints one JSON line with the card's name and
power limit; --out PATH also writes it to a file.

  python scripts/bench_octree_ndc.py [--depth 8] [--hw 800] [--images 8] [--rounds 3] [--reso 512] [--out PATH]
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_octree import build_tree, timed  # noqa: E402
from plenoctree_b200.nerf.utils import pose_spherical  # noqa: E402
from plenoctree_b200.octree import NDCConfig, VolumeRenderer  # noqa: E402
from plenoctree_b200.octree.extraction import calculate_grid_weights  # noqa: E402


def forward_facing(n, seed=0):
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        ax, ay = rs.uniform(-0.1, 0.1, 2)
        cx, sx, cy, sy = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay)
        c2w = np.eye(4, dtype=np.float32)
        c2w[:3, :3] = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
        c2w[:3, 3] = rs.uniform(-0.2, 0.2, 3)
        out.append(c2w)
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:    # the numbers are still worth printing; say what is missing
        return torch.cuda.get_device_name(), f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=8)
    ap.add_argument("--hw", type=int, default=800)
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reso", type=int, default=512)
    ap.add_argument("--step", type=float, default=1e-3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    tree, _, _ = build_tree(args.depth, dev)
    hw, focal = args.hw, 1111.1111 * args.hw / 800
    ndc = NDCConfig(hw, hw, focal)
    poses = {"world": [pose_spherical(360.0 * i / args.images, -30.0, 4.0) for i in range(args.images)],
             "ndc": forward_facing(args.images)}
    rend = {"world": VolumeRenderer(tree, step_size=args.step), "ndc": VolumeRenderer(tree, step_size=args.step, ndc=ndc)}
    gt = torch.rand((hw, hw, 3), device=dev, generator=torch.Generator(device=dev).manual_seed(3))
    reso = args.reso
    sig = 40.0 * torch.rand(reso ** 3, device=dev, generator=torch.Generator(device=dev).manual_seed(4))
    sig = torch.where(torch.rand(reso ** 3, device=dev, generator=torch.Generator(device=dev).manual_seed(5)) < 0.02,
                      sig, torch.zeros_like(sig))

    class DS:
        pass

    def work(mode):
        r, ps = rend[mode], poses[mode]
        ds = DS()
        ds.camtoworlds, ds.w, ds.h, ds.focal = np.stack(ps), hw, hw, focal
        with torch.no_grad():
            return {
                "render_fast_ms": lambda i: r.render_persp(ps[i % len(ps)], hw, hw, focal, fast=True),
                "render_full_ms": lambda i: r.render_persp(ps[i % len(ps)], hw, hw, focal, fast=False),
                "train_pass_ms": lambda i: r.train_persp(ps[i % len(ps)], gt, hw, hw, focal),
                "grid_weights_ms": lambda i: calculate_grid_weights(ds, sig, reso, tree.invradius, tree.offset,
                                                                    step_size=args.step,
                                                                    ndc=ndc if mode == "ndc" else None),
            }

    from plenoctree_b200.octree import Rays
    from plenoctree_b200.octree.renderer import make_camera
    plain = VolumeRenderer(tree, step_size=args.step)
    cams = [make_camera(c, hw, hw, focal) for c in poses["ndc"]]
    with torch.no_grad():
        pre = [Rays(*rend["ndc"]._ndc_rays(None, c, 0, hw)) for c in cams]
    detour = {
        "ndc_rays_ms": lambda i: rend["ndc"]._ndc_rays(None, cams[i % len(cams)], 0, hw),
        "forward_precomputed_fast_ms": lambda i: plain.forward(pre[i % len(pre)], fast=True),
        "forward_precomputed_full_ms": lambda i: plain.forward(pre[i % len(pre)], fast=False),
    }
    res = {m: {} for m in ("world", "ndc", "ndc_detour")}
    for rnd in range(args.rounds):
        for mode in ("world", "ndc"):
            for k, fn in work(mode).items():
                n = 1 if k == "grid_weights_ms" else len(poses[mode])
                if rnd == 0:
                    timed(fn, n)      # warm-up of every shape
                with torch.no_grad():
                    res[mode].setdefault(k, []).append(round(timed(fn, n), 3))
                tree.grad = None
        for k, fn in detour.items():
            with torch.no_grad():
                if rnd == 0:
                    timed(fn, len(cams))
                res["ndc_detour"].setdefault(k, []).append(round(timed(fn, len(cams)), 3))
    name, power = card()
    out = {"bench": "octree_ndc", "gpu": name, "power_limit": power, "depth": args.depth, "hw": hw,
           "images": args.images, "reso": reso, "rounds": args.rounds, "leaves": int(tree.n_internal * 8), **res}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

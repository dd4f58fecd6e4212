"""Cost of depth and opacity in the octree render: 800x800 render_persp on the c5_octree_opt tree of bench_extras.py
(256^3-equivalent SH16, built by bench_octree.build_tree), with return_depth off (pob_octree_render) and on
(pob_octree_render_depth), for fast=False and fast=True, alternated over three rounds in one process.  CUDA events
around `--images` renders per mode and round.  Prints one JSON line, with the card's name and power limit read in the
same run.

  python scripts/bench_octree_depth.py [--depth 7] [--images 20] [--rounds 3] [--hw 800]
"""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

from bench_octree import build_tree  # noqa: E402
from bench_octree_momentum import card  # noqa: E402
from plenoctree_b200.nerf.rays import pose_spherical  # noqa: E402
from plenoctree_b200.octree import VolumeRenderer  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=7)
    ap.add_argument("--images", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--hw", type=int, default=800)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    tree, n_occ, _ = build_tree(args.depth, dev)
    H = W = args.hw
    focal = 0.5 * W / math.tan(0.5 * 0.6911112070083618)
    rs = np.random.RandomState(20200823)
    poses = [pose_spherical(rs.uniform(-180, 180), rs.uniform(-90, 0), 4.0) for _ in range(8)]
    r = VolumeRenderer(tree, step_size=1e-4)
    modes = {f"{'depth' if dep else 'rgb'}_{'fast' if fast else 'full'}": (dep, fast)
             for fast in (False, True) for dep in (False, True)}

    def render(k, i):
        dep, fast = modes[k]
        return r.render_persp(poses[i % 8], W, H, focal, fast=fast, return_depth=dep)

    res = {k: [] for k in modes}
    with torch.no_grad():
        for k in modes:                                 # warm-up; the colour of both entry points must agree
            for i in range(2):
                render(k, i)
        for fast in (False, True):
            a = render(f"rgb_{'fast' if fast else 'full'}", 0)
            b = render(f"depth_{'fast' if fast else 'full'}", 0)[0]
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        for _ in range(args.rounds):
            for k in modes:
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                s.record()
                for i in range(args.images):
                    render(k, i)
                e.record()
                torch.cuda.synchronize()
                res[k].append(s.elapsed_time(e) / args.images)
    out = {"metric": f"octree render_persp {H}x{W}, return_depth off / on (c5_octree_opt: 256^3-equivalent SH16)",
           "card": card(), "nodes": int(tree.n_internal), "occupied_voxels": int(n_occ),
           "images_per_round": args.images, "rounds": args.rounds}
    for k, v in res.items():
        out[k] = {"ms_per_image": [round(x, 4) for x in v]}
    for fast in ("full", "fast"):
        out[f"depth_over_rgb_{fast}"] = round(float(np.mean(res[f"depth_{fast}"]) / np.mean(res[f"rgb_{fast}"])), 4)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

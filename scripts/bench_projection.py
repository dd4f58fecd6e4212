"""Vanilla NeRF -> PlenOctree SH projection (octree.extraction step2 with use_viewdirs), 1 GPU.

On the depth-8 SH16 and SH25 trees of scripts/bench_octree.py (S = 8 samples per leaf, as --samples_per_cell's
default), times step2's projection of a vanilla model with random weights at D = 100 and D = 10,000 directions:
the point stage (trunk and a_p on the tensor cores), the direction tables and the projection kernel, with CUDA events
after a warm-up launch.  D = 100 covers every leaf; D = 10,000 covers the first --blocks leaf blocks, and the time of
the whole tree is extrapolated from the per-pair time (reported as such).  Prints one JSON line per (tree, D) with the
card's name and power limit read in the same run; --out PATH also writes them to a file.

  python scripts/bench_projection.py [--depth 8] [--blocks 64]
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

from bench_octree import build_tree  # noqa: E402
from plenoctree_b200.octree import projection as P  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return torch.cuda.get_device_name(), f"unknown ({e})"


def vanilla_layers(seed):
    rs = np.random.RandomState(seed)
    dims = [(63 if i == 0 else (319 if i == 5 else 256), 256) for i in range(8)]
    dims += [(256, 1), (256, 256), (256 + 27, 128), (128, 3)]
    return [(rs.uniform(-1, 1, (i, o)).astype(np.float32) * np.float32(np.sqrt(6.0 / (i + o))),
             rs.uniform(-0.05, 0.05, o).astype(np.float32)) for i, o in dims]


def time_projection(nerf, sh_deg, D, points, S):
    """(ms point stage, ms direction tables, ms projection) summed over the launches that cover `points`"""
    n_cells = points.shape[0]
    cpb = P.CELLS_PER_BLOCK
    n_blk = (n_cells + cpb - 1) // cpb
    per = P.blocks_per_launch(S, D, sh_deg) * cpb
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ms = np.zeros(3)
    for i in range(0, n_cells, per):
        pts = points[i:i + per].reshape(-1, 3).contiguous()
        nb = min(n_blk, (i + per + cpb - 1) // cpb) - i // cpb
        ev[0].record()
        a, sig = nerf.point_stage(pts)
        ev[1].record()
        tables = P.directions(nerf, sh_deg, D, i // cpb, nb)
        ev[2].record()
        P.project_cells(nerf, a, sig, S, sh_deg, tables, cpb)
        ev[3].record()
        torch.cuda.synchronize()
        ms += [ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3])]
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=8)
    ap.add_argument("--blocks", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_projection needs a GPU"
    dev = torch.device("cuda")
    name, power = card()
    S = 8
    nerf = P.VanillaNerf({"MLP_0": vanilla_layers(1)}, (0, 10, False), 4, num_fine_samples=0, device=dev)
    lines = []
    for sh_dim in (16, 25):
        sh_deg = int(round(sh_dim ** 0.5)) - 1
        tree = build_tree(args.depth, dev, sh_dim)[0]
        leaves = torch.where(tree.depths == tree.max_depth)[0]
        g = torch.Generator(device=dev).manual_seed(20200823)
        for D in (100, 10000):
            n = leaves.shape[0] if D == 100 else min(leaves.shape[0], args.blocks * P.CELLS_PER_BLOCK)
            u = torch.rand((n, S, 3), device=dev, generator=g)
            pts = tree[leaves[:n]].sample(S, uniforms=u)
            time_projection(nerf, sh_deg, D, pts[:P.CELLS_PER_BLOCK], S)            # warm-up
            ms = time_projection(nerf, sh_deg, D, pts, S)
            pairs = n * S * D
            rec = {"bench": "sh_projection", "gpu": name, "power_limit": power, "tree": f"depth {args.depth} SH{sh_dim}",
                   "leaves_in_tree": int(leaves.shape[0]), "leaves_timed": int(n), "samples_per_cell": S, "D": D,
                   "ms_point_stage": round(float(ms[0]), 3), "ms_direction_tables": round(float(ms[1]), 3),
                   "ms_projection": round(float(ms[2]), 3),
                   "ns_per_pair": round(float(ms.sum()) * 1e6 / pairs, 5),
                   "projection_ns_per_pair": round(float(ms[2]) * 1e6 / pairs, 5)}
            if n < leaves.shape[0]:
                rec["whole_tree_s_extrapolated"] = round(float(ms.sum()) / n * int(leaves.shape[0]) / 1e3, 2)
            print(json.dumps(rec), flush=True)
            lines.append(rec)
        del tree
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()

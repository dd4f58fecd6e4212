"""Octree-side measurements (BASELINE configs[4] and the extraction middle), 1 GPU:
  * VolumeRenderer.render_persp 800x800 on a synthetic depth-8 (512^3-equivalent) SH16 tree, fast and full quality;
  * one octree.optimization training image (fused render + MSE gradient + scatter) and the SGD update;
  * calculate_grid_weights on a 512^3 sigma grid.
Each line reports time (CUDA events, L2 flushed by the >126 MB working set), leaf visits per ray and the achieved
fraction of the HBM roofline for the algorithmic bytes stated in DESIGN.md.  Writes gpurun_out/bench_octree.json.

  python scripts/bench_octree.py [--depth 8] [--images 10] [--hw 800]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from plenoctree_b200.nerf.utils import pose_spherical  # noqa: E402
from plenoctree_b200.octree import N3Tree, VolumeRenderer  # noqa: E402
from plenoctree_b200.octree.extraction import calculate_grid_weights  # noqa: E402


def synthetic_mask(reso, dev):
    """a thick spherical shell plus a few solid blobs: ~2-3 % occupancy, like a converted synthetic scene."""
    ax = (torch.arange(reso, device=dev, dtype=torch.float32) + 0.5) / reso * 2 - 1
    x, y, z = torch.meshgrid(ax, ax, ax, indexing="ij")
    r = torch.sqrt(x * x + y * y + z * z)
    m = (r > 0.62) & (r < 0.66)
    g = torch.Generator().manual_seed(20200823)
    for _ in range(6):
        c = (torch.rand(3, generator=g) * 1.0 - 0.5).tolist()
        rad = 0.08 + 0.1 * float(torch.rand(1, generator=g))
        m |= ((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) < rad * rad
    return m


def build_tree(depth, dev, sh_dim=16):
    reso = 2 ** (depth + 1)
    mask = synthetic_mask(reso, dev)
    D = 3 * sh_dim + 1
    tree = N3Tree(N=2, data_dim=D, depth_limit=depth, init_reserve=500000, geom_resize_fact=1.0, radius=1.3,
                  center=[0, 0, 0], data_format=f"SH{sh_dim}", map_location=dev)
    idx = torch.nonzero(mask)
    arr = (torch.arange(reso, device=dev, dtype=torch.float32) + 0.5) / reso
    ax = [(arr - tree.offset[a]) / tree.invradius[a] for a in range(3)]
    grid = torch.stack([ax[0][idx[:, 0]], ax[1][idx[:, 1]], ax[2][idx[:, 2]]], dim=1).contiguous()
    t0 = time.time()
    for _ in range(depth - 1):
        tree[grid].refine()
    for j in range(0, grid.shape[0], 2000000):
        tree[grid[j:j + 2000000]].refine()
    torch.cuda.synchronize()
    build_s = time.time() - t0
    tree.shrink_to_fit()
    g = torch.Generator(device=dev).manual_seed(1)
    n = tree.n_internal
    tree.data[:n, ..., :-1] = 0.5 * torch.randn(tree.data[:n, ..., :-1].shape, device=dev, generator=g)
    deep = (tree.parent_depth[:n, 1] == depth)[:, None, None, None]
    sig = 40.0 * torch.rand(tree.data[:n, ..., -1].shape, device=dev, generator=g)
    tree.data[:n, ..., -1] = torch.where(deep, sig, torch.zeros_like(sig))
    return tree, int(mask.sum()), build_s


def timed(fn, n):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(n):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=8)
    ap.add_argument("--images", type=int, default=10)
    ap.add_argument("--hw", type=int, default=800)
    ap.add_argument("--step", type=float, default=1e-4)
    ap.add_argument("--grid-cams", type=int, default=8)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = float(peaks.get("hbm_gbs", 6501.9)) if isinstance(peaks, dict) else 6501.9
    out = {"config": {"depth": args.depth, "hw": args.hw, "step_size": args.step, "images": args.images},
           "hbm_peak_gbps": hbm}

    tree, n_occ, build_s = build_tree(args.depth, dev)
    n = tree.n_internal
    out["tree"] = {"nodes": n, "leaves": int(tree.n_leaves), "occupied_finest_voxels": n_occ, "build_s": build_s,
                   "data_gb": n * 8 * tree.data_dim * 4 / 1e9}
    H = W = args.hw
    focal = 0.5 * W / np.tan(0.5 * 0.6911112070083618)
    rs = np.random.RandomState(20200823)
    poses = [pose_spherical(rs.uniform(-180, 180), rs.uniform(-90, 0), 4.0) for _ in range(args.images)]
    r = VolumeRenderer(tree, step_size=args.step)
    K, D = 16, tree.data_dim

    for fast in (False, True):
        counters = torch.zeros(2, dtype=torch.int64, device=dev)
        with torch.no_grad():
            r.render_persp(poses[0], W, H, focal, fast=fast)
            ms = timed(lambda i: r.render_persp(poses[i % len(poses)], W, H, focal, fast=fast), args.images)
            for p in poses:
                r.render_persp(p, W, H, focal, fast=fast, counters=counters)
        visits, hits = [int(v) / len(poses) for v in counters.cpu().tolist()]
        # algorithmic bytes: per leaf visit the child entries along the descent are L1/L2-resident (shared by the 4
        # lanes and by neighbouring rays); the compulsory part is sigma (4 B) per visit + 3K coefficients per hit
        alg = visits * 4 + hits * 3 * K * 4
        out[f"render_persp_fast{int(fast)}"] = {
            "ms_per_image": ms, "fps": 1e3 / ms, "rays_per_s": H * W / ms * 1e3, "leaf_visits_per_ray": visits / (H * W),
            "contributing_per_ray": hits / (H * W), "algorithmic_gb_per_image": alg / 1e9,
            "achieved_gbps": alg / 1e9 / (ms / 1e3), "frac_of_hbm_peak": alg / 1e9 / (ms / 1e3) / hbm}
        print(json.dumps({f"render_persp_fast{int(fast)}": out[f"render_persp_fast{int(fast)}"]}), flush=True)

    # training image: fused render + gradient + scatter, then SGD
    with torch.no_grad():
        gts = [r.render_persp(p, W, H, focal).clamp_(0, 1) for p in poses[:4]]
    for g in gts:
        g.add_(0.05 * torch.randn_like(g)).clamp_(0, 1)
    sq = torch.zeros(1, dtype=torch.float64, device=dev)
    r.train_persp(poses[0], gts[0], W, H, focal, sq_err=sq)
    tree.sgd_step(0.0)
    ms_train = timed(lambda i: r.train_persp(poses[i % 4], gts[i % 4], W, H, focal, sq_err=sq), args.images)
    ms_sgd_sparse = timed(lambda i: tree.sgd_step(0.0), 3)   # gradient buffer already zero: read-only pass
    def step(i):
        r.train_persp(poses[i % 4], gts[i % 4], W, H, focal, sq_err=sq)
        tree.sgd_step(1e-3)
    ms_step = timed(step, args.images)
    hits_full = out["render_persp_fast0"]["contributing_per_ray"] * H * W
    visits_full = out["render_persp_fast0"]["leaf_visits_per_ray"] * H * W
    alg_train = 2 * (visits_full * 4 + hits_full * 3 * K * 4) + hits_full * D * 4 * 2  # two marches + RED scatter (rd+wr)
    out["train_image"] = {"ms_render_grad_scatter": ms_train, "ms_sgd_pass_zero_grad": ms_sgd_sparse,
                          "ms_per_image_with_sgd": ms_step, "images_per_s": 1e3 / ms_step,
                          "rays_per_s": H * W / ms_step * 1e3, "algorithmic_gb_per_image": alg_train / 1e9,
                          "achieved_gbps": alg_train / 1e9 / (ms_train / 1e3),
                          "frac_of_hbm_peak": alg_train / 1e9 / (ms_train / 1e3) / hbm,
                          "sgd_dense_gb": 2 * n * 8 * D * 4 / 1e9}
    print(json.dumps({"train_image": out["train_image"]}), flush=True)

    # extraction middle: grid weights on a 512^3 sigma grid
    reso = 2 ** (args.depth + 1)
    mask = synthetic_mask(reso, dev)
    sig = torch.where(mask, 40.0 * torch.rand(mask.shape, device=dev), torch.zeros((), device=dev)).reshape(-1)

    class DS:
        pass
    ds = DS()
    ds.w, ds.h, ds.focal = W, H, focal
    ds.camtoworlds = np.stack(poses[:args.grid_cams])
    calculate_grid_weights(ds, sig, reso, tree.invradius, tree.offset, step_size=args.step)
    ms_gw = timed(lambda i: calculate_grid_weights(ds, sig, reso, tree.invradius, tree.offset, step_size=args.step), 2)
    out["grid_weights"] = {"reso": reso, "cameras": args.grid_cams, "ms_total": ms_gw,
                           "ms_per_camera": ms_gw / args.grid_cams,
                           "rays_per_s": args.grid_cams * H * W / ms_gw * 1e3}
    print(json.dumps({"grid_weights": out["grid_weights"]}), flush=True)

    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "gpurun_out", "bench_octree.json"), "w"), indent=1)


if __name__ == "__main__":
    main()

"""Compressed PlenOctrees on the device, 1 GPU: the 800x800 frame time and the device bytes of the fp32 tree that
scripts/bench_octree.py builds (depth 8, SH16), and of its octree.compression output at --bits 16 and a small
--bits, rendered as stored (pob_octree_render_quant).  Times are CUDA events over --images poses, fast (early stop)
and full quality.  Prints one JSON line per tree; --out PATH also writes the whole result as JSON.

The median cut runs on the host (compression.median_cut, one basis function per worker process): at depth 8 it is
minutes of CPU per bit width, and the frame times do not depend on it beyond the palette indices it assigns.

  python scripts/bench_octree_compressed.py [--depth 8] [--images 10] [--hw 800] [--small-bits 4] [--out PATH]
"""
import argparse
import json
import os
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_octree import build_tree, timed  # noqa: E402
from plenoctree_b200.nerf.utils import pose_spherical  # noqa: E402
from plenoctree_b200.octree import VolumeRenderer, load_tree  # noqa: E402
from plenoctree_b200.octree.compression import compress_tree, median_cut  # noqa: E402


def _cut(args):
    pts, bits = args
    palette, index = median_cut(pts, bits)
    return palette.astype(np.float16), index.astype(np.uint16)


def compress(z, bits, sigma_thresh=2.0):
    """compression.compress_tree(z, bits, sigma_thresh) (unweighted, retain 0), its per-basis median cuts in parallel"""
    out = compress_tree({k: v for k, v in z.items() if k != "data"}, quantize=False)
    data = z["data"]
    N = data.shape[1]
    sigma = data[..., -1].astype(np.float32).reshape(-1).copy()
    keep = sigma > sigma_thresh
    sigma[~keep] = 0.0
    K = (data.shape[-1] - 1) // 3
    coeffs = data[..., :-1].reshape(-1, 3, K).astype(np.float32)[keep]
    with ProcessPoolExecutor(max_workers=min(K, os.cpu_count() or 1)) as ex:
        cuts = list(ex.map(_cut, [(np.ascontiguousarray(coeffs[:, :, i]), bits) for i in range(K)]))
    maps = []
    for _, index in cuts:
        full = np.zeros(keep.shape[0], dtype=np.uint16)
        full[keep] = index
        maps.append(full.reshape(-1, N, N, N))
    out["quant_colors"] = np.stack([p for p, _ in cuts])
    out["quant_map"] = np.stack(maps)
    out["sigma"] = sigma.reshape(-1, N, N, N)
    return out


def frame_ms(tree, poses, hw, focal, step):
    r = VolumeRenderer(tree, step_size=step)
    res = {}
    for fast in (False, True):
        with torch.no_grad():
            r.render_persp(poses[0], hw, hw, focal, fast=fast)
            res[f"ms_per_frame_fast{int(fast)}"] = timed(
                lambda i: r.render_persp(poses[i % len(poses)], hw, hw, focal, fast=fast), len(poses))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=8)
    ap.add_argument("--images", type=int, default=10)
    ap.add_argument("--hw", type=int, default=800)
    ap.add_argument("--step", type=float, default=1e-4)
    ap.add_argument("--small-bits", type=int, default=4)
    ap.add_argument("--out", type=str, default=None, help="also write the result as JSON to this path")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    tree, _, _ = build_tree(args.depth, dev)
    n = tree.n_internal
    H = W = args.hw
    focal = 0.5 * W / np.tan(0.5 * 0.6911112070083618)
    rs = np.random.RandomState(20200823)
    poses = [pose_spherical(rs.uniform(-180, 180), rs.uniform(-90, 0), 4.0) for _ in range(args.images)]
    out = {"config": vars(args), "gpu": torch.cuda.get_device_name(0), "nodes": n, "leaves": n * 8}
    # the tree as N3Tree.save writes it (fp16 data): the fp32 render is of exactly those values
    z = tree.state()
    tree.data[:n] = torch.from_numpy(z["data"].astype(np.float32)).to(dev)
    out["fp32"] = {"device_bytes": tree.data[:n].nbytes + tree.child[:n].nbytes,
                   **frame_ms(tree, poses, W, focal, args.step)}
    print(json.dumps({"fp32": out["fp32"]}), flush=True)
    for bits in (16, args.small_bits):
        q = load_tree(compress(z, bits))
        out[f"bits{bits}"] = {"device_bytes": q.device_bytes(), **frame_ms(q, poses, W, focal, args.step)}
        print(json.dumps({f"bits{bits}": out[f"bits{bits}"]}), flush=True)
        del q
    if args.out:
        json.dump(out, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()

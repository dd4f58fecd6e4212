"""Time octree compression (median-cut palettes) on the host (numpy) against the device (csrc/quantize.cu).

  python scripts/bench_compression.py [--depth 8] [--host_basis 1] [--bits 16]

On the scripts/bench_octree.py tree at SH16 and SH25, unweighted and --weighted, prints one JSON line with:
  host_s_per_basis   numpy median_cut of `--host_basis` basis functions, wall-clock seconds each
  device_ms_tree     pob_quantize_median_cut of every basis function of the tree in one call (CUDA events)
  device_ms_basis    device_ms_tree / basis functions
  compress_tree_s    compress_tree(..., device="cuda") end to end (host copies and fp16 casts included, no deflate)
and whether the device map and palette equal the host's for the basis functions timed on the host.  The card's name
and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_octree import build_tree  # noqa: E402
from plenoctree_b200.octree import compression as C  # noqa: E402
from plenoctree_b200.octree import quantize as Q  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (r.stdout.strip().splitlines() or ["unknown, unknown"])[0].split(", ")
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=8)
    ap.add_argument("--bits", type=int, default=16)
    ap.add_argument("--host_basis", type=int, default=1, help="basis functions timed on the host per case")
    args = ap.parse_args()
    name, power = card()
    res = {"card": name, "power_limit": power, "depth": args.depth, "bits": args.bits, "cases": []}
    for sh_dim in (16, 25):
        tree, _, _ = build_tree(args.depth, torch.device("cuda"), sh_dim=sh_dim)
        z = tree.state()
        del tree
        data = z["data"]
        sigma = data[..., -1].astype(np.float32).reshape(-1)
        keep = sigma > np.float32(2.0)
        coeffs = data[..., :-1].reshape(-1, 3, sh_dim).astype(np.float32)[keep]
        pts = torch.from_numpy(np.ascontiguousarray(coeffs.transpose(2, 0, 1))).cuda()
        for weighted in (False, True):
            w = 1.0 - np.exp(-0.01 * sigma[keep].astype(np.float64)) if weighted else None
            Q.median_cut_batch(pts[:1, :1000], args.bits, None if w is None else w[:1000])   # warm-up
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            times = []
            for _ in range(3):
                torch.cuda.synchronize()
                e0.record()
                pal, idx = Q.median_cut_batch(pts, args.bits, w)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
            host_s, equal = [], True
            for i in range(args.host_basis):
                t0 = time.perf_counter()
                hp, hi = C.median_cut(coeffs[:, :, i], args.bits, w)
                host_s.append(time.perf_counter() - t0)
                equal &= bool(np.array_equal(hi.astype(np.uint16), idx[i].cpu().numpy().view(np.uint16)))
                equal &= hp.tobytes() == pal[i].cpu().numpy().tobytes()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            C.compress_tree(dict(z), args.bits, 2.0, 0, weighted, device="cuda")
            torch.cuda.synchronize()
            ct = time.perf_counter() - t0
            res["cases"].append({"sh": sh_dim, "weighted": weighted, "kept_voxels": int(keep.sum()),
                                 "host_s_per_basis": [round(x, 3) for x in host_s],
                                 "device_ms_tree": [round(x, 2) for x in times],
                                 "device_ms_basis": round(min(times) / sh_dim, 2),
                                 "host_over_device_per_basis": round(min(host_s) * 1e3 / (min(times) / sh_dim), 1),
                                 "compress_tree_s": round(ct, 3), "equal_to_host": equal})
            print(json.dumps(res["cases"][-1]), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

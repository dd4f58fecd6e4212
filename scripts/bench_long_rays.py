"""Cost of long rays (`--num_coarse_samples` + `--num_fine_samples` up to 1024): for (64, 128), (128, 256),
(128, 384) and (256, 768), the eager fp16 training step (SH degree 3, 10 000 sparsity points) at batch 1024 and at
4096 where its workspace fits, MLP-samples/s (rays x (2 Nc + Nf) + 10 000 per step, which makes the configs
comparable), one 800x800 render_image, and CUDA-event times of the per-ray kernels at 4096 rays with the bytes each
must move (BYTES below) over that time.  Prints the card name and power limit beside the numbers.

    python scripts/bench_long_rays.py [--steps 10] [--reps 20]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from plenoctree_b200._lib import RenderConfig, check, lib, ptr  # noqa: E402
from plenoctree_b200.nerf import train as T  # noqa: E402
from plenoctree_b200.nerf.models import NerfModel, Rays, ctypes_ref  # noqa: E402
from plenoctree_b200.nerf.rays import random_rays_np  # noqa: E402
from plenoctree_b200.nerf.utils import generate_rays, pose_spherical, render_image  # noqa: E402
from scripts.bench_model_flags import card, timed  # noqa: E402

CONFIGS = ((64, 128), (128, 256), (128, 384), (256, 768))
BATCHES = (1024, 4096)
NSP = 10000
KERNEL_RAYS = 4096

# bytes each per-ray kernel must read and write per sample (fp32): compositing reads (rgb, sigma) and z and writes
# the weight; its backward reads (rgb, sigma) and z and writes G (4 floats); resampling reads the coarse z and weight
# per coarse sample, one u per new sample, and writes every union sample
BYTES = {"composite_fwd": lambda nc, nf: 24 * (nc + nf),
         "composite_bwd": lambda nc, nf: 36 * (nc + nf),
         "sample_pdf": lambda nc, nf: 8 * nc + 4 * nf + 4 * (nc + nf)}


def train_step_ms(nc, nf, R, steps, warmup):
    c = RenderConfig(3, nc, nf, 1, R, NSP)
    need = int(lib.pob_train_workspace_bytes(ctypes_ref(c), 1))
    free, _ = torch.cuda.mem_get_info()
    if need + (4 << 30) > free:
        return None, need
    model = NerfModel(sh_deg=3, num_coarse_samples=nc, num_fine_samples=nf, max_rays=R, sparsity_npoints=NSP)
    model.init_params()
    state = T.TrainState(model)
    o, d, v, px = random_rays_np(R, 0)
    batch = {"rays": Rays(*(torch.from_numpy(a).cuda() for a in (o, d, v))), "pixels": torch.from_numpy(px).cuda()}
    for _ in range(warmup):
        T.train_step(model, state, batch, 1e-4)
    ms = timed(lambda: T.train_step(model, state, batch, 1e-4), steps)
    del model, state, batch
    torch.cuda.empty_cache()
    return ms, need


def render_ms(nc, nf):
    model = NerfModel(sh_deg=3, num_coarse_samples=nc, num_fine_samples=nf, max_rays=8192)
    model.init_params()
    W = 800
    rays = generate_rays(W, W, 0.5 * W / np.tan(0.5 * 0.6911112070083618), pose_spherical(30.0, -30.0, 4.0)[None])
    frame = Rays(rays.origins[0], rays.directions[0], rays.viewdirs[0])
    render_image(model, frame)
    ms = timed(lambda: render_image(model, frame), 1)
    del model
    torch.cuda.empty_cache()
    return ms


def kernel_ms(nc, nf, reps):
    """the three per-ray kernels standalone at KERNEL_RAYS rays of a partially opaque field (nf = 0: compositing
    only, at N = nc)"""
    R, N = KERNEL_RAYS, nc + nf
    rs = np.random.RandomState(0)
    rgbs = torch.from_numpy(np.concatenate([rs.uniform(0, 1, (R, N, 3)), rs.uniform(0, 2, (R, N, 1))], -1)
                            .astype(np.float32)).cuda()
    z = torch.from_numpy(np.sort(rs.uniform(2, 6, (R, N)), 1).astype(np.float32)).cuda()
    zc = z[:, :nc].contiguous()
    d = torch.from_numpy(rs.normal(size=(R, 3)).astype(np.float32)).cuda()
    px = torch.rand((R, 3), device="cuda")
    comp, disp, acc = torch.empty((R, 3), device="cuda"), torch.empty(R, device="cuda"), torch.empty(R, device="cuda")
    w = torch.empty((R, N), device="cuda")
    G = torch.empty((R, N, 4), device="cuda")
    sq = torch.zeros(1, device="cuda")
    u = torch.rand((R, max(nf, 1)), device="cuda")
    wc = torch.rand((R, nc), device="cuda")
    zo = torch.empty((R, N), device="cuda")
    calls = {
        "composite_fwd": lambda: check(lib.pob_composite(ptr(rgbs), ptr(z), ptr(d), R, N, 1, ptr(comp), ptr(disp),
                                                         ptr(acc), ptr(w), None)),
        "composite_bwd": lambda: check(lib.pob_composite_bwd(ptr(rgbs), ptr(z), ptr(d), ptr(comp), ptr(px), R, N, 1,
                                                             0.37, ptr(G), ptr(sq), None)),
        "sample_pdf": lambda: check(lib.pob_sample_pdf(ptr(zc), ptr(wc), ptr(u), 1, R, nc, nf, ptr(zo), None)),
    }
    if nf == 0:
        del calls["sample_pdf"]
    out = {}
    for k, fn in calls.items():
        fn()
        ms = timed(fn, reps)
        out[k] = dict(ms=ms, gbps=BYTES[k](nc, nf) * R / (ms * 1e-3) / 1e9)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    rows = []
    for nc, nf in CONFIGS:
        row = dict(nc=nc, nf=nf, step={})
        for R in BATCHES:
            ms, need = train_step_ms(nc, nf, R, a.steps, a.warmup)
            mlp_samples = R * (2 * nc + nf) + NSP
            row["step"][R] = dict(workspace_gb=need / 1e9, ms=ms, rays_per_s=None if ms is None else R / ms * 1e3,
                                  mlp_samples_per_s=None if ms is None else mlp_samples / ms * 1e3)
        row["render_800_ms"] = render_ms(nc, nf)
        k = kernel_ms(nc, nf, a.reps)
        kc = kernel_ms(nc, 0, a.reps)
        row["kernels_4096"] = k
        row["kernels_4096_coarse"] = kc
        # one training step at 4096 rays runs compositing forward and backward at Nc and at Nc + Nf, and resampling
        # once: their share of the step at batch 4096
        per_ray = sum(x["composite_fwd"]["ms"] + x["composite_bwd"]["ms"] for x in (k, kc)) + k["sample_pdf"]["ms"]
        st = row["step"][4096]["ms"]
        row["per_ray_share_of_4096_step"] = None if st is None else per_ray / st
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(dict(card=card(), workload="SH16 eager fp16 train_step + 10 000 sparsity points; render_image "
                                                 "800x800 fp16; per-ray kernels standalone at 4096 rays",
                          rows=rows)), flush=True)


if __name__ == "__main__":
    main()

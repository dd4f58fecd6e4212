"""Cost of the model flags against the default model: bench.py's training workload (SH degree 3, i.e. 16 SH
coefficients; 4096 rays x (64 + 128) samples, 10 000 sparsity points, eager fp16 train_step) and one 800x800 render
(render_image, fp16) for each variant of one group, alternated in one process over several rounds.  The first variant
of every group is the baseline: the default encoder (0, 10), a relu trunk and relu density.  Prints the card name and
power limit beside the numbers.

    python scripts/bench_model_flags.py posenc | net_activation | sigma_activation [--steps 20] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from plenoctree_b200.nerf import train as T  # noqa: E402
from plenoctree_b200.nerf.models import NerfModel, Rays  # noqa: E402
from plenoctree_b200.nerf.rays import random_rays_np  # noqa: E402
from plenoctree_b200.nerf.utils import generate_rays, pose_spherical, render_image  # noqa: E402

R, NC, NF, NSP = 4096, 64, 128, 10000
BASE = dict(sh_deg=3, num_coarse_samples=NC, num_fine_samples=NF, near=2.0, far=6.0, white_bkgd=True, lindisp=False,
            min_deg_point=0, max_deg_point=10, legacy_posenc_order=False, net_activation="relu",
            sigma_activation="relu")
# group -> variant -> the flags it sets beside BASE; the first variant is the baseline
GROUPS = {
    "posenc": {"0_10": {}, "0_8": dict(max_deg_point=8), "0_10_legacy": dict(legacy_posenc_order=True)},
    "net_activation": {"relu": {}, "elu": dict(net_activation="elu"), "softplus": dict(net_activation="softplus"),
                       "tanh": dict(net_activation="tanh")},
    "sigma_activation": {"relu": {}, "softplus": dict(sigma_activation="softplus")},
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def setup(flags):
    model = NerfModel.from_flags(types.SimpleNamespace(**{**BASE, **flags}), max_rays=R, sparsity_npoints=NSP)
    model.init_params()
    state = T.TrainState(model)
    o, d, v, px = random_rays_np(R, 0)
    batch = {"rays": Rays(*(torch.from_numpy(a).cuda() for a in (o, d, v))), "pixels": torch.from_numpy(px).cuda()}
    return model, state, batch


def timed(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("group", choices=sorted(GROUPS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    variants = GROUPS[a.group]
    runs = {k: setup(flags) for k, flags in variants.items()}
    W = 800
    rays = generate_rays(W, W, 0.5 * W / np.tan(0.5 * 0.6911112070083618), pose_spherical(30.0, -30.0, 4.0)[None])
    frame = Rays(rays.origins[0], rays.directions[0], rays.viewdirs[0])
    for model, state, batch in runs.values():
        for _ in range(a.warmup):
            T.train_step(model, state, batch, 1e-4)
        render_image(model, frame)
    torch.cuda.synchronize()
    step = {k: [] for k in variants}
    render = {k: [] for k in variants}
    for _ in range(a.rounds):
        for k, (model, state, batch) in runs.items():
            step[k].append(timed(lambda: T.train_step(model, state, batch, 1e-4), a.steps))
            render[k].append(timed(lambda: render_image(model, frame), 1))
    base = next(iter(variants))
    out = dict(card=card(), workload=f"SH16 {R} rays x ({NC}+{NF}) + {NSP} sparsity points, eager fp16 train_step; "
                                     f"{W}x{W} render_image fp16",
               step_ms=step, render_800_ms=render,
               step_ratio_median={k: float(np.median(step[k]) / np.median(step[base])) for k in variants},
               render_ratio_median={k: float(np.median(render[k]) / np.median(render[base])) for k in variants})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

"""Cost of the trunk activations (`--net_activation elu | softplus | tanh`) against relu: bench.py's training workload
(SH degree 3, i.e. 16 SH coefficients; 4096 rays x (64 + 128) samples, 10 000 sparsity points, eager fp16 train_step)
and one 800x800 render (render_image, fp16), the four activations alternated in one process over several rounds.
Prints the card name and power limit beside the numbers.

    python scripts/bench_net_activation.py [--steps 20] [--rounds 3]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from plenoctree_b200.nerf import train as T  # noqa: E402
from plenoctree_b200.nerf.models import NerfModel, Rays  # noqa: E402
from plenoctree_b200.nerf.rays import random_rays_np  # noqa: E402
from plenoctree_b200.nerf.utils import generate_rays, pose_spherical, render_image  # noqa: E402
from scripts.bench_sigma_activation import card, timed  # noqa: E402

R, NC, NF, NSP = 4096, 64, 128, 10000
ACTS = ("relu", "elu", "softplus", "tanh")


def setup(act):
    model = NerfModel(sh_deg=3, num_coarse_samples=NC, num_fine_samples=NF, max_rays=R, sparsity_npoints=NSP,
                      net_activation=act)
    model.init_params()
    state = T.TrainState(model)
    o, d, v, px = random_rays_np(R, 0)
    batch = {"rays": Rays(*(torch.from_numpy(a).cuda() for a in (o, d, v))), "pixels": torch.from_numpy(px).cuda()}
    return model, state, batch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    runs = {act: setup(act) for act in ACTS}
    W = 800
    rays = generate_rays(W, W, 0.5 * W / np.tan(0.5 * 0.6911112070083618), pose_spherical(30.0, -30.0, 4.0)[None])
    frame = Rays(rays.origins[0], rays.directions[0], rays.viewdirs[0])
    for model, state, batch in runs.values():
        for _ in range(a.warmup):
            T.train_step(model, state, batch, 1e-4)
        render_image(model, frame)
    torch.cuda.synchronize()
    step = {k: [] for k in ACTS}
    render = {k: [] for k in ACTS}
    for _ in range(a.rounds):
        for act, (model, state, batch) in runs.items():
            step[act].append(timed(lambda: T.train_step(model, state, batch, 1e-4), a.steps))
            render[act].append(timed(lambda: render_image(model, frame), 1))
    out = dict(card=card(), workload=f"SH16 {R} rays x ({NC}+{NF}) + {NSP} sparsity points, eager fp16 train_step; "
                                     f"{W}x{W} render_image fp16",
               step_ms=step, render_800_ms=render,
               step_ratio_median={k: float(np.median(step[k]) / np.median(step["relu"])) for k in ACTS[1:]},
               render_ratio_median={k: float(np.median(render[k]) / np.median(render["relu"])) for k in ACTS[1:]})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

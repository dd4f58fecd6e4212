"""Vanilla NeRF (use_viewdirs) rendering against NeRF-SH, 1 GPU.

Times an 800 x 800 frame of utils.render_image (randomized False, chunk 8192) of a vanilla model with random weights
at (64, 128) samples against the same frame of an SH16 NeRF-SH model, and the vanilla model with a softplus trunk and
condition layer (the one vanilla instantiation whose ptxas allocation spills) against the SH16 model with a softplus
trunk, the four alternated in one process for --rounds rounds after a warm-up frame each, with a device synchronise around each frame.  Then times the vanilla eval_points
(one view direction per point) on 2^22 points with CUDA events, and splits one vanilla frame's kernel time by phase
(pob_timing: the forward with its view tables, and the per-ray stages).  Prints one JSON line with the card's name and
power limit read in the same run.

  python scripts/bench_vanilla.py [--rounds 3]
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_projection import card  # noqa: E402
from oracle import nerf_sh_oracle as O  # noqa: E402
from oracle import projection_oracle as PJ  # noqa: E402
from plenoctree_b200 import _lib  # noqa: E402
from plenoctree_b200.nerf import utils as NU  # noqa: E402
from plenoctree_b200.nerf.models import NerfModel  # noqa: E402
from plenoctree_b200.nerf.rays import generate_rays, pose_spherical  # noqa: E402
from plenoctree_b200.nerf.vanilla import VanillaNerfModel  # noqa: E402

W = 800


def frame_ms(model, rays):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    NU.render_image(model, rays, chunk=8192)
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    mlps = {"MLP_0": PJ.init_params(21), "MLP_1": PJ.init_params(22)}
    for layers in mlps.values():
        layers[8] = (layers[8][0] * 8.0, layers[8][1] + 2.0)
    van = VanillaNerfModel(mlps, max_rays=8192)
    van_sp = VanillaNerfModel(mlps, max_rays=8192, net_activation="softplus")
    sh = NerfModel(sh_deg=3, max_rays=8192)
    sh.set_params(np.concatenate([O.init_flat_params(3, 1, bias_scale=0.05), O.init_flat_params(3, 2, 0.05)]))
    sh_sp = NerfModel(sh_deg=3, max_rays=8192, net_activation="softplus")
    sh_sp.set_params(sh.params.cpu())
    r = generate_rays(W, W, 0.5 * W / np.tan(0.5 * 0.6911112070083618), pose_spherical(30.0, -30.0, 4.0)[None])
    rays = NU.Rays(*[torch.from_numpy(np.ascontiguousarray(x[0], np.float32)).cuda() for x in r])
    frame_ms(van, rays), frame_ms(sh, rays), frame_ms(van_sp, rays), frame_ms(sh_sp, rays)   # warm-up of every shape
    t_van, t_sh, t_sp, t_sh_sp = [], [], [], []
    for _ in range(a.rounds):
        t_van.append(frame_ms(van, rays))
        t_sh.append(frame_ms(sh, rays))
        t_sp.append(frame_ms(van_sp, rays))
        t_sh_sp.append(frame_ms(sh_sp, rays))
    # eval_points rate
    m = 1 << 22
    rs = np.random.RandomState(0)
    pts = torch.from_numpy(rs.uniform(-1.5, 1.5, (m, 3)).astype(np.float32)).cuda()
    vd = torch.nn.functional.normalize(torch.from_numpy(rs.normal(size=(m, 3)).astype(np.float32)), dim=-1).cuda()
    van.eval_points(pts, vd)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        van.eval_points(pts, vd)
    e1.record()
    torch.cuda.synchronize()
    pts_ms = e0.elapsed_time(e1) / 5
    # kernel time split of one vanilla frame
    _lib.lib.pob_timing_enable(1)
    NU.render_image(van, rays, chunk=8192)
    torch.cuda.synchronize()
    ms = (_lib.ctypes.c_double * 5)()
    _lib.lib.pob_timing_read(ms, None)
    _lib.lib.pob_timing_enable(0)
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power, "frame": f"{W}x{W}", "samples": [64, 128],
                      "vanilla_frame_ms": [round(x, 2) for x in t_van], "sh16_frame_ms": [round(x, 2) for x in t_sh],
                      "vanilla_over_sh16": round(min(t_van) / min(t_sh), 4),
                      "vanilla_softplus_frame_ms": [round(x, 2) for x in t_sp],
                      "sh16_softplus_frame_ms": [round(x, 2) for x in t_sh_sp],
                      "vanilla_eval_points_per_s": round(m / (pts_ms * 1e-3)),
                      "vanilla_frame_kernel_ms": {"forward_and_view_tables": round(ms[0], 2),
                                                  "per_ray_stages": round(ms[3], 2)}}))


if __name__ == "__main__":
    main()

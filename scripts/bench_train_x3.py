"""Step time of the fp16x3 training step against the fp16 step on bench.py's workload (SH degree 3, i.e. 16 SH
coefficients; 4096 rays x (64 + 128) samples, 10 000 sparsity points), eager train_step, the two alternated in one
process.  Prints the card name and power limit beside the numbers.

    python scripts/bench_train_x3.py [--steps 20] [--rounds 3] [--profile OUT_DIR]

--profile: one separate run per precision under torch.profiler (CUDA activities), per-kernel totals printed and the
tables written to OUT_DIR.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from plenoctree_b200._lib import PREC_FP16, PREC_FP16X3  # noqa: E402
from plenoctree_b200.nerf import train as T  # noqa: E402
from plenoctree_b200.nerf.models import NerfModel, Rays  # noqa: E402
from plenoctree_b200.nerf.rays import random_rays_np  # noqa: E402

R, NC, NF, NSP = 4096, 64, 128, 10000
PRECS = {"fp16": PREC_FP16, "fp16x3": PREC_FP16X3}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def setup():
    model = NerfModel(sh_deg=3, num_coarse_samples=NC, num_fine_samples=NF, max_rays=R, sparsity_npoints=NSP)
    model.init_params()
    state = T.TrainState(model)
    o, d, v, px = random_rays_np(R, 0)
    batch = {"rays": Rays(*(torch.from_numpy(a).cuda() for a in (o, d, v))), "pixels": torch.from_numpy(px).cuda()}
    return model, state, batch


def time_steps(model, state, batch, prec, steps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(steps):
        T.train_step(model, state, batch, 1e-4, precision=prec)
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", default=None)
    a = ap.parse_args()
    model, state, batch = setup()
    for prec in PRECS.values():
        for _ in range(a.warmup):
            T.train_step(model, state, batch, 1e-4, precision=prec)
    torch.cuda.synchronize()
    res = {k: [] for k in PRECS}
    for _ in range(a.rounds):
        for name, prec in PRECS.items():
            res[name].append(time_steps(model, state, batch, prec, a.steps))
    out = dict(card=card(), workload=f"SH16 {R} rays x ({NC}+{NF}) + {NSP} sparsity points, eager train_step",
               step_ms={k: v for k, v in res.items()},
               ratio_median=float(np.median(res["fp16x3"]) / np.median(res["fp16"])))
    print(json.dumps(out), flush=True)
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(a.profile, exist_ok=True)
        for name, prec in PRECS.items():
            with profile(activities=[ProfilerActivity.CUDA]) as p:
                for _ in range(5):
                    T.train_step(model, state, batch, 1e-4, precision=prec)
                torch.cuda.synchronize()
            tab = p.key_averages().table(sort_by="cuda_time_total", row_limit=20)
            open(os.path.join(a.profile, f"kernels_{name}.txt"), "w").write(tab)
            print(f"== {name} (5 steps)\n{tab}", flush=True)


if __name__ == "__main__":
    main()

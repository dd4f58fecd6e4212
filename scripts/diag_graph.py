"""Diagnostic: where does a graph-replayed train step diverge from the eager one?  Runs the four-step sequence of
tests/test_train.py::test_graphed_train_step_matches_eager in several ways (host syncs between steps or not, eager
or graph-replayed) and prints which final states are bit-identical, plus the (lr, step) pair the device held after
every replay."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from tests.support.mlp_stages import _setup
from plenoctree_b200.nerf.models import NerfModel, Rays
from plenoctree_b200.nerf import train as T

R = 256
fc, ff, rays, px, _, _, _ = _setup(3, R, 128, 0, 33)
b12 = torch.from_numpy(np.concatenate([rays[0], rays[1], rays[2], px], axis=1)).cuda()
lrs = [5e-4, 4e-4, 3e-4, 2e-4]
batch = {"rays": Rays(b12[:, 0:3], b12[:, 3:6], b12[:, 6:9]), "pixels": b12[:, 9:12]}


def make():
    model = NerfModel(sh_deg=3, max_rays=R, sparsity_npoints=1000)
    model.set_params(np.concatenate([fc, ff]))
    return model, T.TrainState(model)


def run(kind, sync):
    model, state = make()
    seen, per_step = [], []
    g = T.GraphedTrainStep(model, state, R) if kind == "graph" else None
    for lr in lrs:
        if kind == "graph":
            g.step(b12, lr)
            seen.append(state.lr_step.clone())
        elif kind == "eager_dev":
            state.lr_step.copy_(torch.tensor([lr, float(state.step)]))       # pageable source: staged synchronously
            T.train_step(model, state, batch, 123.0, lr_step_on_device=True)
        else:
            T.train_step(model, state, batch, lr)
        per_step.append((model.params.clone(), state.m.clone(), state._draw_buf.clone()))
        if sync:
            torch.cuda.synchronize()
    torch.cuda.synchronize()
    return dict(p=model.params.clone(), m=state.m.clone(), v=state.v.clone(), seen=[s.tolist() for s in seen],
                per_step=per_step)


runs = {}
for kind in ("eager", "eager_dev", "graph"):
    for sync in (True, False):
        for rep in range(2 if not sync else 1):
            runs[(kind, sync, rep)] = run(kind, sync)
ref = runs[("eager", True, 0)]
for key, r in runs.items():
    first_bad = next((i for i, (a, b) in enumerate(zip(ref["per_step"], r["per_step"]))
                      if not (torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]))), None)
    draws_bad = next((i for i, (a, b) in enumerate(zip(ref["per_step"], r["per_step"])) if not torch.equal(a[2], b[2])), None)
    print(key, "p==ref", torch.equal(ref["p"], r["p"]), "max|dp|", float((ref["p"] - r["p"]).abs().max()),
          "first step with p/m mismatch", first_bad, "first step with draw mismatch", draws_bad, "seen", r["seen"])

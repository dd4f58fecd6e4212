"""Writes tests/golden/ref_projection.npz by executing the reference's own code for the SH projection of a vanilla
NeRF (octree.extraction with use_viewdirs):

  - a torch NerfModel(use_viewdirs=True, sh_deg=4) of the reference (octree/nerf/models.py) restored by its
    restore_model_state_from_jaxnerf from a flax-format checkpoint that plenoctree_b200.nerf.checkpoints wrote (the
    Dense_0..11 numbering; flax itself is replaced by this package's msgpack reader, as make_golden.py does);
  - its eval_points_raw(points, viewdirs, cross_broadcast=True) at fixed points x directions;
  - sh_proj.ProjectFunctionNeRF through extraction's project_nerf_to_sh call pattern, with
    spherical_uniform_sampling patched to return given (theta, phi);
  - sh_proj.EvalSH of every (l, m), l <= 4, at random directions in float64.

Weights come from oracle/projection_oracle.init_params(seed), so the fixture stores seeds and outputs, not weights.
Run from the repository root: python tests/golden/make_golden_projection.py
"""
import math
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
import make_golden as G  # noqa: E402

from oracle import projection_oracle as PJ  # noqa: E402

SEEDS = (5101, 5102)
SH_DEG = 4


def main():
    from plenoctree_b200.nerf import checkpoints as C
    G._use_reference_octree()
    from octree.nerf import models as ref_models
    from octree.nerf import sh_proj
    mlps = {"MLP_0": PJ.init_params(SEEDS[0]), "MLP_1": PJ.init_params(SEEDS[1])}
    tmp = tempfile.mkdtemp()
    sd = {"optimizer": {"target": {"params": C.vanilla_to_flax_params(mlps)}}}
    with open(os.path.join(tmp, "checkpoint_7"), "wb") as f:
        f.write(C.msgpack_serialize(sd))
    fake_flax = types.ModuleType("flax")
    fake_training = types.ModuleType("flax.training")
    fake_ckpt = types.ModuleType("flax.training.checkpoints")
    fake_ckpt.restore_checkpoint = lambda train_dir, target=None: C.restore_flax_state_dict(train_dir)
    fake_training.checkpoints = fake_ckpt
    fake_flax.training = fake_training
    sys.modules.update({"flax": fake_flax, "flax.training": fake_training, "flax.training.checkpoints": fake_ckpt})
    try:
        model = ref_models.NerfModel(use_viewdirs=True, sh_deg=SH_DEG, num_rgb_channels=3, num_coarse_samples=64,
                                     num_fine_samples=128)
        model = ref_models.restore_model_state_from_jaxnerf(types.SimpleNamespace(train_dir=tmp), model).eval()
    finally:
        for k in ("flax", "flax.training", "flax.training.checkpoints"):
            sys.modules.pop(k, None)
    rs = np.random.RandomState(5103)
    pts = rs.uniform(-1.2, 1.2, size=(24, 3)).astype(np.float32)
    theta = np.arccos(2.0 * rs.uniform(size=40) - 1.0).astype(np.float32)
    phi = (2.0 * math.pi * rs.uniform(size=40)).astype(np.float32)
    with torch.no_grad():
        dirs = sh_proj.spher2cart(torch.from_numpy(theta), torch.from_numpy(phi))
        raw_rgb, raw_sigma = model.eval_points_raw(torch.from_numpy(pts), dirs, cross_broadcast=True)
        orig = sh_proj.spherical_uniform_sampling
        sh_proj.spherical_uniform_sampling = lambda n, device="cpu": (torch.from_numpy(theta).to(device),
                                                                      torch.from_numpy(phi).to(device))
        try:
            out = {}
            for deg in range(1, 5):   # extraction.project_nerf_to_sh: the model's rgb at every (point, direction)
                coeffs, sigma = sh_proj.ProjectFunctionNeRF(
                    order=deg, sperical_func=lambda v: model.eval_points_raw(torch.from_numpy(pts), v,
                                                                             cross_broadcast=True),
                    batch_size=pts.shape[0], sample_count=theta.shape[0], device="cpu")
                out[f"coeffs_deg{deg}"] = coeffs.reshape(pts.shape[0], -1).numpy()
                out[f"sigma_deg{deg}"] = sigma.numpy()
        finally:
            sh_proj.spherical_uniform_sampling = orig
    bdirs = rs.normal(size=(64, 3))
    bdirs /= np.linalg.norm(bdirs, axis=1, keepdims=True)
    bt = torch.from_numpy(bdirs)
    evalsh = np.stack([sh_proj.EvalSH(l, m, bt).numpy() for l in range(5) for m in range(-l, l + 1)], axis=-1)
    state = model.state_dict()
    keys = sorted(state)
    np.savez_compressed(os.path.join(HERE, "ref_projection.npz"), seeds=np.array(SEEDS), sh_deg=SH_DEG, deg_view=4,
                        points=pts, theta=theta, phi=phi, dirs=dirs.numpy(), raw_rgb=raw_rgb.numpy(),
                        raw_sigma=raw_sigma.numpy(), basis_dirs=bdirs, evalsh=evalsh, keys=np.array(keys),
                        sums=np.array([float(state[k].double().sum()) for k in keys]), **out)
    print("ref_projection.npz", raw_rgb.shape, len(keys), "tensors")


if __name__ == "__main__":
    main()

"""Writes tests/golden/ref_vanilla.npz by executing the reference's own code for a vanilla NeRF (use_viewdirs,
sh_deg -1), the model nerf_sh.eval renders with --config nerf_sh/config/misc/og_nerf:

  - nerf_sh/nerf/models.py::NerfModel.__call__ and model_utils.py, unmodified, over the numpy stand-ins for jax / flax
    (tests/golden/jax_stub.py, as make_golden.py runs the NeRF-SH forward), 64 + 128 samples, deterministic and
    randomized with injected draws (stratified jitter, inverse-CDF uniforms and, randomized, noise_std 0.7 density
    noise), for four models: deg_view 4 standard order relu (built from the flags of the reference's
    nerf_sh/config/misc/og_nerf.yaml read by its update_flags rule), deg_view 10 legacy order, deg_view 0, and an
    elu trunk and condition layer with softplus density.  The coarse and fine depths the reference used are recorded
    by wrapping model_utils.sample_along_rays / sample_pdf (their results pass through unchanged), so a renderer can be
    run on the reference's own fine depths;
  - the torch twin octree/nerf/models.py::NerfModel(use_viewdirs=True).eval_points_raw(points, viewdirs) (one view
    direction per point), restored by its restore_model_state_from_jaxnerf from a flax-format checkpoint written by
    plenoctree_b200.nerf.checkpoints, fine and coarse MLP, for the relu models.

Weights come from tests/support/vanilla_ref.golden_layers (oracle/projection_oracle.init_params with the Dense_8
kernel scaled by SIGMA_SCALE and SIGMA_SHIFT added to its bias: partially opaque rays); the fixture stores seeds and
outputs, not weights.  Run from the repository root: python tests/golden/make_golden_vanilla.py
"""
import collections
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
import make_golden as G  # noqa: E402

from oracle import nerf_sh_oracle as O  # noqa: E402
from tests.support import vanilla_ref as VR  # noqa: E402

SIGMA_SCALE, SIGMA_SHIFT = 4.0, 0.5
NOISE_STD = 0.7
B, NC, NF = 32, 64, 128
# tag -> (seed, deg_view, legacy_posenc_order, net_activation, sigma_activation)
CASES = {"og_nerf": (6101, 4, False, "relu", "relu"), "dv10_legacy": (6111, 10, True, "relu", "relu"),
         "dv0": (6121, 0, False, "relu", "relu"), "elu_softplus": (6131, 4, False, "elu", "softplus")}


def layers_of(seed, deg_view, legacy):
    return VR.golden_layers(seed, deg_view, legacy, SIGMA_SCALE, SIGMA_SHIFT)


def og_nerf_flags():
    """utils.update_flags (nerf_sh/nerf/utils.py:233-244) of the reference's og_nerf config onto its flag defaults"""
    with open(os.path.join(G.REF, "nerf_sh", "config", "misc", "og_nerf.yaml")) as f:
        return yaml.load(f, Loader=yaml.FullLoader)


def gen_call(out):
    import jax_stub
    names = jax_stub.install()
    fake_utils = types.ModuleType("nerf_sh.nerf.utils")
    fake_utils.Rays = collections.namedtuple("Rays", ("origins", "directions", "viewdirs"))
    fake_utils.TrainState = object
    sys.modules["nerf_sh.nerf.utils"] = fake_utils
    try:
        from nerf_sh.nerf import model_utils as MU
        from nerf_sh.nerf import models as RM
        import flax.linen as nn
        nn.elu = lambda x: np.where(x > 0, x, np.expm1(np.minimum(x, np.float32(0)))).astype(np.float32)
        acts = {"relu": nn.relu, "elu": nn.elu, "softplus": nn.softplus}
        rs = np.random.RandomState(6100)
        poses = np.stack([O.pose_spherical(rs.uniform(-180, 180), rs.uniform(-90, 0), 4.0) for _ in range(4)])
        rays_all = O.generate_rays(40, 30, 55.5, poses)
        pick = rs.choice(4 * 30 * 40, B, replace=False)
        o, d, v = [np.ascontiguousarray(np.asarray(r).reshape(-1, 3)[pick]).astype(np.float32) for r in rays_all]
        t_rand = rs.uniform(size=(B, NC)).astype(np.float32)
        u_f = rs.uniform(size=(B, NF)).astype(np.float32)
        n_c = rs.normal(size=(B, NC, 1)).astype(np.float32)
        n_f = rs.normal(size=(B, NC + NF, 1)).astype(np.float32)
        out.update(origins=o, directions=d, viewdirs=v, t_rand=t_rand, u=u_f, noise_coarse=n_c, noise_fine=n_f)
        flags = og_nerf_flags()
        out["og_nerf_config"] = np.array(json.dumps(flags, sort_keys=True))
        depths = []
        orig_sar, orig_pdf = MU.sample_along_rays, MU.sample_pdf

        def sar(*a, **k):
            z, p = orig_sar(*a, **k)
            depths.append(np.asarray(z))
            return z, p

        def pdf(*a, **k):
            z, p = orig_pdf(*a, **k)
            depths.append(np.asarray(z))
            return z, p
        MU.sample_along_rays, MU.sample_pdf = sar, pdf
        try:
            for tag, (seed, dv, legacy, act, sact) in CASES.items():
                mlps = layers_of(seed, dv, legacy)
                nc, nf, wb = ((flags["num_coarse_samples"], flags["num_fine_samples"], flags["white_bkgd"])
                              if tag == "og_nerf" else (NC, NF, True))
                model = RM.NerfModel(num_coarse_samples=nc, num_fine_samples=nf, use_viewdirs=True, sh_deg=-1,
                                     sg_dim=-1, near=2.0, far=6.0, noise_std=NOISE_STD, net_depth=8, net_width=256,
                                     net_depth_condition=1, net_width_condition=128, net_activation=acts[act],
                                     skip_layer=4, num_rgb_channels=3, num_sigma_channels=1, white_bkgd=wb,
                                     min_deg_point=0, max_deg_point=10, deg_view=dv, lindisp=False,
                                     rgb_activation=nn.sigmoid, sigma_activation=acts[sact],
                                     legacy_posenc_order=legacy)
                model.MLP_0._params = mlps["MLP_0"]
                model.MLP_1._params = mlps["MLP_1"]
                for rtag, rnd in (("det", False), ("rand", True)):
                    depths.clear()
                    ret = model(jax_stub.Key(uniform=t_rand, normal=n_c), jax_stub.Key(uniform=u_f, normal=n_f),
                                fake_utils.Rays(o, d, v), rnd)
                    out[f"{tag}_{rtag}_z_coarse"], out[f"{tag}_{rtag}_z_fine"] = depths
                    for lvl, (c, di, ac) in zip(("coarse", "fine"), ret):
                        out[f"{tag}_{rtag}_{lvl}_rgb"], out[f"{tag}_{rtag}_{lvl}_disp"] = np.asarray(c), np.asarray(di)
                        out[f"{tag}_{rtag}_{lvl}_acc"] = np.asarray(ac)
        finally:
            MU.sample_along_rays, MU.sample_pdf = orig_sar, orig_pdf
    finally:
        jax_stub.uninstall(names)
        for k in [k for k in sys.modules if k.startswith("nerf_sh")]:
            sys.modules.pop(k, None)


def gen_twin(out):
    from plenoctree_b200.nerf import checkpoints as C
    G._use_reference_octree()
    from octree.nerf import models as ref_models
    rs = np.random.RandomState(6200)
    pts = rs.uniform(-1.2, 1.2, size=(48, 3)).astype(np.float32)
    vd = rs.normal(size=(48, 3))
    vd = (vd / np.linalg.norm(vd, axis=1, keepdims=True)).astype(np.float32)
    out.update(twin_points=pts, twin_viewdirs=vd)
    for tag, (seed, dv, legacy, act, _) in CASES.items():
        if act != "relu":
            continue
        mlps = layers_of(seed, dv, legacy)
        tmp = tempfile.mkdtemp()
        with open(os.path.join(tmp, "checkpoint_7"), "wb") as f:
            f.write(C.msgpack_serialize({"optimizer": {"target": {"params": C.vanilla_to_flax_params(mlps)}}}))
        fake_flax = types.ModuleType("flax")
        fake_training = types.ModuleType("flax.training")
        fake_ckpt = types.ModuleType("flax.training.checkpoints")
        fake_ckpt.restore_checkpoint = lambda train_dir, target=None: C.restore_flax_state_dict(train_dir)
        fake_training.checkpoints = fake_ckpt
        fake_flax.training = fake_training
        sys.modules.update({"flax": fake_flax, "flax.training": fake_training, "flax.training.checkpoints": fake_ckpt})
        try:
            model = ref_models.NerfModel(use_viewdirs=True, sh_deg=-1, num_rgb_channels=3, num_coarse_samples=64,
                                         num_fine_samples=128, deg_view=dv, legacy_posenc_order=legacy)
            model = ref_models.restore_model_state_from_jaxnerf(types.SimpleNamespace(train_dir=tmp), model).eval()
        finally:
            for k in ("flax", "flax.training", "flax.training.checkpoints"):
                sys.modules.pop(k, None)
        with torch.no_grad():
            for coarse in (False, True):
                rgb, sigma = model.eval_points_raw(torch.from_numpy(pts), torch.from_numpy(vd), coarse=coarse)
                key = f"twin_{tag}_{'coarse' if coarse else 'fine'}"
                out[key + "_raw_rgb"], out[key + "_raw_sigma"] = rgb.numpy(), sigma.numpy()


def main():
    out = {}
    gen_call(out)
    gen_twin(out)
    out["cases"] = np.array(json.dumps(CASES))
    out["sigma_scale_shift"] = np.array([SIGMA_SCALE, SIGMA_SHIFT], np.float32)
    out["noise_std"] = np.float32(NOISE_STD)
    assert all(np.asarray(a).dtype != np.float64 for a in out.values()), "float64 leaked through the stand-ins"
    np.savez_compressed(os.path.join(HERE, "ref_vanilla.npz"), **out)
    print("ref_vanilla.npz", len(out), "arrays")


if __name__ == "__main__":
    main()

"""Generate tests/golden/ref_posenc.npz by EXECUTING the reference's point encoder and models with the flags
min_deg_point, max_deg_point and legacy_posenc_order (nerf_sh/nerf/utils.py:119-124,155-159):

  - the JAX posenc (nerf_sh/nerf/model_utils.py:145-173) and NerfModel.__call__ (nerf_sh/nerf/models.py:216-348),
    unmodified over the numpy stand-ins for jax / flax (tests/golden/jax_stub.py);
  - the torch twin's posenc (octree/nerf/model_utils.py:161-190) and NerfModel.eval_points_raw
    (octree/nerf/models.py:211-252) with the same flags;
  - the torch twin's restore_model_state_from_jaxnerf (octree/nerf/models.py:66-113) loading a flax checkpoint that
    plenoctree_b200.nerf.checkpoints wrote for a model with a non-default encoder.

    python tests/golden/make_golden_posenc.py

It runs in its own process because importing the reference's nerf_sh package defines its flags.
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, O, _use_reference_octree  # noqa: E402
from oracle import posenc_oracle as PO  # noqa: E402

# (min_deg, max_deg, legacy): the default order's legacy twin, a narrower range in both orders, the bare point, and a
# range that starts above 0
VARIANTS = [(0, 10, True), (2, 8, False), (2, 8, True), (0, 0, False), (3, 10, False)]
CKPT_VARIANT = (2, 8, True)
SH_DEG = 2


def tag(pe):
    return f"{pe[0]}_{pe[1]}_{'legacy' if pe[2] else 'std'}"


def gen_ref_posenc():
    import jax_stub
    rs = np.random.RandomState(2718)
    x = rs.uniform(-4, 4, size=(64, 3)).astype(np.float32)
    x[:4] = [[0, 0, 0], [1.5, -1.5, 1.5], [-4, 4, -4], [1e-3, -2e-3, 3e-3]]
    poses = np.stack([O.pose_spherical(rs.uniform(-180, 180), rs.uniform(-90, 0), 4.0) for _ in range(2)])
    rays_all = O.generate_rays(20, 15, 27.75, poses)
    B = 8
    pick = rs.choice(2 * 15 * 20, B, replace=False)
    o, d, v = [np.ascontiguousarray(np.asarray(r).reshape(-1, 3)[pick]).astype(np.float32) for r in rays_all]
    pts = rs.uniform(-1.5, 1.5, size=(48, 3)).astype(np.float32)
    out = dict(x=x, origins=o, directions=d, viewdirs=v, points=pts, sh_deg=SH_DEG,
               variants=np.array(VARIANTS, dtype=np.int32), ckpt_variant=np.array(CKPT_VARIANT, dtype=np.int32))
    flats = {}
    for k, pe in enumerate(VARIANTS):
        flats[pe] = [PO.init_flat_params(SH_DEG, 9100 + 10 * k + m, bias_scale=0.05, pe=pe) for m in range(2)]

    # ---- the JAX model over the numpy stand-ins ----
    names = jax_stub.install()
    fake_ds = types.ModuleType("nerf_sh.nerf.datasets")
    fake_ds.dataset_dict = {"blender": None, "llff": None, "nsvf": None}
    sys.modules["nerf_sh.nerf.datasets"] = fake_ds
    try:
        from nerf_sh.nerf import models as RM, utils as RU
        import nerf_sh.nerf.model_utils as MU
        import flax.linen as nn
        for pe in VARIANTS:
            out[f"jax_enc_{tag(pe)}"] = np.asarray(MU.posenc(x, pe[0], pe[1], pe[2])).astype(np.float32)

            def ptree(flat):
                return {f"Dense_{j}": {"kernel": w.numpy(), "bias": b.numpy()}
                        for j, (w, b) in enumerate(PO.unflatten(flat, SH_DEG, pe))}
            variables = {"params": {"MLP_0": ptree(flats[pe][0]), "MLP_1": ptree(flats[pe][1])}}
            model = RM.NerfModel(num_coarse_samples=32, num_fine_samples=32, use_viewdirs=False, sh_deg=SH_DEG,
                                 sg_dim=-1, near=2.0, far=6.0, noise_std=None, net_depth=8, net_width=256,
                                 net_depth_condition=1, net_width_condition=128, net_activation=nn.relu, skip_layer=4,
                                 num_rgb_channels=3 * (SH_DEG + 1) ** 2, num_sigma_channels=1, white_bkgd=True,
                                 min_deg_point=pe[0], max_deg_point=pe[1], deg_view=4, lindisp=False,
                                 rgb_activation=nn.sigmoid, sigma_activation=nn.relu, legacy_posenc_order=pe[2])
            ret = model.apply(variables, jax_stub.Key(seed=2), jax_stub.Key(seed=3), RU.Rays(o, d, v), False)
            for lvl, (c, di, ac) in zip(("coarse", "fine"), ret):
                out[f"call_{tag(pe)}_{lvl}_rgb"] = np.asarray(c).astype(np.float32)
                out[f"call_{tag(pe)}_{lvl}_disp"] = np.asarray(di).astype(np.float32)
                out[f"call_{tag(pe)}_{lvl}_acc"] = np.asarray(ac).astype(np.float32)
    finally:
        jax_stub.uninstall(names)
        for k in [k for k in sys.modules if k.startswith("nerf_sh")]:
            sys.modules.pop(k, None)

    # ---- the torch twin ----
    _use_reference_octree()
    from octree.nerf import model_utils as ref_mu, models as ref_models
    K = (SH_DEG + 1) ** 2

    def twin(pe):
        return ref_models.NerfModel(use_viewdirs=False, sh_deg=SH_DEG, num_rgb_channels=3 * K, num_coarse_samples=32,
                                    num_fine_samples=32, min_deg_point=pe[0], max_deg_point=pe[1],
                                    legacy_posenc_order=pe[2])
    for pe in VARIANTS:
        out[f"torch_enc_{tag(pe)}"] = ref_mu.posenc(torch.from_numpy(x), pe[0], pe[1], pe[2]).numpy()
        model = twin(pe)
        for name, flat in zip(("MLP_0", "MLP_1"), flats[pe]):
            mlp = getattr(model, name)
            params = PO.unflatten(flat, SH_DEG, pe)
            with torch.no_grad():
                for i in range(8):
                    mlp.input_layers[i].weight.copy_(params[i][0].T)
                    mlp.input_layers[i].bias.copy_(params[i][1])
                mlp.sigma_layer.weight.copy_(params[8][0].T)
                mlp.sigma_layer.bias.copy_(params[8][1])
                mlp.rgb_layer.weight.copy_(params[9][0].T)
                mlp.rgb_layer.bias.copy_(params[9][1])
        with torch.no_grad():
            rgb, sig = model.eval().eval_points_raw(torch.from_numpy(pts))
        out[f"twin_raw_rgb_{tag(pe)}"], out[f"twin_raw_sigma_{tag(pe)}"] = rgb.numpy(), sig.numpy()

    # ---- the twin's loader on a flax checkpoint written here for a non-default encoder ----
    from plenoctree_b200.nerf import checkpoints as C
    pe = CKPT_VARIANT
    flat = np.concatenate(flats[pe])
    step = 321
    blob = C.msgpack_serialize(C.train_state_dict(flat, flat * 0, flat * 0, step, SH_DEG, pe))
    tmp = tempfile.mkdtemp()
    with open(os.path.join(tmp, f"checkpoint_{step}"), "wb") as f:
        f.write(blob)
    fake_flax = types.ModuleType("flax")
    fake_training = types.ModuleType("flax.training")
    fake_ckpt = types.ModuleType("flax.training.checkpoints")
    fake_ckpt.restore_checkpoint = lambda train_dir, target=None: C.restore_flax_state_dict(train_dir)
    fake_training.checkpoints = fake_ckpt
    fake_flax.training = fake_training
    sys.modules.update({"flax": fake_flax, "flax.training": fake_training, "flax.training.checkpoints": fake_ckpt})
    try:
        model = ref_models.restore_model_state_from_jaxnerf(types.SimpleNamespace(train_dir=tmp), twin(pe)).eval()
    finally:
        for k in ("flax", "flax.training", "flax.training.checkpoints"):
            sys.modules.pop(k, None)
    with torch.no_grad():
        rgb_f, sig_f = model.eval_points_raw(torch.from_numpy(pts))
        rgb_c, sig_c = model.eval_points_raw(torch.from_numpy(pts), coarse=True)
    sd = model.state_dict()
    out.update(ckpt_raw_rgb_fine=rgb_f.numpy(), ckpt_raw_sigma_fine=sig_f.numpy(), ckpt_raw_rgb_coarse=rgb_c.numpy(),
               ckpt_raw_sigma_coarse=sig_c.numpy(),
               ckpt_dense0_shape=np.array(sd["MLP_1.input_layers.0.weight"].shape),
               ckpt_dense5_shape=np.array(sd["MLP_1.input_layers.5.weight"].shape))
    assert all(np.asarray(a).dtype != np.float64 for a in out.values() if isinstance(a, np.ndarray))
    np.savez_compressed(os.path.join(HERE, "ref_posenc.npz"), **out)
    print("ref_posenc.npz", len(out), "arrays")


if __name__ == "__main__":
    torch.manual_seed(20200823)
    torch.set_num_threads(8)
    gen_ref_posenc()

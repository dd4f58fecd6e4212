"""Generate tests/golden/ref_net_activation.npz by EXECUTING the reference with the trunk activations of the flag
net_activation (nerf_sh/nerf/models.py:362, octree/nerf/models.py:265; applied after every trunk layer,
model_utils.py:69), once per activation elu / softplus / tanh:

  - the JAX NerfModel.__call__ (nerf_sh/nerf/models.py:216-348) and train_step's loss (nerf_sh/train.py:51-116) with
    nn.elu / nn.softplus / nn.tanh, unmodified over the numpy stand-ins for jax / flax (tests/golden/jax_stub.py, with
    elu and tanh added here), as make_golden_softplus.py does;
  - the torch twin's NerfModel.eval_points_raw (octree/nerf/models.py:211-252) with torch.nn.ELU / Softplus / Tanh;
  - the twin's restore_model_state_from_jaxnerf (octree/nerf/models.py:66-113) loading a flax checkpoint that
    plenoctree_b200.nerf.checkpoints wrote (the checkpoint does not record the activation, in the reference either).

    python tests/golden/make_golden_net_activation.py

The trunk kernels are scaled so that every layer's pre-activations span both signs over several units: the three
activations then differ from relu, and from each other, on every layer.  It runs in its own process because importing
the reference's nerf_sh package defines its flags.
"""
import dataclasses
import os
import sys
import tempfile
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, O, _use_reference_octree  # noqa: E402

ACTIVATIONS = ("elu", "softplus", "tanh")                    # flax names; the twin's classes: ELU, Softplus, Tanh
TORCH_CLASSES = {"elu": "ELU", "softplus": "Softplus", "tanh": "Tanh"}
SH_DEG, B, N, NF, NSP = 3, 16, 64, 128, 40
TRUNK_SCALE = 1.3          # Dense_0..Dense_7 kernels
SIGMA_SCALE = 10.0         # Dense_8 kernel (as make_golden_softplus.py)
SEEDS = (7301, 7302)


def scaled_flats():
    """the two MLPs' flat parameters (oracle initialisation, biases 0.05) with the trunk and sigma kernels scaled"""
    flats = []
    dims = O.layer_dims(SH_DEG)
    for s in SEEDS:
        f = O.init_flat_params(SH_DEG, s, bias_scale=0.05)
        off = 0
        for j, (a, b) in enumerate(dims):
            if j < 8:
                f[off:off + a * b] *= TRUNK_SCALE
            elif j == 8:
                f[off:off + a * b] *= SIGMA_SCALE
            off += a * b + b
        flats.append(f)
    return flats


def inputs():
    rs = np.random.RandomState(4242)
    poses = np.stack([O.pose_spherical(rs.uniform(-180, 180), rs.uniform(-90, 0), 4.0) for _ in range(3)])
    rays_all = O.generate_rays(40, 30, 55.5, poses)
    pick = rs.choice(3 * 30 * 40, B, replace=False)
    o, d, v = [np.ascontiguousarray(np.asarray(r).reshape(-1, 3)[pick]).astype(np.float32) for r in rays_all]
    px = rs.uniform(size=(B, 3)).astype(np.float32)
    t_rand = rs.uniform(size=(B, N)).astype(np.float32)
    u_f = rs.uniform(size=(B, NF)).astype(np.float32)
    sp01 = rs.uniform(size=(NSP, 3)).astype(np.float32)
    pts = rs.uniform(-1.5, 1.5, size=(64, 3)).astype(np.float32)
    return o, d, v, px, t_rand, u_f, sp01, pts


def gen_jax(out, flats, o, d, v, px, t_rand, u_f, sp01):
    import jax_stub
    names = jax_stub.install()
    fake_ds = types.ModuleType("nerf_sh.nerf.datasets")
    fake_ds.dataset_dict = {"blender": None, "llff": None, "nsvf": None}
    sys.modules["nerf_sh.nerf.datasets"] = fake_ds
    try:
        from absl import flags
        import nerf_sh.train as RT
        from nerf_sh.nerf import models as RM, utils as RU
        import nerf_sh.nerf.model_utils as MU
        import flax.linen as nn
        import jax.random as jr
        # the stand-ins of flax.linen's elu and tanh (jax_stub.py carries relu, sigmoid and softplus)
        nn.elu = lambda x: np.where(x > 0, x, np.expm1(np.minimum(x, np.float32(0)))).astype(np.float32)
        nn.tanh = lambda x: np.tanh(x).astype(np.float32)
        FLAGS = flags.FLAGS
        FLAGS(["make_golden"])
        FLAGS.randomized = True
        FLAGS.sparsity_weight = 1e-2
        FLAGS.sparsity_npoints = NSP
        FLAGS.sparsity_radius = 1.5
        FLAGS.sparsity_length = 0.05
        FLAGS.weight_decay_mult = 0.25

        def ptree(flat):
            return {f"Dense_{j}": {"kernel": w.numpy(), "bias": b.numpy()} for j, (w, b) in enumerate(O.unflatten(flat, SH_DEG))}
        variables = {"params": {"MLP_0": ptree(flats[0]), "MLP_1": ptree(flats[1])}}
        # every key carries the injected draws, told apart by shape ([B,N] jitter, [B,NF] inverse-CDF uniforms,
        # [NSP,3] sparsity points)
        table = {tuple(t_rand.shape): t_rand, tuple(u_f.shape): u_f, tuple(sp01.shape): sp01}
        orig_uniform = jr.uniform

        def uniform(key, shape, dtype=np.float32, minval=0.0, maxval=1.0):
            base = table[tuple(shape)]
            return (base * np.float32(maxval - minval) + np.float32(minval)).astype(np.float32)
        jr.uniform = RT.random.uniform = MU.random.uniform = uniform
        try:
            for act in ACTIVATIONS:
                model = RM.NerfModel(num_coarse_samples=N, num_fine_samples=NF, use_viewdirs=False, sh_deg=SH_DEG,
                                     sg_dim=-1, near=2.0, far=6.0, noise_std=None, net_depth=8, net_width=256,
                                     net_depth_condition=1, net_width_condition=128, net_activation=getattr(nn, act),
                                     skip_layer=4, num_rgb_channels=3 * (SH_DEG + 1) ** 2, num_sigma_channels=1,
                                     white_bkgd=True, min_deg_point=0, max_deg_point=10, deg_view=4, lindisp=False,
                                     rgb_activation=nn.sigmoid, sigma_activation=nn.relu, legacy_posenc_order=False)
                for tag, rnd in (("det", False), ("rand", True)):
                    ret = model.apply(variables, jax_stub.Key(seed=2), jax_stub.Key(seed=3), RU.Rays(o, d, v), rnd)
                    for lvl, (c, di, ac) in zip(("coarse", "fine"), ret):
                        out[f"{act}_call_{tag}_{lvl}_rgb"] = np.asarray(c).astype(np.float32)
                        out[f"{act}_call_{tag}_{lvl}_disp"] = np.asarray(di).astype(np.float32)
                        out[f"{act}_call_{tag}_{lvl}_acc"] = np.asarray(ac).astype(np.float32)

                @dataclasses.dataclass
                class Opt:
                    target: dict

                    def apply_gradient(self, grad, learning_rate=None):
                        return self
                state = RU.TrainState(optimizer=Opt(variables))
                _, stats, _ = RT.train_step(model, jax_stub.Key(seed=1), state,
                                            {"rays": RU.Rays(o, d, v), "pixels": px}, 5e-4)
                for k in ("loss", "psnr", "loss_c", "psnr_c", "loss_sp", "weight_l2"):
                    out[f"{act}_{k}"] = np.float32(getattr(stats, k))
        finally:
            jr.uniform = orig_uniform
    finally:
        jax_stub.uninstall(names)
        for k in [k for k in sys.modules if k.startswith("nerf_sh")]:
            sys.modules.pop(k, None)


def gen_twin(out, flats, pts):
    _use_reference_octree()
    from octree.nerf import models as ref_models
    K = (SH_DEG + 1) ** 2

    def twin(act):
        return ref_models.NerfModel(use_viewdirs=False, sh_deg=SH_DEG, num_rgb_channels=3 * K, num_coarse_samples=N,
                                    num_fine_samples=NF, net_activation=getattr(torch.nn, TORCH_CLASSES[act])())
    for act in ACTIVATIONS:
        model = twin(act)
        for name, flat in zip(("MLP_0", "MLP_1"), flats):
            mlp = getattr(model, name)
            params = O.unflatten(flat, SH_DEG)
            with torch.no_grad():
                for i in range(8):
                    mlp.input_layers[i].weight.copy_(params[i][0].T)
                    mlp.input_layers[i].bias.copy_(params[i][1])
                mlp.sigma_layer.weight.copy_(params[8][0].T)
                mlp.sigma_layer.bias.copy_(params[8][1])
                mlp.rgb_layer.weight.copy_(params[9][0].T)
                mlp.rgb_layer.bias.copy_(params[9][1])
        with torch.no_grad():
            rgb_f, sig_f = model.eval().eval_points_raw(torch.from_numpy(pts))
            rgb_c, sig_c = model.eval_points_raw(torch.from_numpy(pts), coarse=True)
        out[f"{act}_twin_raw_rgb_fine"], out[f"{act}_twin_raw_sigma_fine"] = rgb_f.numpy(), sig_f.numpy()
        out[f"{act}_twin_raw_rgb_coarse"], out[f"{act}_twin_raw_sigma_coarse"] = rgb_c.numpy(), sig_c.numpy()

    # the twin's loader on a flax checkpoint written by this package, into a model of each activation
    from plenoctree_b200.nerf import checkpoints as C
    flat = np.concatenate(flats)
    step = 654
    blob = C.msgpack_serialize(C.train_state_dict(flat, flat * 0, flat * 0, step, SH_DEG))
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
        for act in ACTIVATIONS:
            model = ref_models.restore_model_state_from_jaxnerf(types.SimpleNamespace(train_dir=tmp), twin(act)).eval()
            with torch.no_grad():
                rgb_f, sig_f = model.eval_points_raw(torch.from_numpy(pts))
            out[f"{act}_ckpt_raw_rgb_fine"], out[f"{act}_ckpt_raw_sigma_fine"] = rgb_f.numpy(), sig_f.numpy()
            if act == ACTIVATIONS[0]:
                sd = model.state_dict()
                out["ckpt_state_keys"] = np.array(sorted(sd.keys()))
                for k in ("MLP_0.input_layers.0.weight", "MLP_1.input_layers.5.weight", "MLP_1.rgb_layer.bias"):
                    out["ckpt_sd_" + k.replace(".", "_")] = sd[k].numpy()[:4]      # shape-defining slice: first rows
    finally:
        for k in ("flax", "flax.training", "flax.training.checkpoints"):
            sys.modules.pop(k, None)


def gen_ref_net_activation():
    flats = scaled_flats()
    o, d, v, px, t_rand, u_f, sp01, pts = inputs()
    out = dict(origins=o, directions=d, viewdirs=v, pixels=px, t_rand=t_rand, u=u_f, sp01=sp01, points=pts,
               sh_deg=SH_DEG, seeds=np.array(SEEDS), trunk_scale=np.float32(TRUNK_SCALE),
               sigma_scale=np.float32(SIGMA_SCALE), sparsity_weight=1e-2, sparsity_radius=1.5, sparsity_length=0.05,
               weight_decay_mult=0.25, ckpt_step=654)
    gen_jax(out, flats, o, d, v, px, t_rand, u_f, sp01)
    gen_twin(out, flats, pts)
    assert all(np.asarray(a).dtype != np.float64 for a in out.values() if isinstance(a, np.ndarray))
    np.savez_compressed(os.path.join(HERE, "ref_net_activation.npz"), **out)
    print("ref_net_activation.npz", {k: float(out[k]) for k in out if k.endswith("_loss")})


if __name__ == "__main__":
    torch.manual_seed(20200823)
    torch.set_num_threads(8)
    gen_ref_net_activation()

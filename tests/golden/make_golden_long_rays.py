"""Generate tests/golden/ref_long_rays.npz by EXECUTING the reference's NerfModel.__call__ and train_step (the
reference tree make_golden.py reads, whose helpers this imports) at sample counts past 256 per ray, (Nc, Nf) =
(128, 384) and (256, 768), unmodified over the numpy stand-ins for jax / flax (tests/golden/jax_stub.py).

    python tests/golden/make_golden_long_rays.py

The harness restates make_golden_softplus.py's (fake dataset module, injected draws told apart by shape, an identity
optimizer); it runs in its own process because importing nerf_sh.train defines the reference's flags.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, O  # noqa: E402

SIZES = ((128, 384), (256, 768))
LOSS_SIZE = (128, 384)


def gen_ref_long_rays():
    """The reference's NerfModel.__call__ (deterministic, and randomized with injected draws) at every (Nc, Nf) of
    SIZES, and train_step's loss_fn at LOSS_SIZE, executed unmodified over the numpy stand-ins."""
    import dataclasses
    import types
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
        FLAGS = flags.FLAGS
        FLAGS(["make_golden"])
        sh_deg, B, NSP = 3, 32, 40
        FLAGS.randomized = True
        FLAGS.sparsity_weight = 1e-2
        FLAGS.sparsity_npoints = NSP
        FLAGS.sparsity_radius = 1.5
        FLAGS.sparsity_length = 0.05
        FLAGS.weight_decay_mult = 0.25
        rs = np.random.RandomState(1702)
        poses = np.stack([O.pose_spherical(rs.uniform(-180, 180), rs.uniform(-90, 0), 4.0) for _ in range(3)])
        rays_all = O.generate_rays(40, 30, 55.5, poses)
        pick = rs.choice(3 * 30 * 40, B, replace=False)
        o, d, v = [np.ascontiguousarray(np.asarray(r).reshape(-1, 3)[pick]).astype(np.float32) for r in rays_all]
        px = rs.uniform(size=(B, 3)).astype(np.float32)
        sp01 = rs.uniform(size=(NSP, 3)).astype(np.float32)
        seeds = (7201, 7202)
        # Dense_8 (sigma) scaled by 10: the random-init field then has opaque and empty stretches along each ray, so
        # the fine level's samples concentrate and the weights are not flat
        flats = []
        for s in seeds:
            f = O.init_flat_params(sh_deg, s, bias_scale=0.05)
            w8 = sum(a * b + b for a, b in O.layer_dims(sh_deg)[:8])
            f[w8:w8 + 256] *= 10.0
            flats.append(f)

        def ptree(flat):
            return {f"Dense_{j}": {"kernel": w.numpy(), "bias": b.numpy()} for j, (w, b) in enumerate(O.unflatten(flat, sh_deg))}
        variables = {"params": {"MLP_0": ptree(flats[0]), "MLP_1": ptree(flats[1])}}
        out = dict(origins=o, directions=d, viewdirs=v, pixels=px, sp01=sp01, sh_deg=sh_deg, seeds=np.array(seeds),
                   sigma_head_scale=np.float32(10.0), sizes=np.array(SIZES), loss_size=np.array(LOSS_SIZE),
                   sparsity_weight=1e-2, sparsity_radius=1.5, sparsity_length=0.05, weight_decay_mult=0.25)
        orig_uniform = jr.uniform
        for N, NF in SIZES:
            model = RM.NerfModel(num_coarse_samples=N, num_fine_samples=NF, use_viewdirs=False, sh_deg=sh_deg,
                                 sg_dim=-1, near=2.0, far=6.0, noise_std=None, net_depth=8, net_width=256,
                                 net_depth_condition=1, net_width_condition=128, net_activation=nn.relu, skip_layer=4,
                                 num_rgb_channels=48, num_sigma_channels=1, white_bkgd=True, min_deg_point=0,
                                 max_deg_point=10, deg_view=4, lindisp=False, rgb_activation=nn.sigmoid,
                                 sigma_activation=nn.relu, legacy_posenc_order=False)
            t_rand = rs.uniform(size=(B, N)).astype(np.float32)
            u_f = rs.uniform(size=(B, NF)).astype(np.float32)
            # every key carries the injected draws, told apart by shape ([B,N] jitter, [B,NF] inverse-CDF uniforms,
            # [NSP,3] sparsity points)
            table = {tuple(t_rand.shape): t_rand, tuple(u_f.shape): u_f, tuple(sp01.shape): sp01}

            def uniform(key, shape, dtype=np.float32, minval=0.0, maxval=1.0):
                base = table[tuple(shape)]
                return (base * np.float32(maxval - minval) + np.float32(minval)).astype(np.float32)
            jr.uniform = RT.random.uniform = MU.random.uniform = uniform
            tag_n = f"{N}_{NF}"
            out[f"t_rand_{tag_n}"], out[f"u_{tag_n}"] = t_rand, u_f
            for tag, rnd in (("det", False), ("rand", True)):
                ret = model.apply(variables, jax_stub.Key(seed=2), jax_stub.Key(seed=3), RU.Rays(o, d, v), rnd)
                for lvl, (c, di, ac) in zip(("coarse", "fine"), ret):
                    out[f"call_{tag_n}_{tag}_{lvl}_rgb"] = np.asarray(c)
                    out[f"call_{tag_n}_{tag}_{lvl}_disp"] = np.asarray(di)
                    out[f"call_{tag_n}_{tag}_{lvl}_acc"] = np.asarray(ac)
            if (N, NF) == LOSS_SIZE:
                @dataclasses.dataclass
                class Opt:
                    target: dict
                    def apply_gradient(self, grad, learning_rate=None):
                        return self
                state = RU.TrainState(optimizer=Opt(variables))
                _, stats, _ = RT.train_step(model, jax_stub.Key(seed=1), state,
                                            {"rays": RU.Rays(o, d, v), "pixels": px}, 5e-4)
                out.update(loss=np.float32(stats.loss), psnr=np.float32(stats.psnr), loss_c=np.float32(stats.loss_c),
                           psnr_c=np.float32(stats.psnr_c), loss_sp=np.float32(stats.loss_sp),
                           weight_l2=np.float32(stats.weight_l2))
        jr.uniform = orig_uniform
    finally:
        jax_stub.uninstall(names)
        for k in [k for k in sys.modules if k.startswith("nerf_sh")]:
            sys.modules.pop(k, None)
    assert all(np.asarray(a).dtype != np.float64 for a in out.values() if isinstance(a, np.ndarray))
    np.savez_compressed(os.path.join(HERE, "ref_long_rays.npz"), **out)
    print("ref_long_rays.npz", {k: float(out[k]) for k in ("loss", "loss_c", "loss_sp", "weight_l2", "psnr")})


if __name__ == "__main__":
    torch.manual_seed(20200823)
    torch.set_num_threads(8)
    gen_ref_long_rays()

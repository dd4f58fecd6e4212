"""CPU oracle for NeRF-SH models with a trunk activation other than relu.  TEST INFRASTRUCTURE ONLY.

The reference's flag net_activation (nerf_sh/nerf/models.py:362; torch twin octree/nerf/models.py:265) selects the
activation applied after every trunk layer (nerf_sh/nerf/model_utils.py:69).  This module restates the parts of
oracle/nerf_sh_oracle.py that apply it (the MLP and everything above it: eval_points_raw, one rendering level,
NerfModel.__call__, loss_fn and its gradient) with the activation as a parameter, and reuses that module's other stages
(posenc, SH, sampling, compositing) unchanged.  With net_activation="relu" every function here reproduces its
nerf_sh_oracle counterpart bit for bit.  Pinned against the reference by tests/golden/ref_net_activation.npz
(tests/golden/make_golden_net_activation.py).
"""
import math

import numpy as np
import torch

from oracle import nerf_sh_oracle as O

# by flax name (nn.relu, nn.elu, nn.softplus, nn.tanh).  softplus is max(x, 0) + log1p(exp(-|x|)): jax.nn.softplus's
# logaddexp(x, 0), without torch.nn.functional.softplus's linear threshold.
NET_ACTIVATIONS = {
    "relu": torch.relu,
    "elu": torch.nn.functional.elu,
    "softplus": lambda x: torch.clamp_min(x, 0.0) + torch.log1p(torch.exp(-x.abs())),
    "tanh": torch.tanh,
}


def activation(name):
    """the activation of a net_activation flag value, matched case-insensitively (the octree side names torch's
    classes: ReLU, ELU, Softplus, Tanh)"""
    return NET_ACTIVATIONS[str(name).lower()]


def mlp(params, enc, net_activation="relu"):
    """nerf_sh_oracle.mlp with the trunk activation as a parameter (model_utils.MLP.__call__, condition=None)."""
    act = activation(net_activation)
    shape = enc.shape[:-1]
    x = enc.reshape(-1, enc.shape[-1])
    inputs = x
    for i in range(O.NET_DEPTH):
        w, b = params[i]
        x = act(O._dense(x, w, b))
        if i % O.SKIP_LAYER == 0 and i > 0:
            x = torch.cat([x, inputs], dim=-1)
    raw_sigma = O._dense(x, params[8][0], params[8][1])
    raw_rgb = O._dense(x, params[9][0], params[9][1])
    return raw_rgb.reshape(*shape, -1), raw_sigma.reshape(*shape, 1)


def eval_points_raw(params, points, net_activation="relu"):
    """NerfModel.eval_points_raw without viewdirs (nerf_sh/nerf/models.py:143-181)."""
    return mlp(params, O.posenc(points), net_activation)


def render_level(params, sh_deg, z_vals, samples, rays, white_bkgd, sigma_noise=None, net_activation="relu"):
    """nerf_sh_oracle.render_level with the trunk activation."""
    origins, directions, viewdirs = rays
    raw_rgb, raw_sigma = mlp(params, O.posenc(samples), net_activation)
    raw_sigma = O.add_gaussian_noise(raw_sigma, sigma_noise)
    if sh_deg >= 0:
        K = (sh_deg + 1) ** 2
        raw_rgb = O.eval_sh(sh_deg, raw_rgb.reshape(*raw_rgb.shape[:-1], -1, K), viewdirs[:, None])
    rgb = torch.sigmoid(raw_rgb)
    sigma = torch.relu(raw_sigma)
    comp_rgb, disp, acc, weights = O.volumetric_rendering(rgb, sigma, z_vals, directions, white_bkgd)
    return (comp_rgb, disp, acc), weights, (rgb, sigma)


def nerf_forward(params_c, params_f, sh_deg, rays, num_coarse, num_fine, near, far, white_bkgd=True,
                 t_rand=None, u=None, lindisp=False, return_aux=False, z_fine=None, sigma_noise=None,
                 net_activation="relu"):
    """nerf_sh_oracle.nerf_forward (NerfModel.__call__) with the trunk activation."""
    origins, directions, viewdirs = rays
    z_vals, samples = O.sample_along_rays(origins, directions, num_coarse, near, far, t_rand, lindisp)
    noise_c, noise_f = sigma_noise if sigma_noise is not None else (None, None)
    out_c, weights, aux_c = render_level(params_c, sh_deg, z_vals, samples, rays, white_bkgd, noise_c, net_activation)
    ret = [out_c]
    aux = {"z_coarse": z_vals, "weights_coarse": weights, "rgbs_coarse": aux_c}
    if num_fine > 0:
        z_mid = 0.5 * (z_vals[..., 1:] + z_vals[..., :-1])
        if z_fine is not None:
            z_vals, samples = z_fine, O.cast_rays(z_fine, origins, directions)
        else:
            z_vals, samples = O.sample_pdf(z_mid, weights[..., 1:-1], origins, directions, z_vals, num_fine, u)
        out_f, weights_f, aux_f = render_level(params_f, sh_deg, z_vals, samples, rays, white_bkgd, noise_f,
                                               net_activation)
        ret.append(out_f)
        aux.update({"z_fine": z_vals, "weights_fine": weights_f, "rgbs_fine": aux_f})
    return (ret, aux) if return_aux else ret


def loss_fn(params_c, params_f, sh_deg, rays, pixels, cfg, t_rand=None, u=None, sp_points=None, z_fine=None,
            sigma_noise=None, net_activation="relu"):
    """nerf_sh_oracle.loss_fn (train_step.loss_fn) with the trunk activation; the sparsity points' raw sigma comes
    from the same trunk."""
    ret, aux = nerf_forward(params_c, params_f, sh_deg, rays, cfg["num_coarse_samples"],
                            cfg["num_fine_samples"], cfg["near"], cfg["far"], cfg["white_bkgd"], t_rand, u,
                            return_aux=True, z_fine=z_fine, sigma_noise=sigma_noise, net_activation=net_activation)
    if cfg.get("sparsity_weight", 0.0) > 0.0 and sp_points is not None:
        mlp_sp = params_f if cfg["num_fine_samples"] > 0 else params_c
        _, sp_sigma = eval_points_raw(mlp_sp, sp_points, net_activation)
        sp_sigma = torch.relu(sp_sigma)
        loss_sp = cfg["sparsity_weight"] * (1.0 - torch.exp(-cfg["sparsity_length"] * sp_sigma).mean())
    else:
        loss_sp = torch.zeros((), dtype=pixels.dtype)
    rgb = ret[-1][0]
    loss = ((rgb - pixels[..., :3]) ** 2).mean()
    psnr = -10.0 * torch.log(loss) / math.log(10.0)
    if len(ret) > 1:
        loss_c = ((ret[0][0] - pixels[..., :3]) ** 2).mean()
        psnr_c = -10.0 * torch.log(loss_c) / math.log(10.0)
    else:
        loss_c = torch.zeros((), dtype=pixels.dtype)
        psnr_c = torch.zeros((), dtype=pixels.dtype)
    all_p = [t for ps in (params_c, params_f) for wb in ps for t in wb]
    weight_l2 = sum((t ** 2).sum() for t in all_p) / sum(t.numel() for t in all_p)
    total = loss + loss_c + loss_sp + cfg.get("weight_decay_mult", 0.0) * weight_l2
    stats = dict(loss=loss, psnr=psnr, loss_c=loss_c, loss_sp=loss_sp, psnr_c=psnr_c, weight_l2=weight_l2)
    stats["_z_fine"] = aux.get("z_fine")
    return total, stats


def loss_and_grads(flat_c, flat_f, sh_deg, rays, pixels, cfg, t_rand=None, u=None, sp_points=None,
                   dtype=torch.float32, z_fine=None, sigma_noise=None, net_activation="relu"):
    """nerf_sh_oracle.loss_and_grads (jax.value_and_grad(loss_fn) via torch autograd) with the trunk activation."""
    fc = torch.tensor(np.asarray(flat_c), dtype=dtype, requires_grad=True)
    ff = torch.tensor(np.asarray(flat_f), dtype=dtype, requires_grad=True)
    cast = lambda a: None if a is None else torch.as_tensor(np.asarray(a)).to(dtype)
    rays_t = tuple(cast(r) for r in rays)
    total, stats = loss_fn(O.unflatten(fc, sh_deg), O.unflatten(ff, sh_deg), sh_deg, rays_t, cast(pixels),
                           cfg, cast(t_rand), cast(u), cast(sp_points), cast(z_fine),
                           None if sigma_noise is None else tuple(cast(a) for a in sigma_noise), net_activation)
    total.backward()
    zf = stats.pop("_z_fine")
    stats = {k: float(v.detach()) for k, v in stats.items()}
    stats["_z_fine"] = None if zf is None else zf.detach().numpy()
    gc = fc.grad.numpy() if fc.grad is not None else np.zeros_like(np.asarray(flat_c))
    gf = ff.grad.numpy() if ff.grad is not None else np.zeros_like(np.asarray(flat_f))
    return stats, gc, gf

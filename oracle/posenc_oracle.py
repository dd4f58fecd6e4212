"""CPU oracle for NeRF-SH models with a non-default point encoder.  TEST INFRASTRUCTURE ONLY.

The reference's flags min_deg_point, max_deg_point and legacy_posenc_order (nerf_sh/nerf/utils.py:119-124,155-159)
select posenc(x, min_deg, max_deg, legacy_posenc_order) (nerf_sh/nerf/model_utils.py:145-173; torch twin
octree/nerf/model_utils.py:161-190) and, through its width W = 3 + 6 (max_deg - min_deg), the shapes of Dense_0
[W, 256] and Dense_5 [256 + W, 256].  This module restates the parts of oracle/nerf_sh_oracle.py that depend on the
encoder with the descriptor pe = (min_deg, max_deg, legacy) as a parameter, and reuses that module's encoder-free
stages (MLP, SH, sampling, compositing) unchanged.  With pe = (0, 10, False) every function here reproduces its
nerf_sh_oracle counterpart bit for bit.  Pinned against the reference by tests/golden/ref_posenc.npz
(tests/golden/make_golden_posenc.py).
"""
import math

import numpy as np
import torch

from oracle import nerf_sh_oracle as O

DEFAULT = (0, 10, False)


def width(pe=DEFAULT):
    """W = 3 + 6 (max_deg - min_deg) (octree/nerf/models.py:182)."""
    return 3 + 6 * (int(pe[1]) - int(pe[0]))


def posenc(x, min_deg=0, max_deg=10, legacy=False):
    """model_utils.posenc (nerf_sh/nerf/model_utils.py:145-173) in the tensor's dtype, both feature orders."""
    if min_deg == max_deg:
        return x
    scales = torch.tensor([2 ** i for i in range(min_deg, max_deg)], dtype=x.dtype)
    xb = x[..., None, :] * scales[:, None]                                    # [..., L, 3]
    if legacy:
        four_feat = torch.sin(torch.stack([xb, xb + 0.5 * math.pi], -2)).reshape(list(x.shape[:-1]) + [-1])
    else:
        xb = xb.reshape(list(x.shape[:-1]) + [-1])
        four_feat = torch.sin(torch.cat([xb, xb + 0.5 * math.pi], dim=-1))
    return torch.cat([x, four_feat], dim=-1)


def encode(x, pe=DEFAULT):
    return posenc(x, int(pe[0]), int(pe[1]), bool(pe[2]))


def feature_index(pe=DEFAULT):
    """[(kind, j, c)] of the W features in order: kind 'x' (j = None), 'sin' or 'cos' of 2^j x_c."""
    mn, mx, legacy = int(pe[0]), int(pe[1]), bool(pe[2])
    out = [("x", None, c) for c in range(3)]
    if mn == mx:
        return out
    degs = range(mn, mx)
    if legacy:
        for j in degs:
            out += [("sin", j, c) for c in range(3)] + [("cos", j, c) for c in range(3)]
    else:
        out += [("sin", j, c) for j in degs for c in range(3)] + [("cos", j, c) for j in degs for c in range(3)]
    return out


def layer_dims(sh_deg, pe=DEFAULT):
    """(in, out) of Dense_0..Dense_9 (nerf_sh/nerf/model_utils.py:60-93) for encoder width W."""
    W = width(pe)
    return [(W if i == 0 else (O.NET_WIDTH + W if i == 5 else cin), cout)
            for i, (cin, cout) in enumerate(O.layer_dims(sh_deg))]


def param_count(sh_deg, pe=DEFAULT):
    return sum(i * o + o for i, o in layer_dims(sh_deg, pe))


def init_flat_params(sh_deg, seed, bias_scale=0.0, pe=DEFAULT):
    """nerf_sh_oracle.init_flat_params with the fan-in of Dense_0 / Dense_5 following W."""
    rs = np.random.RandomState(seed)
    parts = []
    for cin, cout in layer_dims(sh_deg, pe):
        a = math.sqrt(6.0 / (cin + cout))
        parts.append(rs.uniform(-a, a, size=(cin, cout)).astype(np.float32).reshape(-1))
        parts.append((rs.uniform(-1, 1, size=(cout,)) * bias_scale).astype(np.float32))
    return np.concatenate(parts)


def unflatten(flat, sh_deg, pe=DEFAULT):
    flat = torch.as_tensor(flat)
    out, off = [], 0
    for cin, cout in layer_dims(sh_deg, pe):
        w = flat[off:off + cin * cout].reshape(cin, cout)
        off += cin * cout
        out.append((w, flat[off:off + cout]))
        off += cout
    assert off == flat.numel()
    return out


def permute_rows(flat, sh_deg, pe_from, pe_to):
    """The same network for another feature order: Dense_0's rows and Dense_5's posenc rows moved so that a model
    with encoder pe_to computes what `flat` computes with pe_from (same degrees, any order)."""
    assert (pe_from[0], pe_from[1]) == (pe_to[0], pe_to[1])
    src = {f: i for i, f in enumerate(feature_index(pe_from))}
    perm = np.array([src[f] for f in feature_index(pe_to)])
    params = [(w.clone(), b.clone()) for w, b in unflatten(torch.from_numpy(np.asarray(flat)).clone(), sh_deg, pe_from)]
    params[0] = (params[0][0][perm], params[0][1])
    w5 = params[5][0]
    params[5] = (torch.cat([w5[:O.NET_WIDTH], w5[O.NET_WIDTH:][perm]]), params[5][1])
    return torch.cat([t.reshape(-1) for wb in params for t in wb]).numpy()


def eval_points_raw(params, points, pe=DEFAULT):
    """NerfModel.eval_points_raw without viewdirs (nerf_sh/nerf/models.py:143-181)."""
    return O.mlp(params, encode(points, pe))


def render_level(params, sh_deg, z_vals, samples, rays, white_bkgd, pe=DEFAULT):
    """nerf_sh_oracle.render_level with the model's encoder."""
    _, _, viewdirs = rays
    raw_rgb, raw_sigma = O.mlp(params, encode(samples, pe))
    if sh_deg >= 0:
        K = (sh_deg + 1) ** 2
        raw_rgb = O.eval_sh(sh_deg, raw_rgb.reshape(*raw_rgb.shape[:-1], -1, K), viewdirs[:, None])
    rgb = torch.sigmoid(raw_rgb)
    sigma = torch.relu(raw_sigma)
    comp_rgb, disp, acc, weights = O.volumetric_rendering(rgb, sigma, z_vals, rays[1], white_bkgd)
    return (comp_rgb, disp, acc), weights, (rgb, sigma)


def nerf_forward(params_c, params_f, sh_deg, rays, num_coarse, num_fine, near, far, white_bkgd=True, t_rand=None,
                 u=None, z_fine=None, pe=DEFAULT):
    """NerfModel.__call__ (nerf_sh/nerf/models.py:216-348) with the model's encoder: [(rgb, disp, acc) per level]."""
    origins, directions, _ = rays
    z_vals, samples = O.sample_along_rays(origins, directions, num_coarse, near, far, t_rand)
    out_c, weights, _ = render_level(params_c, sh_deg, z_vals, samples, rays, white_bkgd, pe)
    ret = [out_c]
    if num_fine > 0:
        if z_fine is not None:
            z_vals, samples = z_fine, O.cast_rays(z_fine, origins, directions)
        else:
            z_mid = 0.5 * (z_vals[..., 1:] + z_vals[..., :-1])
            z_vals, samples = O.sample_pdf(z_mid, weights[..., 1:-1], origins, directions, z_vals, num_fine, u)
        out_f, _, _ = render_level(params_f, sh_deg, z_vals, samples, rays, white_bkgd, pe)
        ret.append(out_f)
    return ret


def loss_and_grads(flat_c, flat_f, sh_deg, rays, pixels, cfg, t_rand=None, u=None, sp_points=None, z_fine=None,
                   dtype=torch.float64, pe=DEFAULT):
    """jax.value_and_grad(train_step.loss_fn) (nerf_sh/train.py:68-116) with the model's encoder, as
    nerf_sh_oracle.loss_and_grads: -> (stats, grad_c, grad_f) as numpy.  The weight-decay denominator is the
    parameter count of both MLPs, which follows W."""
    fc = torch.tensor(np.asarray(flat_c), dtype=dtype, requires_grad=True)
    ff = torch.tensor(np.asarray(flat_f), dtype=dtype, requires_grad=True)
    cast = lambda a: None if a is None else torch.as_tensor(np.asarray(a)).to(dtype)
    rays_t = tuple(cast(r) for r in rays)
    px = cast(pixels)
    pc, pf = unflatten(fc, sh_deg, pe), unflatten(ff, sh_deg, pe)
    ret = nerf_forward(pc, pf, sh_deg, rays_t, cfg["num_coarse_samples"], cfg["num_fine_samples"], cfg["near"],
                       cfg["far"], cfg["white_bkgd"], cast(t_rand), cast(u), cast(z_fine), pe)
    sw = cfg.get("sparsity_weight", 0.0)
    if sw > 0.0 and sp_points is not None:
        _, sp_sigma = eval_points_raw(pf if cfg["num_fine_samples"] > 0 else pc, cast(sp_points), pe)
        loss_sp = sw * (1.0 - torch.exp(-cfg["sparsity_length"] * torch.relu(sp_sigma)).mean())
    else:
        loss_sp = torch.zeros((), dtype=dtype)
    loss = ((ret[-1][0] - px[..., :3]) ** 2).mean()
    loss_c = ((ret[0][0] - px[..., :3]) ** 2).mean() if len(ret) > 1 else torch.zeros((), dtype=dtype)
    all_p = [t for ps in (pc, pf) for wb in ps for t in wb]
    weight_l2 = sum((t ** 2).sum() for t in all_p) / sum(t.numel() for t in all_p)
    total = loss + loss_c + loss_sp + cfg.get("weight_decay_mult", 0.0) * weight_l2
    total.backward()
    stats = {k: float(v.detach()) for k, v in (("loss", loss), ("loss_c", loss_c), ("loss_sp", loss_sp),
                                                 ("weight_l2", weight_l2))}
    return stats, fc.grad.numpy(), ff.grad.numpy()

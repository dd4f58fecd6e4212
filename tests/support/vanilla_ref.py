"""fp64 restatement of the reference's NerfModel with use_viewdirs (nerf_sh/nerf/models.py:143-214,216-348,
model_utils.py:30-94) for the vanilla render tests: the vanilla MLP of oracle/projection_oracle.py (pinned to the
executed reference by tests/golden/ref_projection.npz) with the flag net_activation after every trunk layer and after
the condition layer (model_utils.py:90), evaluated with one view direction per point, and both levels of the render
through nerf_sh_oracle's per-ray stages.  In the dtype of the inputs."""
import numpy as np
import torch

from oracle import nerf_sh_oracle as O
from oracle import posenc_oracle as PO
from oracle.net_activation_oracle import activation
from oracle.projection_oracle import _t, init_params

U = 2.0 ** -24          # fp32 unit roundoff
C_BRANCH = 512          # fp32 accumulation: 256 + 128 + 3 sums in sequence, activation ulps (kernels.h) included
RGB_TOL = 1e-3          # test_render.test_nerf_forward_vs_oracle: fp16, same sample positions, max-abs


def golden_layers(seed, deg_view, legacy, sigma_scale, sigma_shift):
    """the weights of a case of tests/golden/ref_vanilla.npz: {"MLP_0", "MLP_1"} from projection_oracle.init_params
    (seeds seed, seed + 1) with the Dense_8 kernel scaled by sigma_scale and sigma_shift added to its bias"""
    pe = (0, 10, bool(legacy))
    mlps = {"MLP_0": init_params(seed, pe, deg_view), "MLP_1": init_params(seed + 1, pe, deg_view)}
    for layers in mlps.values():
        layers[8] = ((layers[8][0] * np.float32(sigma_scale)).astype(np.float32),
                     (layers[8][1] + np.float32(sigma_shift)).astype(np.float32))
    return mlps


def trunk(layers, points, pe=PO.DEFAULT, act="relu"):
    """(h7 [N, 256], raw sigma [N, 1]) of points [N, 3]; projection_oracle.trunk with the activation as a flag"""
    dt = points.dtype
    f = activation(act)
    enc = PO.encode(points, pe)
    x = enc
    for i in range(8):
        x = f(x @ _t(layers[i][0], dt) + _t(layers[i][1], dt))
        if i == 4:
            x = torch.cat([x, enc], dim=-1)
    return x, x @ _t(layers[8][0], dt) + _t(layers[8][1], dt)


def view_branch(layers, h7, viewdirs, pe=PO.DEFAULT, deg_view=4, act="relu"):
    """raw rgb [N, 3] of the view branch from h7 [N, 256] and one view direction per row, viewdirs [N, 3]"""
    dt = h7.dtype
    bott = h7 @ _t(layers[9][0], dt) + _t(layers[9][1], dt)
    x = torch.cat([bott, PO.posenc(viewdirs, 0, deg_view, bool(pe[2]))], dim=-1)
    z = activation(act)(x @ _t(layers[10][0], dt) + _t(layers[10][1], dt))
    return z @ _t(layers[11][0], dt) + _t(layers[11][1], dt)


def eval_points_paired(layers, points, viewdirs, pe=PO.DEFAULT, deg_view=4, act="relu"):
    """eval_points_raw(points [N, 3], viewdirs [N, 3]) with one direction per point: (raw_rgb [N, 3], raw_sigma [N, 1])"""
    h, sigma = trunk(layers, points, pe, act)
    return view_branch(layers, h, viewdirs, pe, deg_view, act), sigma


def _render_level(layers, z_vals, rays, white_bkgd, pe, deg_view, act, sigma_act, noise):
    origins, directions, viewdirs = rays
    B, N = z_vals.shape
    samples = O.cast_rays(z_vals, origins, directions).reshape(-1, 3)
    vd = viewdirs[:, None, :].expand(B, N, 3).reshape(-1, 3)
    raw_rgb, raw_sigma = eval_points_paired(layers, samples, vd, pe, deg_view, act)
    raw_sigma = O.add_gaussian_noise(raw_sigma.reshape(B, N, 1), noise)
    sigma = activation(sigma_act)(raw_sigma)
    rgb = torch.sigmoid(raw_rgb.reshape(B, N, 3))
    comp_rgb, disp, acc, weights = O.volumetric_rendering(rgb, sigma, z_vals, directions, white_bkgd)
    return (comp_rgb, disp, acc), weights


def render_rays(layers_c, layers_f, rays, num_coarse, num_fine, near, far, white_bkgd=True, t_rand=None, u=None,
                z_fine=None, lindisp=False, pe=PO.DEFAULT, deg_view=4, act="relu", sigma_act="relu",
                sigma_noise=None):
    """NerfModel.__call__ with use_viewdirs: [(rgb, disp, acc)_coarse, (rgb, disp, acc)_fine], rays = (origins,
    directions, viewdirs) [B, 3] each; z_fine pins the fine level's depths as nerf_sh_oracle.nerf_forward does."""
    origins, directions, _ = rays
    z_vals, _ = O.sample_along_rays(origins, directions, num_coarse, near, far, t_rand, lindisp)
    noise_c, noise_f = sigma_noise if sigma_noise is not None else (None, None)
    out_c, weights = _render_level(layers_c, z_vals, rays, white_bkgd, pe, deg_view, act, sigma_act, noise_c)
    ret = [out_c]
    if num_fine > 0:
        if z_fine is None:
            z_mid = 0.5 * (z_vals[..., 1:] + z_vals[..., :-1])
            z_fine, _ = O.sample_pdf(z_mid, weights[..., 1:-1], origins, directions, z_vals, num_fine, u)
        out_f, _ = _render_level(layers_f, z_fine, rays, white_bkgd, pe, deg_view, act, sigma_act, noise_f)
        ret.append(out_f)
    return ret


# ---- device-side probes and scenes shared by the vanilla GPU tests -------------------------------------------------
def _mlps(seed, pe=PO.DEFAULT, deg_view=4, sigma_scale=8.0):
    mlps = {"MLP_0": init_params(seed, pe, deg_view), "MLP_1": init_params(seed + 1, pe, deg_view)}
    for layers in mlps.values():                      # a dense blob around the origin: partially opaque rays
        layers[8] = (layers[8][0] * sigma_scale, layers[8][1] + 2.0)
    return mlps


def _rays(R, seed):
    rs = np.random.RandomState(seed)
    o = rs.normal(size=(R, 3))
    o = (o / np.linalg.norm(o, axis=1, keepdims=True) * 4.0).astype(np.float32)
    d = (rs.uniform(-0.6, 0.6, (R, 3)) - o).astype(np.float32)
    d = (d / np.linalg.norm(d, axis=1, keepdims=True) * rs.uniform(0.8, 1.2, (R, 1))).astype(np.float32)
    v = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    return o, d, v


def _h7_fp16(mlps_layers, pts, pe, act_code):
    """the fp16 h7 the kernel's heads MMA reads, probed through pob_eval_points_raw: Dense_9 of a plain-SH25 blob of
    the same trunk set to unit columns, so raw rgb column j is h7[k] exactly (fp32 sums of one fp16 product)"""
    from plenoctree_b200 import ops
    K = 25
    trunk = [np.asarray(a, np.float32).reshape(-1) for k, b in mlps_layers[:9] for a in (k, b)]
    h = np.zeros((pts.shape[0], 256), np.float32)
    for k0 in range(0, 256, 3 * K):
        n = min(3 * K, 256 - k0)
        w9 = np.zeros((256, 3 * K), np.float32)
        w9[np.arange(k0, k0 + n), np.arange(n)] = 1.0
        flat = np.concatenate(trunk + [w9.reshape(-1), np.zeros(3 * K, np.float32)])
        blob = ops.pack_weights(torch.from_numpy(flat).cuda(), 4, posenc=pe)
        rgb, _ = ops.eval_points_raw(blob, 4, pts, posenc=pe, net_activation=act_code)
        h[:, k0:k0 + n] = rgb[:, :n].cpu().numpy()
    return h.astype(np.float64)


def _view_features(v32, deg_view, legacy):
    """posenc(v, 0, deg_view, legacy) in fp64 of the fp32 sine arguments the direction tables form: x 2^l is exact,
    the cosine's argument is the fp32 sum x 2^l + fp32(pi / 2)"""
    m, L = v32.shape[0], deg_view
    xb = (v32[:, None, :] * (2.0 ** np.arange(L, dtype=np.float32))[:, None]).astype(np.float32)     # [m, L, 3]
    xc = (xb + np.float32(0.5 * np.pi)).astype(np.float32)
    s, c = np.sin(xb.astype(np.float64)), np.sin(xc.astype(np.float64))
    four = np.stack([s, c], 2).reshape(m, -1) if legacy else np.concatenate([s.reshape(m, -1), c.reshape(m, -1)], 1)
    return np.concatenate([v32.astype(np.float64), four], 1)

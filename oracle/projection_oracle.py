"""CPU oracle for the SH projection of a vanilla NeRF (use_viewdirs) in octree extraction.  TEST INFRASTRUCTURE ONLY.

Restates the reference's vanilla MLP (octree/nerf/model_utils.py:112-158: trunk Dense_0..7 with the skip after
layer 4, Dense_8 raw sigma, Dense_9 bottleneck without activation, Dense_10 on [bottleneck, posenc(viewdir, 0,
deg_view)] with relu, Dense_11 raw rgb), eval_points_raw(..., cross_broadcast=True) (octree/nerf/models.py:211-252)
and ProjectFunctionNeRF (octree/nerf/sh_proj.py:273-306) at given (theta, phi), in the dtype of the inputs.
A vanilla parameter set is [(kernel [in, out], bias [out]) x 12] (plenoctree_b200.nerf.checkpoints' layout).
Pinned against the reference by tests/golden/ref_projection.npz (tests/golden/make_golden_projection.py).
"""
import math

import numpy as np
import torch

from oracle import nerf_sh_oracle as O
from oracle import posenc_oracle as PO


def layer_dims(pe=PO.DEFAULT, deg_view=4):
    W = PO.width(pe)
    dims = [(W if i == 0 else (256 + W if i == 5 else 256), 256) for i in range(8)]
    return dims + [(256, 1), (256, 256), (256 + 3 + 6 * deg_view, 128), (128, 3)]


def init_params(seed, pe=PO.DEFAULT, deg_view=4, bias_scale=0.05):
    """glorot-uniform kernels and uniform(-bias_scale, bias_scale) biases from numpy RandomState(seed)"""
    rs = np.random.RandomState(seed)
    out = []
    for cin, cout in layer_dims(pe, deg_view):
        a = math.sqrt(6.0 / (cin + cout))
        out.append((rs.uniform(-a, a, size=(cin, cout)).astype(np.float32),
                    rs.uniform(-bias_scale, bias_scale, size=cout).astype(np.float32)))
    return out


def _t(a, dtype):
    return torch.as_tensor(np.asarray(a)).to(dtype)


def trunk(layers, points, pe=PO.DEFAULT):
    """(h7 [B, 256], raw sigma [B, 1]) of points [B, 3]"""
    dt = points.dtype
    enc = PO.encode(points, pe)
    x = enc
    for i in range(8):
        x = torch.relu(x @ _t(layers[i][0], dt) + _t(layers[i][1], dt))
        if i == 4:
            x = torch.cat([x, enc], dim=-1)
    return x, x @ _t(layers[8][0], dt) + _t(layers[8][1], dt)


def eval_points_raw(layers, points, viewdirs, pe=PO.DEFAULT, deg_view=4):
    """eval_points_raw(points [B, 3], viewdirs [M, 3], cross_broadcast=True) -> (raw_rgb [B, M, 3], raw_sigma [B, 1])"""
    dt = points.dtype
    h, sigma = trunk(layers, points, pe)
    bott = h @ _t(layers[9][0], dt) + _t(layers[9][1], dt)
    venc = PO.posenc(viewdirs, 0, deg_view, bool(pe[2]))
    B, M = bott.shape[0], venc.shape[0]
    x = torch.cat([bott[:, None, :].expand(B, M, -1), venc[None].expand(B, M, -1)], dim=-1)
    z = torch.relu(x @ _t(layers[10][0], dt) + _t(layers[10][1], dt))
    return z @ _t(layers[11][0], dt) + _t(layers[11][1], dt), sigma


def spher2cart(theta, phi):
    r = torch.sin(theta)
    return torch.stack([r * torch.cos(phi), r * torch.sin(phi), torch.cos(theta)], dim=-1)


def project(layers, points, dirs, sh_deg, pe=PO.DEFAULT, deg_view=4):
    """ProjectFunctionNeRF over the directions dirs [D, 3]: (coeffs [B, 3, K], raw sigma [B, 1])"""
    raw_rgb, sigma = eval_points_raw(layers, points, dirs, pe, deg_view)
    Y = O.sh_basis(sh_deg, dirs)
    return torch.einsum("bsc,sk->bck", raw_rgb, Y) * (4.0 * math.pi / dirs.shape[0]), sigma


def a_p(layers, points, pe=PO.DEFAULT):
    """a_p = W10_b (W9 h7 + b9) + b10 [B, 128] of the split view branch"""
    dt = points.dtype
    h, _ = trunk(layers, points, pe)
    bott = h @ _t(layers[9][0], dt) + _t(layers[9][1], dt)
    return bott @ _t(layers[10][0][:256], dt) + _t(layers[10][1], dt)


def leaf_rows(layers, points, dirs, sh_deg, pe=PO.DEFAULT, deg_view=4):
    """step2's leaf rows for points [n, S, 3] that all use dirs [D, 3]: mean over S of [coeff (c K + k), sigma]"""
    n, S, _ = points.shape
    coeffs, sigma = project(layers, points.reshape(-1, 3), dirs, sh_deg, pe, deg_view)
    rows = torch.cat([coeffs.reshape(n * S, -1), sigma], dim=-1)
    return rows.reshape(n, S, -1).mean(dim=1)

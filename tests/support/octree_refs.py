"""fp64 references of the octree march, shaded from a visit list, and their budgets."""
import numpy as np

from oracle import octree_oracle as OO
from tests.support.octree_scenes import STOP, f64


U24 = 2.0 ** -24

# ---- bars (measured on an H100 80 GB HBM3 at a 400 W power limit; the largest value over all trees in brackets)
# render: |rgb - fp64| per ray and channel in units of 2^-24 * (1 + n_hits + sum_j tau_j + sum_j w_j sum_k (|b_k| + 1) |c_jk|)
# (the 1 is the background composite; a basis value's rounding is absolute, not relative, since its polynomial cancels)
RGB_ALLOW = 1.6             # [0.80]
# backward: per element, in units of 2^-24 * sum over the contributing visits reaching it of |term| x its rounding depth
# (see bwd64); the fp32 oracle's own backward measures [0.65] in this unit on the CPU
GRAD_ALLOW = 1.4            # [0.70]
# training pass: the same unit, the upstream gradient carrying the forward's error (RGB_ALLOW x its unit), which
# dominates the unit: the kernel's own image sets the clamp mask and g, so its rgb error does not reach the gradient
TRAIN_ALLOW = 0.13          # [0.065]
# sum of squared errors (float per thread and CTA, double across CTAs): 2^-24 * sum (2 |diff| U + 16 diff^2)
SQ_ALLOW = 0.06             # [0.031]
STOP_MARGIN = 1e-4          # relative distance of the fp64 transmittance from stop_thresh for exact early-stop paths
SENSITIVITY = 10.0


def _sh64(K, d):
    """the SH basis of OO.sh_basis in fp64"""
    x, y, z = (np.asarray(d, dtype=f64)[:, a] for a in range(3))
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    C1, C2, C3, C4 = OO.SH_C1, OO.SH_C2, OO.SH_C3, OO.SH_C4
    b = [np.full_like(x, OO.SH_C0), -C1 * y, C1 * z, -C1 * x,
         C2[0] * xy, C2[1] * yz, C2[2] * (2.0 * zz - xx - yy), C2[3] * xz, C2[4] * (xx - yy),
         C3[0] * y * (3 * xx - yy), C3[1] * xy * z, C3[2] * y * (4 * zz - xx - yy), C3[3] * z * (2 * zz - 3 * xx - 3 * yy),
         C3[4] * x * (4 * zz - xx - yy), C3[5] * z * (xx - yy), C3[6] * x * (xx - 3 * yy),
         C4[0] * xy * (xx - yy), C4[1] * yz * (3 * xx - yy), C4[2] * xy * (7 * zz - 1), C4[3] * yz * (7 * zz - 3),
         C4[4] * (zz * (35 * zz - 30) + 3), C4[5] * xz * (7 * zz - 3), C4[6] * (xx - yy) * (7 * zz - 1),
         C4[7] * xz * (xx - 3 * yy), C4[8] * (xx * (xx - 3 * yy) - yy * (3 * xx - yy))]
    return np.stack(b[:K], axis=1)


def _layout(otree):
    rgba = str(otree.data_format).upper().startswith("RGBA")
    return rgba, (1 if rgba else (otree.data_dim - 1) // 3)


def _rows(otree, leaf):
    return otree.data.reshape(-1, otree.data_dim)[leaf]


def _first(ray, R):
    return np.searchsorted(ray, np.arange(R))


def _excl(x, ray, first):
    """exclusive prefix sum of x within each ray's (contiguous) segment"""
    c = np.cumsum(x) - x
    return c - c[first[ray]] if x.size else c


def fwd64(otree, vis, v, bg, sigma_thresh=0.0, rows=None, delta_t=None):
    """fp64 forward of the march in `vis` on the fp32 tree data -> dict (rgb [R,3], U [R,3] the bar unit / 2^-24, and
    the per-visit quantities the backward needs)"""
    rgba, K = _layout(otree)
    ray, R = vis["ray"], vis["miss"].shape[0]
    rows = (_rows(otree, vis["leaf"]) if rows is None else rows).astype(f64)
    dt = (vis["delta_t"] if delta_t is None else delta_t).astype(f64)
    ds = vis["delta_scale"].astype(f64)[ray]
    basis = np.ones((R, 1)) if rgba else _sh64(K, v)
    b = basis[ray]
    babs = np.abs(basis) + (0.0 if rgba else 1.0)   # a basis value's rounding is absolute (its polynomial cancels)
    sig = rows[:, -1]
    hit = sig > sigma_thresh
    tau = np.where(hit, dt * ds * sig, 0.0)
    first = _first(ray, R)
    S = _excl(tau, ray, first)
    T = np.exp(-S)
    w = np.where(hit, T * -np.expm1(-tau), 0.0)
    coef = rows[:, :3 * K].reshape(-1, 3, K)
    pre = np.einsum("vk,vck->vc", b, coef)
    apre = np.einsum("vk,vck->vc", babs[ray], np.abs(coef))
    col = 1.0 / (1.0 + np.exp(-pre))
    out = np.stack([np.bincount(ray, w * col[:, c], minlength=R) for c in range(3)], axis=1)
    tend = np.exp(-np.bincount(ray, tau, minlength=R))
    stopped = vis["stopped"] if sigma_thresh > 0 else np.zeros(R, dtype=bool)
    scale = 1.0 / np.where(stopped, 1.0 - tend, 1.0)[:, None]          # early termination renormalises
    out = np.where(stopped[:, None], out * scale, out + tend[:, None] * bg)
    nh = np.bincount(ray, hit, minlength=R)
    U = (1.0 + nh + np.bincount(ray, tau, minlength=R))[:, None] + np.stack(
        [np.bincount(ray, w * apre[:, c], minlength=R) for c in range(3)], axis=1)
    U = U * scale
    return dict(rgb=out, U=U, hit=hit, tau=tau, S=S, T=T, w=w, col=col, apre=apre, basis=basis, babs=babs, tend=tend,
                dt=dt, ds=ds,
                nh_before=_excl(hit.astype(f64), ray, first), first=first)


def bwd64(otree, vis, f, g, gerr, bg):
    """fp64 backward (both svox passes) from the forward `f` of the same visit list and the upstream gradient g [R,3].
    -> (touched packed leaves [U], gradient [U, D], bar unit / 2^-24 [U, D]); gerr [R,3] bounds the error of g in the
    forward's unit."""
    rgba, K = _layout(otree)
    D = otree.data_dim
    ray, R = vis["ray"], vis["miss"].shape[0]
    h = np.nonzero(f["hit"])[0]
    r = ray[h]
    s, w, T, tau, S = f["col"][h], f["w"][h], f["T"][h], f["tau"][h], f["S"][h]
    gh, gabs = g[r], (np.abs(g) + gerr)[r]
    b = f["basis"][r]
    tnext = T * np.exp(-tau)
    # pass 1: colour
    coef = w[:, None] * s * (1.0 - s) * gh                                       # [H,3]
    dcol = (coef[:, :, None] * b[:, None, :]).reshape(-1, 3 * K)
    depth = 1.0 + f["nh_before"][h] + S
    # the weight carries T_j's rounding (1 - att cancels when tau is small), s (1 - s) the absolute rounding of 1 - s
    ds1 = s * (1.0 - s)
    acol = ((gabs * (ds1 * T[:, None] + w[:, None] * (ds1 * (depth[:, None] + f["apre"][h]) + 1.0)))[:, :, None]
            * f["babs"][r][:, None, :]).reshape(-1, 3 * K)
    # pass 2: density, accum_j = sum_{i > j} w_i total_i + T_end * bg * sum(g)
    total = (s * gh).sum(axis=1)
    wt = np.zeros(ray.shape[0])
    wt[h] = f["w"][h] * total
    after = np.bincount(ray, wt, minlength=R)[ray] - (_excl(wt, ray, f["first"]) + wt)
    accum = after[h] + f["tend"][r] * bg * g[r].sum(axis=1)
    dsig = f["dt"][h] * f["ds"][h] * (total * tnext - accum)
    asig = f["dt"][h] * f["ds"][h] * ((s * gabs).sum(axis=1) * tnext * (depth + tau) + (gabs * f["U"][r]).sum(axis=1))
    uniq, inv = np.unique(vis["leaf"][h], return_inverse=True)
    grad = np.zeros((uniq.size, D))
    unit = np.zeros((uniq.size, D))
    for c in range(3 * K):
        grad[:, c] = np.bincount(inv, dcol[:, c], minlength=uniq.size)
        unit[:, c] = np.bincount(inv, acol[:, c], minlength=uniq.size)
    grad[:, D - 1] = np.bincount(inv, dsig, minlength=uniq.size)
    unit[:, D - 1] = np.bincount(inv, asig, minlength=uniq.size)
    return uniq, grad, unit


def _safe_fast_rays(f, vis):
    """rays whose fp64 transmittance after every contributing visit stays STOP_MARGIN (relative) away from STOP"""
    after = f["T"] * np.exp(-f["tau"])
    near = f["hit"] & (np.abs(after - STOP) <= STOP_MARGIN * STOP)
    return np.bincount(vis["ray"], near, minlength=vis["miss"].shape[0]) == 0


def _check_grad(name, otree, got, uniq, grad, unit, allow, tag):
    """kernel gradient got [n*N^3, D] against the fp64 one: exact 0 off the touched leaves, per-element bar on them"""
    rest = np.ones(got.shape[0], dtype=bool)
    rest[uniq] = False
    n_nonzero_rest = int((got[rest] != 0).sum())
    assert n_nonzero_rest == 0, (name, tag, n_nonzero_rest)
    e = np.abs(got[uniq].astype(f64) - grad) / (U24 * np.maximum(unit, 1e-300))
    e[(unit == 0) & (got[uniq] == 0)] = 0.0
    worst = float(e.max())
    assert worst <= allow, (name, tag, worst, np.unravel_index(np.argmax(e), e.shape))
    return worst

"""The octree march at production depth (csrc/octree.cu): exact leaf paths and fp64 bounds for the renderer, its
backward, the fused training pass and SGD.

tests/test_octree.py holds these kernels to the float32 oracle on trees of depth 2-4 with N = 2, sigma >= 0 and a white
background, at bars scaled to the largest value.  Here the trees are what production meets and what the kernel's
special paths need: a depth-8 SH16 shell (the path cache of the N = 2 walk resumes at its cap, level CACHED - 1 = 7), a
depth-9 shell, N = 3 and N = 4 trees (query_leaf and its cube scaling), and a chain refined to depths 12, 16 and 26 with
rays starting on the chain (the plain walk below level 22).  Every cell holds data, coarse leaves included, about 20 % of
sigma is negative, the boxes are anisotropic and off-centre, rays start outside and inside the box, and a camera with an
axis-aligned c2w sits on cell-face planes (zero direction components, positions exactly on boundaries).

- Path: the kernel rounds every position and step like the float32 oracle, so its `visits` / `hits` counters must equal
  the oracle's march, per launch and per single-ray launch.  With fast=True (early termination) that holds on rays
  whose fp64 transmittance never comes within STOP_MARGIN of stop_thresh.
- Values: fp64 references shade the oracle's visit list (leaf, fp32 delta_t, fp32 delta_scale) with fp64 basis,
  sigmoid, exp, transmittance and background.  Bars are per ray (render) and per element (gradients), in units of the
  rounding each one accumulates, and were measured on an H100.  Elements no contributing visit reaches must be 0.
- Sensitivity: three one-visit perturbations of the fp64 reference (sibling cell's data, parent's cell size, one SH term
  dropped) each move a checked value by more than SENSITIVITY x its bar.
"""
import functools
import json
import os
import time

import numpy as np
import pytest

from oracle import octree_oracle as OO
from tests.test_octree import OUT, assert_device_tree_build_matches, to_device_tree

f32, f64 = np.float32, np.float64
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
# SGD: data - lr * g is one fused, correctly rounded operation, within 2^-24 * (|data| + |lr g|) of fp64  [0.998]
STOP_MARGIN = 1e-4          # relative distance of the fp64 transmittance from stop_thresh for exact early-stop paths
SENSITIVITY = 10.0
STOP = 1e-2                 # svox fast=True: sigma_thresh = stop_thresh = 1e-2
N_SINGLE = 32               # single-ray launches per ray set


def _record(name, payload):
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, "parity_octree_march.json")
    data = json.load(open(path)) if os.path.exists(path) else {}
    data[name] = payload
    json.dump(data, open(path, "w"), indent=1)


# ---------------------------------------------------------------------------------------------------------
# trees
# ---------------------------------------------------------------------------------------------------------
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


def _shell_voxels(N, L, region, rs, R=0.32):
    """voxel centres (unit cube) of the level-L cells that a sphere of radius R about the box centre passes through,
    restricted to the directions in `region` (octant signs; 0 = both)"""
    reso = N ** (L + 1)
    n = int(8 * 4 * np.pi * R * R * reso * reso / 2 ** sum(1 for s in region if s))
    v = rs.normal(size=(n, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    for a, s in enumerate(region):
        if s:
            v[:, a] = s * np.abs(v[:, a])
    idx = np.unique(np.floor((0.5 + R * v) * reso).astype(np.int64), axis=0)
    return (idx + 0.5) / reso


def _to_world(otree, unit):
    return ((np.asarray(unit, dtype=f64) - otree.offset) / otree.invradius).astype(f32)


def _fill(otree, rs, tau_cell=0.6, cap_level=12):
    """every cell of every node: coefficients N(0,1); sigma sized to an optical depth of up to tau_cell across the
    cell (capped at level cap_level), 20 % of it negated"""
    n, N = otree.n_internal, otree.N
    otree.data[:n] = rs.normal(0, 1, size=otree.data[:n].shape).astype(f32)
    lvl = np.minimum(otree.parent_depth[:n, 1], cap_level).astype(f64)
    cell = (N ** -(lvl + 1.0)) / otree.invradius.astype(f64).mean()          # world cell size
    sig = rs.uniform(0, tau_cell, size=otree.data[:n, ..., -1].shape) / cell[:, None, None, None]
    sig[rs.rand(*sig.shape) < 0.2] *= -1.0
    otree.data[:n, ..., -1] = sig.astype(f32)


SPECS = {
    # name: N, depth, format, radius, center, shell region (None = chain tree)
    "n2_d8_sh16": (2, 8, "SH16", (1.1, 0.8, 1.4), (0.15, -0.1, 0.05), (1, 1, 0)),
    "n2_d9_sh4": (2, 9, "SH4", (0.9, 1.3, 1.05), (-0.2, 0.1, 0.3), (1, -1, 1)),
    "n3_d4_sh16": (3, 4, "SH16", (1.2, 1.0, 0.85), (0.05, 0.2, -0.1), (-1, 1, 1)),
    "n4_d3_sh9": (4, 3, "SH9", (0.8, 1.25, 1.0), (0.1, 0.0, 0.25), (1, 1, -1)),
    "chain_d26_rgba": (2, 26, "RGBA", (1.3, 0.95, 1.15), (-0.05, 0.12, 0.0), None),
}
CHAIN = ((0.3712345, 0.6184021, 0.4421377, 12), (0.6931472, 0.2718282, 0.5772157, 16),
         (0.0137035, 0.0291172, 0.0083145, 26))


def _build(name):
    """-> oracle tree, list of refine() point sets (world), world points of occupied cells"""
    N, L, fmt, radius, center, region = SPECS[name]
    K = 1 if fmt == "RGBA" else int(fmt[2:])
    D = 4 if fmt == "RGBA" else 3 * K + 1
    rs = np.random.RandomState(sum(map(ord, name)))
    otree = OO.N3Tree(N=N, data_dim=D, depth_limit=L, init_reserve=1024, geom_resize_fact=1.5, radius=radius,
                      center=center, data_format=fmt)
    refines = []
    if region is None:
        for *p, depth in CHAIN:
            w = _to_world(otree, [p])
            while True:
                node, _, _, _ = otree.query(w)
                if otree.parent_depth[node[0], 1] >= depth:
                    break
                otree.refine_at(w)
                refines.append(w)
        pts = _to_world(otree, [p[:3] for p in CHAIN])
    else:
        pts = _to_world(otree, _shell_voxels(N, L, region, rs))
        for _ in range(L):
            otree.refine_at(pts)
            refines.append(pts)
        if name.startswith("n3") and otree.n_internal % 2 == 0:
            # an odd node count makes the SGD length n_internal * 27 * 49 odd: the kernel's scalar tail runs
            extra = _to_world(otree, [[0.5 - 0.4 * s if s else 0.02 for s in region]])
            assert otree.refine_at(extra)
            refines.append(extra)
    _fill(otree, rs)
    return otree, refines, pts


def _unit_rand(rs, n):
    v = rs.normal(size=(n, 3))
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(f32)


def _face_world(otree, a, target):
    """a world coordinate whose tree coordinate (offset + invradius * x, rounded like the kernel) is exactly target"""
    off, inv = otree.offset[a], otree.invradius[a]
    x = f32((f64(target) - off) / inv)
    for _ in range(4096):
        t = f32(off + f32(inv * x))
        if t == target:
            return x
        x = np.nextafter(x, f32(np.inf) if t < target else f32(-np.inf))
    raise AssertionError("no world coordinate maps onto the face plane")


def _cameras(otree):
    """two axis-aligned cameras whose origins lie on cell-face planes in the two axes across the view direction:
    one outside the box looking down -z, one inside looking down -x"""
    N = otree.N
    faces = (f32(0.5), f32(0.25)) if N != 3 else (f32(1.0 / 3.0), f32(2.0 / 3.0))
    out = []
    for rot, axes, along in ((np.eye(3), (0, 1), (2, 1.35)), (np.array([[0, 0, 1], [1, 0, 0], [0, 1, 0]]), (1, 2), (0, 0.7))):
        c2w = np.eye(4, dtype=f32)
        c2w[:3, :3] = rot
        for a, t in zip(axes, faces):
            c2w[a, 3] = _face_world(otree, a, t)
        c2w[along[0], 3] = _to_world(otree, [[along[1]] * 3])[0, along[0]]
        out.append(c2w)
    return out


CAM_W, CAM_H, CAM_F = 24, 24, 16.0


def _ray_sets(name, otree, pts):
    """-> list of (set name, origins, dirs, step_size, background)"""
    rs = np.random.RandomState(7 + sum(map(ord, name)))
    rad = 0.5 / otree.invradius.astype(f64)
    cen = (0.5 - otree.offset.astype(f64)) / otree.invradius.astype(f64)
    cams = [OO.persp_rays(c, CAM_W, CAM_H, CAM_F) for c in _cameras(otree)]
    if SPECS[name][5] is None:
        o = np.repeat(pts, 96, axis=0)
        return [("chain_points", o, _unit_rand(rs, o.shape[0]), 2e-6, 0.25),
                ("camera_out", cams[0][0], cams[0][1], 2e-6, 1.0),
                ("camera_in", cams[1][0], cams[1][1], 2e-6, 0.25)]
    n = 384
    o = (cen + 3.0 * rad.max() * _unit_rand(rs, n)).astype(f32)
    tgt = pts[rs.randint(0, pts.shape[0], n)] + (rs.uniform(-0.02, 0.02, (n, 3)) * rad).astype(f32)
    d = (tgt - o) / np.linalg.norm(tgt - o, axis=1, keepdims=True)
    d[: n // 8] *= -1.0                                                   # some miss the box
    inside = np.concatenate([pts[rs.randint(0, pts.shape[0], n // 2)],      # in occupied cells
                             (cen + rad * rs.uniform(-0.95, 0.95, (n - n // 2, 3)))]).astype(f32)
    return [("orbit", o, d.astype(f32), 1e-5, 1.0),
            ("inside", inside, _unit_rand(rs, n), 1e-3, 0.25),
            ("camera_out", cams[0][0], cams[0][1], 1e-5, 0.25),
            ("camera_in", cams[1][0], cams[1][1], 1e-3, 1.0)]


@functools.lru_cache(maxsize=None)
def world(name):
    t0 = time.time()
    otree, refines, pts = _build(name)
    sets = []
    for sname, o, d, step, bg in _ray_sets(name, otree, pts):
        v = d.copy()
        vis = OO.march_visits(otree, o, d, v, step, bg)
        visf = OO.march_visits(otree, o, d, v, step, bg, STOP, STOP)
        sets.append(dict(name=sname, o=o, d=d, v=v, step=step, bg=bg, vis=vis, visf=visf))
    return dict(otree=otree, refines=refines, pts=pts, sets=sets, build_s=time.time() - t0)


@functools.lru_cache(maxsize=None)
def device_tree(name):
    return to_device_tree(world(name)["otree"])


# ---------------------------------------------------------------------------------------------------------
# references shaded from a visit list
# ---------------------------------------------------------------------------------------------------------
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


# ---------------------------------------------------------------------------------------------------------
# CPU: the visit list is the march
# ---------------------------------------------------------------------------------------------------------
def shade_f32(otree, vis, v, bg, sigma_thresh, stop_thresh):
    """float32 shading of a visit list in volume_render's operation order, visit by visit -> rgb, visits, hits"""
    rgba, K = _layout(otree)
    ray, R = vis["ray"], vis["miss"].shape[0]
    basis = None if rgba else OO.sh_basis(K, v)
    first = _first(ray, R)
    k = np.arange(ray.size) - first[ray]
    out = np.zeros((R, 3), dtype=f32)
    light = np.ones(R, dtype=f32)
    for step in range(int(k.max()) + 1 if k.size else 0):
        sel = np.nonzero(k == step)[0]
        a = ray[sel]
        rows = _rows(otree, vis["leaf"][sel])
        sigma, dt, ds = rows[:, -1], vis["delta_t"][sel], vis["delta_scale"][a]
        hh = sigma > f32(sigma_thresh)
        a, rows, sigma, dt, ds = a[hh], rows[hh], sigma[hh], dt[hh], ds[hh]
        att = np.exp(-dt * ds * sigma).astype(f32)
        weight = (light[a] * (f32(1.0) - att)).astype(f32)
        if rgba:
            pre = rows[:, :3]
        else:
            pre = np.zeros((a.size, 3), dtype=f32)
            for c in range(3):
                for j in range(K):
                    pre[:, c] = (pre[:, c] + basis[a, j] * rows[:, c * K + j]).astype(f32)
        out[a] = (out[a] + weight[:, None] * OO._sigmoid(pre)).astype(f32)
        light[a] = (light[a] * att).astype(f32)
    st = vis["stopped"]
    out[st] = (out[st] * (f32(1.0) / (f32(1.0) - light[st]))[:, None]).astype(f32)
    rest = ~st & ~vis["miss"]
    out[rest] = (out[rest] + light[rest][:, None] * f32(bg)).astype(f32)
    out[vis["miss"]] = f32(bg)
    hits = np.bincount(ray, _rows(otree, vis["leaf"])[:, -1] > f32(sigma_thresh), minlength=R)
    return out, np.bincount(ray, minlength=R), hits


@pytest.mark.parametrize("N,fmt", [(2, "SH9"), (3, "RGBA"), (2, "RGBA")])
def test_visit_list_reproduces_volume_render(N, fmt):
    rs = np.random.RandomState(3 + N)
    K = 1 if fmt == "RGBA" else int(fmt[2:])
    otree = OO.N3Tree(N=N, data_dim=4 if fmt == "RGBA" else 3 * K + 1, depth_limit=3, radius=(1.2, 0.9, 1.0),
                      center=(0.1, -0.1, 0.05), data_format=fmt)
    pts = _to_world(otree, rs.uniform(0.1, 0.9, size=(60, 3)))
    for _ in range(3):
        otree.refine_at(pts)
    _fill(otree, rs, tau_cell=1.5)
    o = np.concatenate([(3.0 * _unit_rand(rs, 96)), pts[:32]]).astype(f32)
    d = np.concatenate([_unit_rand(rs, 96) * -1.0, _unit_rand(rs, 32)]).astype(f32)
    d[:64] = ((pts[rs.randint(0, 60, 64)] - o[:64]) / np.linalg.norm(pts[rs.randint(0, 60, 64)] - o[:64], axis=1,
                                                                        keepdims=True)).astype(f32)
    for th in (0.0, STOP):
        vis = OO.march_visits(otree, o, d, d, 1e-3, 0.25, th, th)
        rgb, visits, hits = OO.volume_render(otree, o, d, d, 1e-3, 0.25, th, th, return_steps=True)
        got, gv, gh = shade_f32(otree, vis, d, 0.25, th, th)
        assert np.array_equal(got.view(np.int32), rgb.view(np.int32))
        assert np.array_equal(gv, visits) and np.array_equal(gh, hits)
        assert np.array_equal(vis["visits"], visits) and np.array_equal(vis["rgb"].view(np.int32), rgb.view(np.int32))
        assert (hits > 0).sum() > 40 and (visits > hits).any()
        if th:
            assert vis["stopped"].sum() > 5
        # the fp64 shading of the same list agrees to float32 precision
        f = fwd64(otree, vis, d, 0.25, th)
        assert np.abs(f["rgb"] - rgb).max() < 1e-4


# ---------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------
NAMES = list(SPECS)


def _renderer(name, step, bg):
    from plenoctree_b200.octree import VolumeRenderer
    return VolumeRenderer(device_tree(name), step_size=step, background_brightness=bg)


def _forward(r, o, d, v, fast, counters=None):
    import torch
    from plenoctree_b200.octree import Rays
    with torch.no_grad():
        return r.forward(Rays(torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(v)), fast=fast,
                         counters=counters)


def _safe_fast_rays(f, vis):
    """rays whose fp64 transmittance after every contributing visit stays STOP_MARGIN (relative) away from STOP"""
    after = f["T"] * np.exp(-f["tau"])
    near = f["hit"] & (np.abs(after - STOP) <= STOP_MARGIN * STOP)
    return np.bincount(vis["ray"], near, minlength=vis["miss"].shape[0]) == 0


def _guards(otree, vis, v, step, bg, f, unit):
    """the largest rgb change each one-visit perturbation of the fp64 reference makes, in the bar's unit"""
    rgba, K = _layout(otree)
    N, D = otree.N, otree.data_dim
    j = int(np.argmax(f["w"]))                       # the visit with the largest weight
    rows = _rows(otree, vis["leaf"]).astype(f64)
    out = {}
    leaf = int(vis["leaf"][j])
    sib = leaf - 1 if leaf % N else leaf + 1           # neighbour along the last axis, same node
    p = rows.copy()
    p[j] = otree.data.reshape(-1, D)[sib]
    out["sibling_data"] = p, None
    dt = vis["delta_t"].astype(f64).copy()
    dt[j] = (dt[j] - step) * N + step                 # exit length measured in the parent's cell
    out["parent_cell_size"] = None, dt
    p = rows.copy()
    p[j, [c * K + K - 1 for c in range(3)]] = 0.0
    out["sh_term_dropped"] = p, None
    r = vis["ray"][j]
    ratios = {}
    for k, (pr, pdt) in out.items():
        g = fwd64(otree, vis, v, bg, rows=pr, delta_t=pdt)["rgb"]
        ratios[k] = float((np.abs(g[r] - f["rgb"][r]) / unit[r]).max())
    return ratios


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_render_exact_path_and_values(name):
    import torch
    W = world(name)
    otree = W["otree"]
    rs = np.random.RandomState(11)
    rec = {"build_s": W["build_s"], "nodes": int(otree.n_internal), "max_depth": int(otree.max_depth)}
    worst = {False: 0.0, True: 0.0}
    guards = {}
    for S in W["sets"]:
        o, d, v, step, bg = S["o"], S["d"], S["v"], S["step"], S["bg"]
        r = _renderer(name, step, bg)
        R = o.shape[0]
        for fast in (False, True):
            vis = S["visf"] if fast else S["vis"]
            f = fwd64(otree, vis, v, bg, STOP if fast else 0.0)
            cnt = torch.zeros(2, dtype=torch.int64, device="cuda")
            got = _forward(r, o, d, v, fast, cnt).cpu().numpy().astype(f64)
            cnt = cnt.cpu().numpy()
            err = np.abs(got - f["rgb"]) / (U24 * f["U"])
            if fast:
                safe = _safe_fast_rays(f, vis)
                rec[f"{S['name']}_fast_rays_excluded"] = int((~safe).sum())
                # the exact path on the safe rays: each ray's counts, from per-ray launches of the safe rays
                err = err[safe]
                assert safe.sum() > 0.9 * R
            else:
                assert cnt[0] == vis["visits"].sum() and cnt[1] == vis["hits"].sum(), (S["name"], cnt)
                rec[f"{S['name']}_visits"] = int(cnt[0])
                rec[f"{S['name']}_hits"] = int(cnt[1])
                g = _guards(otree, vis, v, step, bg, f, U24 * f["U"])
                for k, x in g.items():
                    guards[f"{S['name']}_{k}"] = x
            worst[fast] = max(worst[fast], float(err.max()))
            assert err.max() <= RGB_ALLOW, (S["name"], fast, float(err.max()))
            # single-ray launches: each ray's own visit / hit counts
            pick = rs.choice(np.nonzero(safe)[0] if fast else np.arange(R), N_SINGLE // 2, replace=False)
            cs = torch.zeros((pick.size, 2), dtype=torch.int64, device="cuda")
            for i, p in enumerate(pick):
                _forward(r, o[p:p + 1], d[p:p + 1], v[p:p + 1], fast, cs[i])
            cs = cs.cpu().numpy()
            assert np.array_equal(cs[:, 0], vis["visits"][pick]) and np.array_equal(cs[:, 1], vis["hits"][pick]), \
                (S["name"], fast)
        assert vis["hits"].sum() > 0
    rec.update(rgb_err_units={"fast_false": worst[False], "fast_true": worst[True]}, rgb_allow=RGB_ALLOW,
               guard_units=guards, guard_ratio_to_bar={k: x / RGB_ALLOW for k, x in guards.items()})
    _record(f"render_{name}", rec)
    for k, x in guards.items():
        assert x > SENSITIVITY * RGB_ALLOW, (k, x / RGB_ALLOW)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_render_persp_bit_identities(name):
    """the camera ray is built with the same rounded operations as OO.persp_rays, so render_persp equals forward on
    those rays bit for bit, and the training pass renders the same image as render_persp(fast=False)"""
    import torch
    W = world(name)
    otree = W["otree"]
    for c2w in _cameras(otree):
        o, d, v = OO.persp_rays(c2w, CAM_W, CAM_H, CAM_F)
        r = _renderer(name, 1e-3, 0.25)
        with torch.no_grad():
            for fast in (False, True):
                a = r.render_persp(c2w, width=CAM_W, height=CAM_H, fx=CAM_F, fast=fast).cpu().numpy()
                b = _forward(r, o, d, v, fast).cpu().numpy()
                assert np.array_equal(a.reshape(-1, 3).view(np.int32), b.view(np.int32))
            ref = r.render_persp(c2w, width=CAM_W, height=CAM_H, fx=CAM_F).cpu().numpy()
            gt = torch.from_numpy(np.random.RandomState(2).uniform(0, 1, (CAM_H, CAM_W, 3)).astype(f32))
            device_tree(name).grad = None
            _, img = r.train_persp(c2w, gt, CAM_W, CAM_H, CAM_F, want_image=True)
            device_tree(name).grad = None
            assert np.array_equal(img.cpu().numpy().view(np.int32), ref.view(np.int32))
        assert (d == 0).sum() >= 2 * CAM_W          # a pixel row and a pixel column run along cell-face planes


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


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_backward_matches_fp64(name):
    import torch
    from plenoctree_b200.octree import Rays
    W = world(name)
    otree = W["otree"]
    tree = device_tree(name)
    rec = {}
    for S in W["sets"][:2]:
        o, d, v, step, bg = S["o"], S["d"], S["v"], S["step"], S["bg"]
        g = np.random.RandomState(5).normal(size=(o.shape[0], 3)).astype(f32)
        f = fwd64(otree, S["vis"], v, bg)
        uniq, grad, unit = bwd64(otree, S["vis"], f, g.astype(f64), np.zeros_like(f["U"]), bg)
        r = _renderer(name, step, bg)
        tree.data.requires_grad_(True)
        tree.data.grad = None
        rgb = r.forward(Rays(torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(v)))
        (rgb * torch.from_numpy(g).cuda()).sum().backward()
        got = tree.data.grad.reshape(-1, otree.data_dim)[: otree.n_internal * otree.N ** 3].cpu().numpy()
        tree.data.grad = None
        tree.data.requires_grad_(False)
        rec[S["name"]] = _check_grad(name, otree, got, uniq, grad, unit, GRAD_ALLOW, S["name"])
        # the march crossed leaves of negative sigma, whose rows _check_grad required to be exactly 0
        assert (_rows(otree, S["vis"]["leaf"])[:, -1] < 0).any()
    _record(f"backward_{name}", {"grad_err_units": rec, "grad_allow": GRAD_ALLOW})


def _train(name, c2w):
    import torch
    W = world(name)
    otree = W["otree"]
    tree = device_tree(name)
    step = W["sets"][2]["step"]
    o, d, v = OO.persp_rays(c2w, CAM_W, CAM_H, CAM_F)
    vis = OO.march_visits(otree, o, d, v, step, 1.0)
    gt = np.random.RandomState(4).uniform(0, 1, size=(CAM_H, CAM_W, 3)).astype(f32)
    r = _renderer(name, step, 1.0)
    tree.grad = None
    sq, img = r.train_persp(c2w, torch.from_numpy(gt), CAM_W, CAM_H, CAM_F, want_image=True)
    got = tree.grad_buffer().reshape(-1, otree.data_dim)[: otree.n_internal * otree.N ** 3].cpu().numpy()
    im = img.cpu().numpy().reshape(-1, 3).astype(f64)
    f = fwd64(otree, vis, v, 1.0)
    scale = f64(f32(1.0 / (CAM_H * CAM_W * 3)))
    gt = gt.reshape(-1, 3).astype(f64)
    inside = (im >= 0) & (im <= 1)                               # the kernel's own clamp decisions
    diff = np.clip(f["rgb"], 0, 1) - gt
    g = np.where(inside, scale * 2.0 * diff, 0.0)
    gerr = np.where(inside, 2.0 * scale * RGB_ALLOW * f["U"], 0.0)
    uniq, grad, unit = bwd64(otree, vis, f, g, gerr, 1.0)
    flips = int((inside != ((f["rgb"] >= 0) & (f["rgb"] <= 1))).sum())
    sq_unit = U24 * float((2 * np.abs(diff) * f["U"] + 16 * diff ** 2).sum())
    sq_err = abs(float(sq.item()) - float((diff ** 2).sum())) / sq_unit
    return otree, tree, got, uniq, grad, unit, flips, sq_err


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_train_pass_matches_fp64(name):
    rec = {}
    for i, c2w in enumerate(_cameras(world(name)["otree"])):
        otree, tree, got, uniq, grad, unit, flips, sq_err = _train(name, c2w)
        rec[f"camera{i}"] = {"grad_err_units": _check_grad(name, otree, got, uniq, grad, unit, TRAIN_ALLOW, "train"),
                             "clamp_decisions_differing_from_fp64": flips, "sq_err_units": sq_err}
        assert sq_err <= SQ_ALLOW, sq_err
        tree.grad = None
    _record(f"train_{name}", dict(rec, train_allow=TRAIN_ALLOW, sq_allow=SQ_ALLOW))


@pytest.mark.gpu
def test_sgd_odd_length_runs_the_tail():
    import torch
    name = "n3_d4_sh16"
    otree, tree, got, *_ = _train(name, _cameras(world(name)["otree"])[0])
    n = otree.n_internal * otree.N ** 3 * otree.data_dim
    assert n % 2 == 1
    g = tree.grad_buffer().reshape(-1)[:n]
    # the scalar tail (the last n % 4 elements) must see nonzero gradients
    g[n - n % 4:] = torch.tensor([0.5, -0.25, 0.125][: n % 4], device="cuda")
    grad = g.cpu().numpy().astype(f64)
    before = tree.data.reshape(-1)[:n].cpu().numpy()
    lr = f32(1e3)
    tree.sgd_step(float(lr))
    after = tree.data.reshape(-1)[:n].cpu().numpy()
    nz = grad != 0
    want = before.astype(f64) - f64(lr) * grad
    bound = U24 * (np.abs(before) + np.abs(f64(lr) * grad))
    assert (np.abs(after[nz] - want[nz]) <= bound[nz]).all()
    assert np.array_equal(after[~nz].view(np.int32), before[~nz].view(np.int32))
    assert float(tree.grad_buffer().abs().max()) == 0.0
    assert nz[n - n % 4:].all() and nz.sum() > 1000
    _record("sgd_n3", {"n": int(n), "nonzero": int(nz.sum()),
                       "max_err_units": float((np.abs(after[nz] - want[nz]) / bound[nz]).max())})


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n2_d9_sh4", "n3_d4_sh16", "n4_d3_sh9"])
def test_topology_query_and_sample(name):
    W = world(name)
    otree = W["otree"]
    N, L, fmt, radius, center, _ = SPECS[name]
    assert_device_tree_build_matches(otree, W["refines"], radius, center, np.random.RandomState(3), query_box=1.6)

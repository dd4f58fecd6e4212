"""Extraction's weight mask at production resolution (csrc/octree.cu `grid_weight_kernel`, behind
`pob_grid_weight_render` and `octree/extraction.py::calculate_grid_weights`): exact voxel paths and fp64 bounds.

`mask = max_weight >= weight_thresh` picks the voxels step 1 refines, so a wrong weight is a wrong tree topology that
nothing after it can see.  tests/test_octree.py holds the kernel to the float32 oracle on a 32^3 grid at 1e-5 absolute.
Here the grids are 96^3 (a reso that is not a power of two), 512^3 (init_grid_depth 8) and 1024^3 (4 GB: the byte
offset of a voxel passes 2^31), marched at the production step 1e-5, with an anisotropic, off-centre box.

- sigma is an integer hash of the flat voxel index, evaluated by the same integer / fp64 expression in torch on the
  device and in numpy on the host, so both sides hold the same float32 grid without a copy.  It is shaped like a
  scene: a solid body, a thin shell, empty space, 20 % of the occupied voxels negative or zero, a tail of shell voxels
  with tau > 90 per visit (the light underflows) and dust with tau ~ 1e-6 (1 - e^-tau is mostly rounding).
- Path: `OO.grid_march_visits` records the float32 march, which depends on the ray geometry alone.  The kernel's `hit`
  buffer must be the set of listed voxels with sigma > 0.  Past the visit where the fp64 transmittance falls below
  2^-100 (CUT) the kernel may stop earlier than the list (`__expf` flushes to 0 near tau = 87, numpy's exp keeps
  denormals to 103), so there only a prefix is required: every kernel hit is a listed hit, every listed hit before
  the cut is a kernel hit.
- Values: per voxel, `wmax` against the fp64 maximum over rays of T (1 - e^-tau), shaded from the list (fp32 delta_t
  and delta_scale; tau, exp, 1 - e^-tau and T in fp64), within WEIGHT_ALLOW units (see `shade64`).  Voxels no
  positive-sigma visit reaches are exactly 0.
- Mask: `wmax >= weight_thresh` equals the fp64 mask on every voxel farther than the bar from the threshold.
- Launch invariants (atomicMax is exact and order-free): camera chunking, camera order, a pre-filled `wmax`, mixed
  camera sizes under a larger tile grid, and the production launch (100 cameras at 800 x 800), bit for bit.
- Extraction at init_grid_depth 8: step 1 (the recomputed mask against fp64, the tree against the oracle's refinement
  of that mask) and step 2 (leaf order, chunking and per-chunk seeds; eval_cells_mean adds partial sums with atomics,
  so the cell means are held to a rerun within CELL_ALLOW units rather than bit for bit).
"""
import ctypes
import functools
import json
import os
import time

import numpy as np
import pytest

from oracle import octree_oracle as OO
from tests.test_octree import OUT, look_at_pose
from tests.test_octree_march import CAM_F, CAM_H, CAM_W, _cameras

f32, f64 = np.float32, np.float64
U24 = 2.0 ** -24

# ---- bars (measured on an H100 80 GB HBM3 at a 400 W power limit; the largest value in brackets)
# weight: |wmax - fp64| per voxel in units of max over the voxel's visits of
#   2^-24 * T_j * (att_j * (1 + tau_j) + (1 - att_j) * (1 + n_j + S_j))
# att_j = e^-tau_j, T_j = e^-S_j, S_j / n_j the optical depth / number of hits before visit j.  The first term is
# `__expf`'s error (2 + 1.17 |x| ulp) and the rounding of tau, both absolute in 1 - att; the second the rounding of
# 1 - att and of the weight, and the relative error `light` accumulates over the earlier visits.
WEIGHT_ALLOW = 4.0          # [2.03]
ORACLE_ALLOW = 2.0          # the float32 oracle (np.exp) in the same unit, on the CPU  [1.48]
CUT = 100.0 * np.log(2.0)   # S_j beyond this: T_j < 2^-100, the kernel may already have stopped
CELL_ALLOW = 8.0            # step 2 cell means against a rerun of eval_cells_mean  [3.98]
SENSITIVITY = 10.0
STEP = 1e-5                 # --renderer_step_size of the reference's configs (octree/config/syn_sh16.json)
WEIGHT_THRESH = 1e-3
N_SINGLE = 32
RADIUS = (1.3, 1.1, 1.45)
CENTER = (0.12, -0.08, 0.05)
FOCAL_800 = 1111.1111       # Blender: 0.5 * 800 / tan(0.5 * camera_angle_x 0.6911)
CAM_DIST = 4.031


def _record(name, payload):
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, "parity_grid_weights.json")
    data = json.load(open(path)) if os.path.exists(path) else {}
    data[name] = payload
    json.dump(data, open(path, "w"), indent=1)
    print(name, json.dumps(payload))


@functools.lru_cache(maxsize=None)
def geometry():
    t = OO.N3Tree(radius=RADIUS, center=CENTER)
    return t.offset.copy(), t.invradius.copy()


# ---------------------------------------------------------------------------------------------------------
# sigma: one integer / fp64 expression, evaluated by numpy (host) and torch (device)
# ---------------------------------------------------------------------------------------------------------
M32 = 0xFFFFFFFF
BODY = (0.47, 0.53, 0.5, 0.17)      # centre, radius (unit cube)
SHELL = 0.33


def _hash(i):
    """32-bit mix of an int64 array (numpy or torch); every product stays below 2^63"""
    h = (i * 0x2C1B3C6D + 0x297A2D39) & M32
    h = h ^ (h >> 15)
    h = (h * 0x5BD1E995) & M32
    h = h ^ (h >> 13)
    h = (h * 0x297A2D39) & M32
    return h ^ (h >> 16)


def _sigma_expr(idx, reso, where, to_f64):
    """sigma of flat voxels idx (int64) as float64: every operation is an exact integer one or a single IEEE fp64
    operation, so numpy and torch (one kernel per operation) produce the same bits"""
    h = _hash(idx)
    u1 = to_f64(h >> 16) / 65536.0
    u2 = to_f64(h & 0xFFFF) / 65536.0
    i, j, k = idx // (reso * reso), (idx // reso) % reso, idx % reso
    dx = (to_f64(i) + 0.5) / reso - BODY[0]
    dy = (to_f64(j) + 0.5) / reso - BODY[1]
    dz = (to_f64(k) + 0.5) / reso - BODY[2]
    r2 = dx * dx + dy * dy + dz * dz
    scale = reso / (RADIUS[0] + RADIUS[1] + RADIUS[2]) * 1.5     # tau across one cell -> sigma
    body = r2 < BODY[3] * BODY[3]
    shell = (r2 > (SHELL - 1.0 / reso) ** 2) & (r2 < (SHELL + 1.0 / reso) ** 2)
    tau = where(body, 0.02 + 2.5 * u1, 0.0)
    tau = where(shell, where(u2 < 0.06, 95.0 + 300.0 * u1, 0.3 + 1.5 * u1), tau)
    occ = body | shell
    tau = where(occ & (u2 >= 0.8) & (u2 < 0.9), -tau, tau)
    tau = where(occ & (u2 >= 0.9), 0.0, tau)
    tau = where(~occ & (u2 < 0.01), 1e-6 * (1.0 + u1), tau)
    return tau * scale


def sigma_host(idx, reso):
    idx = np.asarray(idx, dtype=np.int64)
    return _sigma_expr(idx, reso, np.where, lambda a: a.astype(f64)).astype(f32)


def sigma_device(reso, chunk=1 << 25):
    import torch
    n = reso ** 3
    out = torch.empty(n, dtype=torch.float32, device="cuda")
    for lo in range(0, n, chunk):
        idx = torch.arange(lo, min(n, lo + chunk), dtype=torch.int64, device="cuda")
        out[lo:lo + idx.numel()] = _sigma_expr(idx, reso, torch.where, lambda a: a.double()).float()
    return out


# ---------------------------------------------------------------------------------------------------------
# cameras
# ---------------------------------------------------------------------------------------------------------
def _aim(origin, target, fx=1e4):
    """c2w of a 1x1 camera (focal fx) whose one ray leaves origin towards target"""
    origin, target = np.asarray(origin, f64), np.asarray(target, f64)
    fwd = (target - origin) / np.linalg.norm(target - origin)
    up = np.array([0.0, 0.0, 1.0]) if abs(fwd[2]) < 0.9 else np.array([1.0, 0.0, 0.0])
    right = np.cross(fwd, up)
    right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    c2w = np.eye(4, dtype=f32)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, up, -fwd, origin
    return c2w


def _world(unit):
    off, inv = geometry()
    return ((np.asarray(unit, f64) - off) / inv).astype(f64)


def single_cams(seed):
    """N_SINGLE aimed 1x1 cameras: from outside at the body and the shell (some grazing), and from inside the box"""
    rs = np.random.RandomState(seed)
    out = []
    for n in range(N_SINGLE):
        if n < 20:
            v = rs.normal(size=3)
            o = np.asarray(CENTER) + CAM_DIST * v / np.linalg.norm(v)
            w = rs.normal(size=3)
            rad = BODY[3] if n % 2 else SHELL * rs.uniform(0.9, 1.02)
            tgt = _world(np.asarray(BODY[:3]) + rad * w / np.linalg.norm(w))
        else:
            o = _world(rs.uniform(0.05, 0.95, 3) if n % 3 else np.asarray(BODY[:3]) + 0.05 * rs.normal(size=3))
            tgt = o + rs.normal(size=3)
        out.append((_aim(o, tgt), 1, 1, 1e4))
    return out


def camera_group(reso):
    """the cameras of one mixed-size launch: production poses at reduced pixel counts (focal scaled), one camera
    inside the box, two axis-aligned cameras on voxel-face planes"""
    if reso >= 1024:
        prod = [(look_at_pose(100, CAM_DIST), 64, 48, FOCAL_800 * 64 / 800)]
    else:
        prod = [(look_at_pose(100 + s, CAM_DIST), 160, 120, FOCAL_800 * 160 / 800) for s in range(8)]
    inside = _aim(_world([0.62, 0.35, 0.44]), _world([0.3, 0.7, 0.55]))
    faces = OO.N3Tree(radius=RADIUS, center=CENTER)
    return prod + [(inside, 64, 48, 50.0)] + [(c, CAM_W, CAM_H, CAM_F) for c in _cameras(faces)]


def cam_rows(cams):
    rows = np.zeros((len(cams), 16), dtype=f32)
    for n, (c2w, W, H, f) in enumerate(cams):
        rows[n, :12] = np.asarray(c2w, f32)[:3, :4].reshape(12)
        rows[n, 12:] = (f, f, W, H)
    return rows


# ---------------------------------------------------------------------------------------------------------
# fp64 references shaded from a visit list
# ---------------------------------------------------------------------------------------------------------
def _first(vis):
    R = vis["miss"].shape[0]
    count = np.bincount(vis["ray"], minlength=R)
    return np.cumsum(count) - count, count


def _excl_cumsum(x, vis, first, count, chunk=2048):
    """per-ray exclusive prefix sums in march order, summed within each ray only (a global cumsum would carry the
    other rays' magnitude into every S)"""
    out = np.zeros_like(x)
    ray = vis["ray"]
    R = count.size
    for r0 in range(0, R, chunk):
        r1 = min(R, r0 + chunk)
        v0, v1 = first[r0], first[r1 - 1] + count[r1 - 1]
        if v1 == v0:
            continue
        rr = ray[v0:v1]
        kk = np.arange(v0, v1) - first[rr]
        P = np.zeros((r1 - r0, int(count[r0:r1].max())))
        P[rr - r0, kk] = x[v0:v1]
        out[v0:v1] = (np.cumsum(P, axis=1) - P)[rr - r0, kk]
    return out


def shade64(vis, sig, delta_t=None, delta_scale=None):
    """fp64 weights of every visit of `vis` over the float32 sigma of its voxels (sig [V]) -> dict of per-visit
    hit, w, unit (the bar unit / 2^-24) and pre (the fp64 transmittance before the visit is >= 2^-100)"""
    first, count = _first(vis)
    dt = (vis["delta_t"] if delta_t is None else delta_t).astype(f64)
    ds = (vis["delta_scale"] if delta_scale is None else delta_scale).astype(f64)[vis["ray"]]
    hit = sig > 0
    tau = np.where(hit, dt * ds * sig.astype(f64), 0.0)
    S = _excl_cumsum(tau, vis, first, count)
    n = _excl_cumsum(hit.astype(f64), vis, first, count)
    T = np.exp(-S)
    att = np.exp(-tau)
    om = -np.expm1(-tau)
    w = np.where(hit, T * om, 0.0)
    unit = np.where(hit, T * (att * (1.0 + tau) + om * (1.0 + n + S)), 0.0)
    return dict(hit=hit, w=w, unit=unit, pre=S <= CUT, tau=tau)


def per_voxel(vox, w, unit, pre):
    """per voxel over the given (hit) visits -> keys, max w over the visits before the cut, max w over all, the
    unit (max over all visits; a visit past the cut adds an absolute 2^-100 / 2^-24), any visit before the cut"""
    unit = unit + np.where(pre, 0.0, 2.0 ** -100 / U24)
    order = np.argsort(vox, kind="stable")
    v = vox[order]
    keys, start = np.unique(v, return_index=True)
    if keys.size == 0:
        z = np.zeros(0)
        return dict(keys=keys, lo=z, hi=z, unit=z, pre=np.zeros(0, bool))
    return dict(keys=keys, lo=np.maximum.reduceat(np.where(pre, w, 0.0)[order], start),
                hi=np.maximum.reduceat(w[order], start), unit=np.maximum.reduceat(unit[order], start),
                pre=np.maximum.reduceat(pre[order].astype(np.uint8), start).astype(bool))


def merge(parts):
    vox = np.concatenate([p["keys"] for p in parts])
    order = np.argsort(vox, kind="stable")
    keys, start = np.unique(vox[order], return_index=True)
    out = dict(keys=keys)
    for k in ("lo", "hi", "unit"):
        out[k] = np.maximum.reduceat(np.concatenate([p[k] for p in parts])[order], start) if keys.size else np.zeros(0)
    out["pre"] = (np.maximum.reduceat(np.concatenate([p["pre"] for p in parts]).astype(np.uint8)[order], start)
                  .astype(bool) if keys.size else np.zeros(0, bool))
    return out


def march(reso, cams, sig_fn=None):
    """oracle march + fp64 shading of every ray of the cameras -> per-voxel reference and path statistics
    (sig_fn: flat voxel indices -> float32 sigma; the hash grid by default)"""
    off, inv = geometry()
    parts, stats = [], dict(rays=0, visits=0, hit_visits=0, negative_sigma_visits=0, rays_cut=0)
    for c2w, W, H, f in cams:
        o, d, _ = OO.persp_rays(c2w, W, H, f)
        vis = OO.grid_march_visits(reso, o, d, off, inv, STEP)
        sig = sigma_host(vis["voxel"], reso) if sig_fn is None else sig_fn(vis["voxel"])
        s = shade64(vis, sig)
        h = s["hit"]
        parts.append(per_voxel(vis["voxel"][h], s["w"][h], s["unit"][h], s["pre"][h]))
        stats["rays"] += int(o.shape[0])
        stats["visits"] += int(vis["ray"].size)
        stats["hit_visits"] += int(h.sum())
        stats["negative_sigma_visits"] += int((sig < 0).sum())
        stats["rays_cut"] += int(np.unique(vis["ray"][h & ~s["pre"]]).size)
    stats["visits_per_ray"] = stats["visits"] / max(stats["rays"], 1)
    return merge(parts), stats


@functools.lru_cache(maxsize=None)
def reference(reso, what):
    t0 = time.time()
    if what == "group":
        ref, stats = march(reso, camera_group(reso))
        return dict(ref=ref, stats=dict(stats, oracle_s=time.time() - t0))
    singles = []
    for cam in single_cams(reso):
        ref, stats = march(reso, [cam])
        singles.append((cam, ref, stats))
    return singles


def weight_err(ref, keys_got, vals_got):
    """-> per-voxel error in units (0 inside [lo, hi]); keys_got must be a subset of ref['keys']"""
    pos = np.searchsorted(ref["keys"], keys_got)
    got = np.zeros(ref["keys"].size)
    got[pos] = vals_got
    err = np.maximum(ref["lo"] - got, got - ref["hi"])
    return np.maximum(err, 0.0) / (U24 * ref["unit"]), got


# ---------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------
def shade_f32(vis, sig, reso, sigma_thresh, stop_thresh):
    """float32 shading of a visit list in grid_weight_render's operation order, iteration by iteration"""
    first, count = _first(vis)
    ray = vis["ray"]
    R = count.size
    k = np.arange(ray.size) - first[ray]
    order = np.argsort(k, kind="stable")
    bounds = np.searchsorted(k[order], np.arange(int(k.max()) + 2 if k.size else 1))
    gw = np.zeros(reso ** 3, dtype=f32)
    light = np.ones(R, dtype=f32)
    stopped = np.zeros(R, dtype=bool)
    for it in range(bounds.size - 1):
        sel = order[bounds[it]:bounds[it + 1]]
        sel = sel[~stopped[ray[sel]]]
        s = sig[sel]
        h = s > f32(sigma_thresh)
        sel, s = sel[h], s[h]
        a = ray[sel]
        att = np.exp(-vis["delta_t"][sel] * vis["delta_scale"][a] * s).astype(f32)
        weight = (light[a] * (f32(1.0) - att)).astype(f32)
        light[a] = (light[a] * att).astype(f32)
        np.maximum.at(gw, vis["voxel"][sel], weight)
        stopped[a[light[a] <= f32(stop_thresh)]] = True
    return gw


def _rand_rays(rs, n, inside):
    off, inv = geometry()
    if inside:
        o = _world(rs.uniform(0.02, 0.98, (n, 3)))
    else:
        v = rs.normal(size=(n, 3))
        o = np.asarray(CENTER) + 3.5 * v / np.linalg.norm(v, axis=1, keepdims=True)
    tgt = _world(rs.uniform(0.1, 0.9, (n, 3)))
    d = tgt - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return o.astype(f32), d.astype(f32)


@pytest.mark.parametrize("sigma_thresh,stop_thresh", [(0.0, 0.0), (3.0, 0.0), (0.0, 1e-2), (1.5, 0.2)])
def test_visit_list_reproduces_grid_weight_render(sigma_thresh, stop_thresh):
    rs = np.random.RandomState(17)
    reso = 40
    off, inv = geometry()
    grid = sigma_host(np.arange(reso ** 3), reso).reshape(reso, reso, reso)
    grid = grid * f32(rs.uniform(0.5, 20.0))            # heavier so that some rays stop / underflow
    o1, d1 = _rand_rays(rs, 300, False)
    o2, d2 = _rand_rays(rs, 200, True)
    o, d = np.concatenate([o1, o2]), np.concatenate([d1, d2])
    d[:20] *= -1.0                                      # some miss the box
    for step in (1e-3, 2e-6):
        want = OO.grid_weight_render(grid, o, d, off, inv, step, sigma_thresh, stop_thresh)
        vis = OO.grid_march_visits(reso, o, d, off, inv, step)
        got = shade_f32(vis, grid.reshape(-1)[vis["voxel"]], reso, sigma_thresh, stop_thresh)
        assert np.array_equal(got.view(np.int32), want.reshape(-1).view(np.int32))
        assert (want > 0).sum() > 300 and vis["miss"].sum() >= 10
        # rays march in order and every visit lies inside the grid
        assert np.all(np.diff(vis["ray"]) >= 0) and vis["voxel"].min() >= 0 and vis["voxel"].max() < reso ** 3


def test_sigma_hash_is_scene_shaped():
    reso = 96
    idx = np.arange(reso ** 3)
    tau = sigma_host(idx, reso).astype(f64) / (reso / sum(RADIUS) * 1.5)
    c = (np.stack(np.unravel_index(idx, (reso,) * 3), axis=1) + 0.5) / reso - np.asarray(BODY[:3])
    r2 = (c * c).sum(axis=1)
    occ = (r2 < BODY[3] ** 2) | ((r2 > (SHELL - 1.0 / reso) ** 2) & (r2 < (SHELL + 1.0 / reso) ** 2))
    assert 0.01 < occ.mean() < 0.2                          # a body and a shell in mostly empty space
    assert 0.15 < (tau[occ] <= 0).mean() < 0.25             # negated or exactly 0
    assert (tau > 90).sum() > 100                           # the underflow tail
    assert ((tau > 0) & (tau < 3e-6)).sum() > 1000          # dust: 1 - e^-tau is mostly rounding
    assert (tau[~occ] == 0).mean() > 0.98


def test_unit_bounds_the_fp32_oracle():
    """the bar's unit, derived in shade64, bounds the float32 oracle (correctly rounded exp) voxel by voxel"""
    reso = 96
    off, inv = geometry()
    grid = sigma_host(np.arange(reso ** 3), reso).reshape(reso, reso, reso)
    cams = camera_group(reso)[:2] + camera_group(reso)[-3:]
    want = np.zeros_like(grid)
    for c2w, W, H, f in cams:
        o, d, _ = OO.persp_rays(c2w, W, H, f)
        OO.grid_weight_render(grid, o, d, off, inv, STEP, out=want)
    ref, stats = march(reso, cams)
    want = want.reshape(-1)
    nz = np.nonzero(want)[0]
    assert np.isin(nz, ref["keys"]).all()
    err, _ = weight_err(ref, nz, want[nz])
    worst = float(err.max())
    _record("fp32_oracle_96", dict(err_units=worst, allow=ORACLE_ALLOW, **stats))
    assert worst <= ORACLE_ALLOW, worst
    assert stats["rays_cut"] > 10 and stats["negative_sigma_visits"] > 1000


def guards(reso):
    """the largest change of a voxel's fp64 maximum, over the single rays, that each perturbation of one ray's
    reference makes, in units of the bar"""
    out = dict(neighbour_sigma=0.0, no_step_in_delta_t=0.0, no_delta_scale=0.0)
    off, inv = geometry()
    for c2w, W, H, f in single_cams(reso):
        o, d, _ = OO.persp_rays(c2w, W, H, f)
        vis = OO.grid_march_visits(reso, o, d, off, inv, STEP)
        if vis["ray"].size == 0:
            continue
        sig = sigma_host(vis["voxel"], reso)
        base = shade64(vis, sig)
        if not base["hit"].any():
            continue
        j = int(np.argmax(base["w"]))
        v = int(vis["voxel"][j])
        nb = v + 1 if v % reso != reso - 1 else v - 1
        sig2 = sig.copy()
        sig2[j] = sigma_host([nb], reso)[0]
        dt2 = vis["delta_t"].astype(f64).copy()
        dt2[j] -= STEP
        cases = dict(neighbour_sigma=shade64(vis, sig2), no_step_in_delta_t=shade64(vis, sig, delta_t=dt2),
                     no_delta_scale=shade64(vis, sig, delta_scale=np.ones(o.shape[0])))
        keys = np.unique(vis["voxel"])

        def dense(s):
            M = np.zeros(keys.size)
            U = np.zeros(keys.size)
            p = np.searchsorted(keys, vis["voxel"])
            np.maximum.at(M, p, s["w"])
            np.maximum.at(U, p, s["unit"])
            return M, U
        M0, U0 = dense(base)
        for k, s in cases.items():
            M1, U1 = dense(s)
            den = WEIGHT_ALLOW * U24 * np.maximum(U0, U1)
            ok = den > 0
            out[k] = max(out[k], float((np.abs(M1 - M0)[ok] / den[ok]).max()))
    return out


@pytest.mark.parametrize("reso", [96, 512])
def test_sensitivity_of_the_fp64_reference(reso):
    g = guards(reso)
    _record(f"guards_{reso}", dict(guard_ratio_to_bar=g, sensitivity=SENSITIVITY))
    for k, x in g.items():
        assert x > SENSITIVITY, (k, x)


# ---------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------
RESOS = [96, 512, 1024]


@functools.lru_cache(maxsize=1)
def device_sigma(reso):
    return sigma_device(reso)


def launch(reso, cams, wmax, hit, max_w=None, max_h=None, step=STEP):
    import torch
    from plenoctree_b200 import _lib
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    off, inv = geometry()
    rows = torch.from_numpy(cam_rows(cams)).cuda()
    o = _lib.OctreeOpts()
    o.step_size, o.background_brightness, o.sigma_thresh, o.stop_thresh = step, 1.0, 0.0, 0.0
    max_w = max(c[1] for c in cams) if max_w is None else max_w
    max_h = max(c[2] for c in cams) if max_h is None else max_h
    check(lib.pob_grid_weight_render(ptr(device_sigma(reso)), reso, ptr(rows), len(cams), int(max_w), int(max_h),
                                     (ctypes.c_float * 3)(*map(float, off)), (ctypes.c_float * 3)(*map(float, inv)),
                                     ctypes.byref(o), ptr(wmax), ptr(hit), stream_ptr()))
    torch.cuda.synchronize()


def take(wmax, hit):
    """nonzero voxels of wmax (indices, values) and of hit (indices), and zero them again"""
    import torch
    kw = torch.nonzero(wmax).reshape(-1)
    vw = wmax[kw].cpu().numpy()
    kh = torch.nonzero(hit).reshape(-1)
    wmax[kw] = 0.0
    hit[kh] = 0
    return kw.cpu().numpy(), vw, kh.cpu().numpy()


def check_launch(ref, kw, vw, kh, tag):
    """path and values of one launch against its fp64 reference -> (largest error in units, mask margin count)"""
    required = ref["keys"][ref["pre"]]
    assert np.isin(kh, ref["keys"]).all(), (tag, "kernel hit a voxel no listed hit reaches")
    assert np.isin(required, kh).all(), (tag, "a listed hit before the cut is missing", np.setdiff1d(required, kh)[:8])
    assert np.isin(kw, ref["keys"]).all(), (tag, "nonzero weight on a voxel no positive-sigma visit reaches")
    err, got = weight_err(ref, kw, vw)
    worst = float(err.max()) if err.size else 0.0
    assert worst <= WEIGHT_ALLOW, (tag, worst, int(ref["keys"][np.argmax(err)]))
    # the mask outside the margin
    m = ref["hi"]
    margin = np.abs(m - WEIGHT_THRESH) <= WEIGHT_ALLOW * U24 * ref["unit"]
    bad = ((got >= f32(WEIGHT_THRESH)) != (m >= WEIGHT_THRESH)) & ~margin
    assert not bad.any(), (tag, int(bad.sum()))
    return worst, int(margin.sum()), int((m >= WEIGHT_THRESH).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("reso", RESOS)
def test_grid_weights_exact_path_and_values(reso):
    import torch
    R = reference(reso, "group")
    ref, stats = R["ref"], R["stats"]
    n = reso ** 3
    wmax = torch.zeros(n, dtype=torch.float32, device="cuda")
    hit = torch.zeros(n, dtype=torch.uint8, device="cuda")
    cams = camera_group(reso)
    # one launch of mixed camera sizes under a larger tile grid than any camera needs
    launch(reso, cams, wmax, hit, max_w=208, max_h=136)
    kw, vw, kh = take(wmax, hit)
    worst, margin, masked = check_launch(ref, kw, vw, kh, "cameras")
    hit_voxels = int(kh.size)
    assert hit_voxels > 1000 and masked > 100
    single_worst, single_cut = 0.0, 0
    for cam, sref, sstats in reference(reso, "single"):
        launch(reso, [cam], wmax, hit)
        kw, vw, kh = take(wmax, hit)
        w, _, _ = check_launch(sref, kw, vw, kh, "single")
        single_worst = max(single_worst, w)
        single_cut += sstats["rays_cut"]
    assert float(wmax.abs().max()) == 0.0 and int(hit.max()) == 0
    _record(f"grid_{reso}", dict(weight_err_units=worst, single_ray_err_units=single_worst, allow=WEIGHT_ALLOW,
                                 mask_margin_voxels=margin, masked_voxels=masked, hit_voxels=hit_voxels,
                                 single_rays_cut=single_cut, **stats))


def _ds(cams):
    class DS:
        pass
    ds = DS()
    ds.camtoworlds = np.stack([c[0] for c in cams])
    ds.w, ds.h, ds.focal = cams[0][1], cams[0][2], cams[0][3]
    return ds


@pytest.mark.gpu
def test_grid_weight_launch_invariants():
    import torch
    from plenoctree_b200.octree.extraction import calculate_grid_weights
    reso = 512
    off, inv = geometry()
    sig = device_sigma(reso)
    prod = camera_group(reso)[:8]
    args = (sig, reso, torch.from_numpy(inv).cuda(), torch.from_numpy(off).cuda(), STEP)
    base = calculate_grid_weights(_ds(prod), *args).reshape(-1)
    bits = base.view(torch.int32)
    one = calculate_grid_weights(_ds(prod), *args, cam_chunk=1).reshape(-1)
    assert torch.equal(one.view(torch.int32), bits)
    rev = calculate_grid_weights(_ds(prod[::-1]), *args, cam_chunk=3).reshape(-1)
    assert torch.equal(rev.view(torch.int32), bits)
    # a pre-filled wmax (how later chunks accumulate): the result is the elementwise maximum
    g = torch.Generator(device="cuda")
    g.manual_seed(3)
    pre = torch.rand(reso ** 3, device="cuda", generator=g) * 2e-3
    pre[torch.rand(reso ** 3, device="cuda", generator=g) < 0.5] = 0.0
    w = pre.clone()
    hit = torch.zeros(reso ** 3, dtype=torch.uint8, device="cuda")
    launch(reso, prod, w, hit)
    assert torch.equal(w.view(torch.int32), torch.maximum(pre, base).view(torch.int32))
    # mixed sizes in one launch equal the cameras launched alone, wmax and hit
    cams = camera_group(reso)[6:] + single_cams(reso)[:4]
    cams = [(c[0], 37, 23, 40.0) if i == 0 else c for i, c in enumerate(cams)]
    w1 = torch.zeros_like(base)
    h1 = torch.zeros_like(hit)
    launch(reso, cams, w1, h1, max_w=200, max_h=130)
    w2 = torch.zeros_like(base)
    h2 = torch.zeros_like(hit)
    for c in cams:
        launch(reso, [c], w2, h2)
    assert torch.equal(w1.view(torch.int32), w2.view(torch.int32)) and torch.equal(h1, h2)
    _record("invariants_512", dict(nonzero=int((base > 0).sum()), prefilled_raised=int((base > pre).sum()),
                                   mixed_hit=int(h1.sum())))


@pytest.mark.gpu
def test_production_launch_matches_single_camera_launches():
    """100 cameras at 800 x 800 around the box (the Blender training set's shape) in one launch, against the same
    cameras launched one by one into the same buffer"""
    import torch
    from plenoctree_b200.octree.extraction import calculate_grid_weights
    reso = 512
    off, inv = geometry()
    sig = device_sigma(reso)
    cams = [(look_at_pose(1000 + s, CAM_DIST), 800, 800, FOCAL_800) for s in range(100)]
    args = (sig, reso, torch.from_numpy(inv).cuda(), torch.from_numpy(off).cuda(), STEP)
    torch.cuda.synchronize()
    t0 = time.time()
    one = calculate_grid_weights(_ds(cams), *args).reshape(-1)
    torch.cuda.synchronize()
    t1 = time.time()
    each = calculate_grid_weights(_ds(cams), *args, cam_chunk=1).reshape(-1)
    torch.cuda.synchronize()
    assert torch.equal(one.view(torch.int32), each.view(torch.int32))
    masked = int((one >= WEIGHT_THRESH).sum())
    assert masked > 10000
    _record("production_launch_512", dict(cameras=100, width=800, height=800, masked_voxels=masked,
                                          nonzero=int((one > 0).sum()), one_launch_s=t1 - t0))


@pytest.mark.gpu
def test_extraction_step1_step2_at_depth_8():
    """step 1 whole at init_grid_depth 8 (sigma grid, grid weights, mask, refinement with a chunked last level) and
    step 2 with 256 samples per cell in at least three leaf chunks, the last one short"""
    import torch
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    from plenoctree_b200.nerf.models import NerfModel
    from plenoctree_b200.octree import N3Tree
    from plenoctree_b200.octree import extraction as E
    L, reso, S, sh_deg = 8, 512, 256, 3
    off, inv = geometry()
    flat = O.init_flat_params(sh_deg, 20200823, bias_scale=0.05)
    nerf = NerfModel(sh_deg=sh_deg)
    nerf.set_params(np.concatenate([flat, flat]))
    # a sparse scene from the random field: the sigma head (Dense_8) scaled and shifted so that the top 1e-3 of the
    # voxels have positive sigma, up to 60
    raw = E._grid_sigmas(nerf, reso, off.tolist(), inv.tolist())
    top = torch.topk(raw, int(raw.numel() * 1e-3)).values
    t, mx = float(top[-1]), float(top[0])
    del raw, top
    o8 = sum(ci * co + co for ci, co in O.layer_dims(sh_deg)[:8])
    width = O.layer_dims(sh_deg)[8][0]
    alpha = 60.0 / (mx - t)
    flat[o8:o8 + width] *= f32(alpha)
    flat[o8 + width] = f32(alpha * (float(flat[o8 + width]) - t))
    nerf.set_params(np.concatenate([flat, flat]))
    cams = camera_group(reso)[:8]
    ds = _ds(cams)
    sig = E._grid_sigmas(nerf, reso, off.tolist(), inv.tolist())
    wm = E.calculate_grid_weights(ds, sig, reso, torch.from_numpy(inv).cuda(), torch.from_numpy(off).cuda(),
                                  step_size=STEP).reshape(-1)
    # the recomputed mask (both calls are deterministic) against fp64, outside the margin
    sig_h = sig.cpu().numpy()
    ref, stats = march(reso, cams, lambda v: sig_h[v])
    kw = torch.nonzero(wm).reshape(-1)
    vw = wm[kw].cpu().numpy()
    kw = kw.cpu().numpy()
    assert np.isin(kw, ref["keys"]).all()
    err, got = weight_err(ref, kw, vw)
    worst = float(err.max())
    assert worst <= WEIGHT_ALLOW, worst
    margin = np.abs(ref["hi"] - WEIGHT_THRESH) <= WEIGHT_ALLOW * U24 * ref["unit"]
    assert not (((got >= f32(WEIGHT_THRESH)) != (ref["hi"] >= WEIGHT_THRESH)) & ~margin).any()
    mask = (wm >= WEIGHT_THRESH).cpu().numpy()
    n_mask = int(mask.sum())
    chunk = n_mask // 3 + 1                              # the last level in three chunks
    assert n_mask > 10000
    tree = N3Tree(N=2, data_dim=3 * 16 + 1, depth_limit=L, init_reserve=500000, geom_resize_fact=1.0, radius=RADIUS,
                  center=CENTER, data_format="SH16")
    assert np.array_equal(tree.offset.cpu().numpy(), off) and np.array_equal(tree.invradius.cpu().numpy(), inv)
    args = E.default_args(init_grid_depth=L, masking_mode="weight", weight_thresh=WEIGHT_THRESH,
                          renderer_step_size=STEP, samples_per_cell=S)
    E.step1(args, tree, nerf, ds, refine_chunk=chunk)
    otree, grid = OO.build_tree_from_grid(mask, L, RADIUS, CENTER, 49, "SH16", refine_chunk=chunk)
    n = otree.n_internal
    assert grid.shape[0] == n_mask and tree.n_internal == n
    assert np.array_equal(tree.child[:n].cpu().numpy(), otree.child[:n])
    assert np.array_equal(tree.parent_depth[:n].cpu().numpy(), otree.parent_depth[:n])
    # step 2: the leaves at depth 8 in the oracle's order, chunk c drawn from seed 20200823 + c
    lv = otree.leaves()
    deep = np.nonzero(otree.leaf_depths(lv) == L)[0]
    assert np.array_equal(tree._all_leaves().cpu().numpy(), lv)
    cpl = deep.size // 3 + 1
    n_chunks = -(-deep.size // cpl)
    assert n_chunks >= 3 and deep.size - (n_chunks - 1) * cpl < cpl
    E.step2(args, tree, nerf, cells_per_launch=cpl)
    got = tree.data.reshape(-1, 49)[torch.from_numpy(otree.pack_index(lv[deep, 0], lv[deep, 1:])).cuda()]
    gen = torch.Generator(device="cuda")

    def cell_means(sel, seed):
        gen.manual_seed(seed)
        u = torch.rand((sel.numel(), S, 3), device="cuda", generator=gen)
        pts = tree[sel].sample(S, uniforms=u)
        return ops.eval_cells_mean(nerf._blob(False), sh_deg, pts.contiguous(), S, precision=nerf.precision)

    # eval_cells_mean adds a cell's partial sums with atomics, so a rerun may round differently: the bar is
    # CELL_ALLOW units of 2^-24 x the column's largest |mean| in the chunk.  The neighbouring chunk's seed must
    # move a value by more than SENSITIVITY bars.
    worst_cell, seed_guard, exact = 0.0, np.inf, 0
    for c in range(n_chunks):
        g = got[c * cpl:(c + 1) * cpl]
        sel = torch.from_numpy(deep[c * cpl:(c + 1) * cpl]).cuda()
        want = cell_means(sel, 20200823 + c)
        unit = U24 * want.abs().amax(dim=0, keepdim=True).clamp_min(1e-30)
        worst_cell = max(worst_cell, float(((g - want).abs() / unit).max()))
        exact += int((g.view(torch.int32) == want.view(torch.int32)).sum())
        other = cell_means(sel, 20200823 + (c + 1 if c + 1 < n_chunks else c - 1))
        seed_guard = min(seed_guard, float(((other - want).abs() / unit).max()) / CELL_ALLOW)
    assert worst_cell <= CELL_ALLOW, worst_cell
    assert seed_guard > SENSITIVITY, seed_guard
    _record("extraction_depth8", dict(weight_err_units=worst, mask_margin_voxels=int(margin.sum()), masked=n_mask,
                                      refine_chunk=chunk, nodes=int(n), deep_leaves=int(deep.size),
                                      cells_per_launch=cpl, chunks=n_chunks, cell_err_units=worst_cell,
                                      cell_allow=CELL_ALLOW, cell_values_bit_equal=exact / float(got.numel()),
                                      seed_guard_ratio_to_bar=seed_guard, **stats))

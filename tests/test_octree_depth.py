"""Depth and opacity from the octree march (csrc/octree.cu, trace_forward / trace_backward with DEPTH = true):
pob_octree_render_depth, pob_octree_render_depth_backward, VolumeRenderer(..., return_depth=True), disparity() and
octree.evaluation --write_disp.

Definitions (include/plenoctree_b200.h): over the contributing visits i of a ray (sigma_i > sigma_thresh), visit i
starting at t_i with step dt_i and weight w_i,
    acc = sum_i w_i,   depth = sum_i w_i z_i,   z_i = (t_i + dt_i / 2) * delta_scale,
a parameter along the ray's direction vector; render_persp multiplies it by the pixel's 1 / |(x, y, -1)| (camera-axis
depth).  Early termination rescales both like the colour; a ray that misses has depth = acc = 0.

- CPU: the fp32 oracle (oracle/octree_depth_oracle.py) keeps octree_oracle.volume_render's rgb bit for bit, depth / acc match the closed form of a uniform box, and the
  oracle's backward for g_depth / g_acc matches central differences of an fp64 forward.
- GPU, on the production-depth trees of tests/test_octree_march.py: colour and counters bit-identical to
  pob_octree_render; depth / acc against fp64 shaded from the oracle's visit lists (t_i rebuilt in float32 exactly as
  the kernel steps it), per ray, in units of the rounding each accumulates, with a sensitivity guard; the backward
  bit-identical to pob_octree_render_backward for a colour-only gradient and held to fp64 for g_depth / g_acc;
  render_persp slabs and camera-axis depth; the evaluation CLI's disparity PNGs.
"""
import ctypes
import os

import numpy as np
import pytest

from oracle import octree_depth_oracle as DO, octree_oracle as OO
from tests.test_octree_march import (CAM_F, CAM_H, CAM_W, NAMES, SENSITIVITY, STOP, U24, _cameras, _fill, _first,
                                     _record as _record_march, _rows, _safe_fast_rays, _to_world, _unit_rand,
                                     device_tree, fwd64, world)

f32, f64 = np.float32, np.float64

# ---- bars (measured on an H100 80 GB HBM3 at a 700 W power limit; the largest value over all trees in brackets)
# acc: |acc - fp64| per ray in units of 2^-24 * (1 + n_hits + sum_j tau_j), times the early-stop rescale
ACC_ALLOW = 1.8             # [0.87]
# depth: |depth - fp64| per ray in units of 2^-24 * (z_max (1 + n_hits + sum_j tau_j) + 3 sum_j w_j |z_j|), times the
# early-stop rescale (z_j carries two roundings and the weighted sum one per visit)
DEPTH_ALLOW = 1.5           # [0.72]
# sigma gradient of g_depth / g_acc: per element, in units of 2^-24 * sum over the contributing visits reaching it of
# dt ds ((|z gz| + |ga|) T_next (1 + n_before + S + tau + 3) + |gz| U_depth + |ga| U_acc)
DGRAD_ALLOW = 0.65          # [0.31]
N_SEQ = 24                  # rays launched one at a time for the bit-identity of the colour-only backward


def _record(name, payload):
    _record_march(f"depth_{name}", payload)


# ---------------------------------------------------------------------------------------------------------
# fp64 references from a visit list
# ---------------------------------------------------------------------------------------------------------
def march_t(otree, o, d, vis):
    """the float32 entry t of every visit, stepped as the kernel steps it: t_0 = tmin, t_{k+1} = fl(t_k + dt_k)"""
    return DO._visit_t(otree, o, d, vis)[0]


def depth64(f, vis, t, sigma_thresh=0.0, z_mode="mid"):
    """fp64 depth / acc [R] of the forward `f` (fwd64 of the same visit list) and their bar units / 2^-24.
    z_mode "entry" / "no_scale" are the sensitivity guard's wrong definitions."""
    ray, R = vis["ray"], vis["miss"].shape[0]
    dt, ds, w = f["dt"], f["ds"], f["w"]
    t = t.astype(f64)
    z = {"mid": (t + 0.5 * dt) * ds, "entry": t * ds, "no_scale": t + 0.5 * dt}[z_mode]
    stopped = vis["stopped"] if sigma_thresh > 0 else np.zeros(R, dtype=bool)
    scale = 1.0 / np.where(stopped, 1.0 - f["tend"], 1.0)
    acc = np.bincount(ray, w, minlength=R) * scale
    depth = np.bincount(ray, w * z, minlength=R) * scale
    hit = f["hit"]
    base = 1.0 + np.bincount(ray, hit, minlength=R) + np.bincount(ray, f["tau"], minlength=R)
    zmax = np.zeros(R)
    np.maximum.at(zmax, ray[hit], np.abs(z[hit]))
    U_acc = base * scale
    U_depth = (zmax * base + 3.0 * np.bincount(ray, w * np.abs(z), minlength=R)) * scale
    return dict(depth=depth, acc=acc, z=z, U_depth=U_depth, U_acc=U_acc)


def dsigma64(f, vis, dz, gz, ga):
    """fp64 sigma gradient of <gz, depth> + <ga, acc> (explicit rays, thresholds 0) -> (touched leaves, grad, unit)"""
    ray, R = vis["ray"], vis["miss"].shape[0]
    h = np.nonzero(f["hit"])[0]
    r = ray[h]
    w, T, tau, S, z = f["w"][h], f["T"][h], f["tau"][h], f["S"][h], dz["z"][h]
    tnext = T * np.exp(-tau)
    tot = z * gz[r] + ga[r]
    wt = np.zeros(ray.shape[0])
    wt[h] = w * tot
    after = (np.bincount(ray, wt, minlength=R)[ray] - (_excl(wt, ray, f["first"]) + wt))[h]
    d = f["dt"][h] * f["ds"][h]
    g = d * (tot * tnext - after)
    depth = 1.0 + f["nh_before"][h] + S
    unit = d * ((np.abs(z * gz[r]) + np.abs(ga[r])) * tnext * (depth + tau + 3.0)
                + np.abs(gz[r]) * dz["U_depth"][r] + np.abs(ga[r]) * dz["U_acc"][r])
    uniq, inv = np.unique(vis["leaf"][h], return_inverse=True)
    return uniq, np.bincount(inv, g, minlength=uniq.size), np.bincount(inv, unit, minlength=uniq.size)


def _excl(x, ray, first):
    c = np.cumsum(x) - x
    return c - c[first[ray]] if x.size else c


# ---------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------
def _small_tree(N, fmt, seed):
    rs = np.random.RandomState(seed)
    K = 1 if fmt == "RGBA" else int(fmt[2:])
    otree = OO.N3Tree(N=N, data_dim=4 if fmt == "RGBA" else 3 * K + 1, depth_limit=3, radius=(1.2, 0.9, 1.0),
                      center=(0.1, -0.1, 0.05), data_format=fmt)
    pts = _to_world(otree, rs.uniform(0.1, 0.9, size=(60, 3)))
    for _ in range(3):
        otree.refine_at(pts)
    _fill(otree, rs, tau_cell=1.5)
    o = (3.0 * _unit_rand(rs, 96)).astype(f32)
    tgt = pts[rs.randint(0, 60, 96)]
    d = ((tgt - o) / np.linalg.norm(tgt - o, axis=1, keepdims=True)).astype(f32)
    d[:8] *= -1.0                                          # some miss the box
    return otree, o, d


@pytest.mark.parametrize("N,fmt", [(2, "SH9"), (3, "RGBA")])
def test_oracle_rgb_unchanged_and_depth_from_the_visit_list(N, fmt):
    otree, o, d = _small_tree(N, fmt, 3 + N)
    for th in (0.0, STOP):
        rgb, visits, hits = OO.volume_render(otree, o, d, d, 1e-3, 0.25, th, th, return_steps=True)
        rgb2, depth, acc, visits2, hits2 = DO.volume_render_depth(otree, o, d, d, 1e-3, 0.25, th, th,
                                                                  return_steps=True)
        assert np.array_equal(rgb.view(np.int32), rgb2.view(np.int32))
        assert np.array_equal(visits, visits2) and np.array_equal(hits, hits2)
        # the fp64 shading of the same visit list agrees to float32 precision
        vis = OO.march_visits(otree, o, d, d, 1e-3, 0.25, th, th)
        dz = depth64(fwd64(otree, vis, d, 0.25, th), vis, march_t(otree, o, d, vis), th)
        assert np.abs(acc - dz["acc"]).max() < 1e-5
        assert np.abs(depth - dz["depth"]).max() < 1e-5 * np.abs(dz["depth"]).max()
        miss = vis["miss"]
        assert miss.sum() >= 8 and not depth[miss].any() and not acc[miss].any()
        if th:
            st = vis["stopped"]
            assert st.sum() > 5 and np.abs(acc[st] - 1.0).max() < 4 * U24


def test_oracle_uniform_box_closed_form():
    """all 8 cells of one node hold the same sigma; a ray along -z through the box crosses two cells: visit 1 from the
    top face e for L/2 + step, visit 2 for L/2 (its step is the exit length minus the step it started past the face)"""
    radius, center, step = (0.7, 1.1, 0.9), (0.2, -0.3, 0.1), 1e-3
    otree = OO.N3Tree(N=2, data_dim=4, depth_limit=1, radius=radius, center=center, data_format="RGBA")
    sigma = 1.3
    otree.data[0, ..., :3] = 0.2
    otree.data[0, ..., 3] = sigma
    h = 2.0
    xy = [(center[0] + 0.31 * radius[0], center[1] - 0.47 * radius[1]), (center[0] - 0.6 * radius[0], center[1] + 0.2 * radius[1])]
    o = np.array([[x, y, center[2] + radius[2] + h] for x, y in xy], dtype=f32)
    d = np.tile(np.array([[0, 0, -1]], dtype=f32), (2, 1))
    L, s_w = 2.0 * radius[2], step * 2.0 * radius[2]          # world box height and world step
    seg = [(h, L / 2 + s_w), (h + L / 2 + s_w, L / 2)]        # (world entry, world length)
    T, depth, acc = 1.0, 0.0, 0.0
    for e, ln in seg:
        w = T * -np.expm1(-sigma * ln)
        depth += w * (e + ln / 2)
        acc += w
        T *= np.exp(-sigma * ln)
    rgb, got_d, got_a = DO.volume_render_depth(otree, o, d, d, step, 1.0)
    assert abs(acc - (1.0 - np.exp(-sigma * (L + s_w)))) < 1e-12
    np.testing.assert_allclose(got_a, acc, rtol=4e-6)
    np.testing.assert_allclose(got_d, depth, rtol=4e-6)
    # early termination after the first cell: acc = 1, depth = that cell's midpoint
    otree.data[0, ..., 3] = 20.0
    _, got_d, got_a = DO.volume_render_depth(otree, o, d, d, step, 1.0, STOP, STOP)
    np.testing.assert_allclose(got_a, 1.0, rtol=2e-7)
    np.testing.assert_allclose(got_d, h + (L / 2 + s_w) / 2, rtol=4e-6)
    # a ray that misses
    _, got_d, got_a = DO.volume_render_depth(otree, o, -d, -d, step, 1.0)
    assert not got_d.any() and not got_a.any()


def test_oracle_backward_matches_central_differences():
    otree, o, d = _small_tree(2, "SH4", 9)
    rs = np.random.RandomState(1)
    R = o.shape[0]
    gz, ga = rs.normal(size=R).astype(f32), rs.normal(size=R).astype(f32)
    step, bg = 1e-3, 0.25
    grad = DO.volume_render_depth_backward(otree, o, d, d, np.zeros((R, 3), f32), step, bg, grad_depth=gz,
                                           grad_acc=ga)
    D = otree.data_dim
    flat = grad.reshape(-1, D)
    assert not flat[:, :D - 1].any()                        # depth and acc reach sigma only
    vis = OO.march_visits(otree, o, d, d, step, bg)
    t = march_t(otree, o, d, vis)
    rows0 = _rows(otree, vis["leaf"]).astype(f64)

    def loss(rows):
        dz = depth64(fwd64(otree, vis, d, bg, rows=rows), vis, t)
        return float((dz["depth"] * gz).sum() + (dz["acc"] * ga).sum())
    hit_leaves = np.unique(vis["leaf"][rows0[:, -1] > 0])
    assert hit_leaves.size > 40
    sel = hit_leaves[rs.choice(hit_leaves.size, 40, replace=False)]
    scale = np.abs(flat[hit_leaves, D - 1]).max()
    for leaf in sel:
        on = vis["leaf"] == leaf
        eps = 1e-4 * abs(float(otree.data.reshape(-1, D)[leaf, -1]))
        rp, rm = rows0.copy(), rows0.copy()
        rp[on, -1] += eps
        rm[on, -1] -= eps
        fd = (loss(rp) - loss(rm)) / (2 * eps)
        assert abs(flat[leaf, D - 1] - fd) <= 2e-5 * scale + 1e-4 * abs(fd), (leaf, flat[leaf, D - 1], fd)
    # untouched leaves are exactly zero
    rest = np.ones(flat.shape[0], dtype=bool)
    rest[hit_leaves] = False
    assert not flat[rest].any()


def test_disparity_rule():
    import torch
    from plenoctree_b200.octree import disparity
    depth = torch.tensor([[2.0], [0.0], [4.0], [1e-12], [3.0], [-1.0]])
    acc = torch.tensor([[0.5], [0.0], [1e-11], [1.0], [0.0], [0.5]])
    want = torch.tensor([[0.25], [1e10], [1e10], [1e10], [1e10], [1e10]])
    assert torch.equal(disparity(depth, acc), want)


# ---------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------
def _renderer(name, step, bg):
    from plenoctree_b200.octree import VolumeRenderer
    return VolumeRenderer(device_tree(name), step_size=step, background_brightness=bg)


def _rays(o, d, v):
    import torch
    from plenoctree_b200.octree import Rays
    return Rays(torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(v))


def _render(r, o, d, v, fast, return_depth):
    import torch
    cnt = torch.zeros(2, dtype=torch.int64, device="cuda")
    with torch.no_grad():
        out = r.forward(_rays(o, d, v), fast=fast, counters=cnt, return_depth=return_depth)
    out = out if return_depth else (out,)
    return tuple(x.cpu().numpy() for x in out) + (cnt.cpu().numpy(),)


def _bits(x):
    return np.ascontiguousarray(x, dtype=f32).view(np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_colour_and_counters_unchanged(name):
    import torch
    W = world(name)
    for S in W["sets"]:
        r = _renderer(name, S["step"], S["bg"])
        for fast in (False, True):
            rgb, cnt = _render(r, S["o"], S["d"], S["v"], fast, False)
            rgb2, depth, acc, cnt2 = _render(r, S["o"], S["d"], S["v"], fast, True)
            assert np.array_equal(_bits(rgb), _bits(rgb2)), (S["name"], fast)
            assert np.array_equal(cnt, cnt2), (S["name"], fast, cnt, cnt2)
            assert depth.shape == acc.shape == (S["o"].shape[0], 1)
    for c2w in _cameras(W["otree"]):
        r = _renderer(name, 1e-3, 0.25)
        with torch.no_grad():
            for fast in (False, True):
                a = r.render_persp(c2w, width=CAM_W, height=CAM_H, fx=CAM_F, fast=fast)
                b, depth, acc = r.render_persp(c2w, width=CAM_W, height=CAM_H, fx=CAM_F, fast=fast, return_depth=True)
                assert torch.equal(a.view(torch.int32), b.view(torch.int32))
                assert depth.shape == acc.shape == (CAM_H, CAM_W, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_depth_and_acc_match_fp64(name):
    W = world(name)
    otree = W["otree"]
    rec = {}
    worst = {"depth": 0.0, "acc": 0.0}
    guards = {}
    for S in W["sets"]:
        o, d, v, step, bg = S["o"], S["d"], S["v"], S["step"], S["bg"]
        r = _renderer(name, step, bg)
        for fast in (False, True):
            vis = S["visf"] if fast else S["vis"]
            th = STOP if fast else 0.0
            f = fwd64(otree, vis, v, bg, th)
            t = march_t(otree, o, d, vis)
            dz = depth64(f, vis, t, th)
            _, depth, acc, _ = _render(r, o, d, v, fast, True)
            depth, acc = depth[:, 0].astype(f64), acc[:, 0].astype(f64)
            keep = _safe_fast_rays(f, vis) if fast else np.ones(o.shape[0], dtype=bool)
            if fast:
                assert keep.sum() > 0.9 * o.shape[0]
            errs = {}
            for k, got in (("depth", depth), ("acc", acc)):
                U = U24 * dz[f"U_{k}"]
                zero = U == 0                                   # rays with no contributing visit: exactly 0
                assert not got[keep & zero].any(), (S["name"], fast, k)
                e = np.abs(got - dz[k]) / np.where(zero, 1.0, U)
                errs[k] = float(e[keep & ~zero].max(initial=0.0))
                worst[k] = max(worst[k], errs[k])
            rec[f"{S['name']}_{'fast' if fast else 'full'}"] = errs
            if not fast:
                for mode in ("entry", "no_scale"):
                    wrong = depth64(f, vis, t, z_mode=mode)["depth"]
                    U = U24 * dz["U_depth"]
                    ok = U > 0
                    guards[f"{S['name']}_{mode}"] = float((np.abs(wrong - dz["depth"])[ok] / U[ok]).max())
    rec.update(worst=worst, depth_allow=DEPTH_ALLOW, acc_allow=ACC_ALLOW, guard_units=guards,
               guard_ratio_to_bar={k: x / DEPTH_ALLOW for k, x in guards.items()})
    _record(f"forward_{name}", rec)
    assert worst["depth"] <= DEPTH_ALLOW and worst["acc"] <= ACC_ALLOW, worst
    for k, x in guards.items():
        assert x > SENSITIVITY * DEPTH_ALLOW, (k, x / DEPTH_ALLOW)


def _disjoint_rays(otree, vis):
    """rays whose contributing (sigma > 0) leaves are pairwise disjoint: in one launch every gradient element then
    receives at most one atomic add, so the result does not depend on the order of the atomics"""
    hit = _rows(otree, vis["leaf"])[:, -1] > 0
    ray = vis["ray"]
    seen, pick = set(), []
    for i in range(vis["miss"].shape[0]):
        leaves = set(vis["leaf"][(ray == i) & hit].tolist())
        if leaves and not (leaves & seen):
            seen |= leaves
            pick.append(i)
    return np.array(pick, dtype=np.int64)


def _c_backward(r, o, d, v, g_rgb, g_depth, g_acc, depth_entry=True, one_ray_per_launch=False):
    """grad_data of pob_octree_render_depth_backward (or pob_octree_render_backward) on explicit rays.
    one_ray_per_launch: the rays are launched one at a time into the same buffer, so every element receives its atomic
    adds in ray order and the result does not depend on the order in which concurrent atomics land."""
    import torch
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    tree = r.tree
    g = torch.zeros_like(tree.data)
    t, opts = tree.c_struct(), r._opts(False)
    dev = lambda x: None if x is None else torch.from_numpy(np.ascontiguousarray(x, dtype=f32)).cuda()   # noqa: E731
    ro, rd, rv, gr, gd, ga = (dev(x) for x in (o, d, v, g_rgb, g_depth, g_acc))
    for i, n in ([(i, 1) for i in range(o.shape[0])] if one_ray_per_launch else [(0, o.shape[0])]):
        src = (ctypes.byref(t), ctypes.byref(opts), ptr(ro[i:]), ptr(rd[i:]), ptr(rv[i:]), n, None, 0, 0)
        gri, gdi, gai = (None if x is None else x.reshape(-1)[i * c:] for x, c in ((gr, 3), (gd, 1), (ga, 1)))
        if depth_entry:
            check(lib.pob_octree_render_depth_backward(*src, ptr(gri), ptr(gdi), ptr(gai), ptr(g), stream_ptr()))
        else:
            check(lib.pob_octree_render_backward(*src, ptr(gri), ptr(g), stream_ptr()))
    return g.reshape(-1, tree.data_dim)[: r.tree.n_internal * r.tree.N ** 3].cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_backward_colour_bits_and_depth_gradient(name):
    import torch
    W = world(name)
    otree = W["otree"]
    D = otree.data_dim
    rec = {}
    for S in W["sets"][:2]:
        o, d, v, step, bg = S["o"], S["d"], S["v"], S["step"], S["bg"]
        R = o.shape[0]
        r = _renderer(name, step, bg)
        rs = np.random.RandomState(5)
        g_rgb = rs.normal(size=(R, 3)).astype(f32)
        # (1) a colour-only gradient: bit-identical to pob_octree_render_backward, rays launched one at a time
        hits = np.nonzero(S["vis"]["hits"] > 0)[0]
        one = hits[rs.choice(hits.size, N_SEQ, replace=False)]
        want = _c_backward(r, o[one], d[one], v[one], g_rgb[one], None, None, depth_entry=False,
                           one_ray_per_launch=True)
        assert want.any()
        zeros = np.zeros(one.size, f32)
        for gd, ga in ((None, None), (zeros, zeros)):
            got = _c_backward(r, o[one], d[one], v[one], g_rgb[one], gd, ga, one_ray_per_launch=True)
            assert np.array_equal(_bits(got), _bits(want)), (S["name"], gd is None)
        # ... and through autograd (rgb, depth, acc), on rays whose leaves are disjoint (one launch, one add per element)
        pick = _disjoint_rays(otree, S["vis"])
        assert pick.size >= 2, pick.size
        so, sd, sv, sg = o[pick], d[pick], v[pick], g_rgb[pick]
        tree = r.tree
        gz, ga = rs.normal(size=R).astype(f32), rs.normal(size=R).astype(f32)
        tree.data.requires_grad_(True)
        tree.data.grad = None
        rgb, depth, acc = r.forward(_rays(so, sd, sv), return_depth=True)
        cu = lambda x: torch.from_numpy(x).cuda()   # noqa: E731
        ((rgb * cu(sg)).sum() + (depth[:, 0] * cu(gz[pick])).sum() + (acc[:, 0] * cu(ga[pick])).sum()).backward()
        auto = tree.data.grad.reshape(-1, D)[: otree.n_internal * otree.N ** 3].cpu().numpy()
        tree.data.grad = None
        tree.data.requires_grad_(False)
        assert np.array_equal(_bits(auto), _bits(_c_backward(r, so, sd, sv, sg, gz[pick], ga[pick])))
        # (2) random g_depth / g_acc alone, all rays: sigma against fp64, coefficients exactly 0, untouched leaves 0
        got = _c_backward(r, o, d, v, None, gz, ga)
        assert not got[:, :D - 1].any()
        f = fwd64(otree, S["vis"], v, bg)
        dz = depth64(f, S["vis"], march_t(otree, o, d, S["vis"]))
        uniq, grad, unit = dsigma64(f, S["vis"], dz, gz.astype(f64), ga.astype(f64))
        rest = np.ones(got.shape[0], dtype=bool)
        rest[uniq] = False
        assert not got[rest].any()
        e = np.abs(got[uniq, D - 1].astype(f64) - grad) / (U24 * np.maximum(unit, 1e-300))
        e[(unit == 0) & (got[uniq, D - 1] == 0)] = 0.0
        rec[S["name"]] = float(e.max())
        assert (got[uniq, D - 1] != 0).sum() > 0.5 * uniq.size
    _record(f"backward_{name}", {"dsigma_err_units": rec, "dgrad_allow": DGRAD_ALLOW})
    for k, x in rec.items():
        assert x <= DGRAD_ALLOW, (k, x)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_persp_slabs_and_camera_axis_depth(name):
    import torch
    W = world(name)
    for c2w in _cameras(W["otree"]):
        r = _renderer(name, 1e-3, 0.25)
        o, d, v = OO.persp_rays(c2w, CAM_W, CAM_H, CAM_F)
        # the camera-axis factor 1 / |(x, y, -1)| of each pixel, as OO.persp_rays forms the norm
        ix, iy = np.meshgrid(np.arange(CAM_W, dtype=f32), np.arange(CAM_H, dtype=f32), indexing="xy")
        x = ((ix - f32(0.5) * f32(CAM_W)) / f32(CAM_F)).astype(f32).reshape(-1)
        y = (-(iy - f32(0.5) * f32(CAM_H)) / f32(CAM_F)).astype(f32).reshape(-1)
        nrm = np.sqrt((x * x + y * y).astype(f32) + f32(1.0)).astype(f32)
        axis = (f32(1.0) / nrm).astype(f32)
        for fast in (False, True):
            with torch.no_grad():
                full = [x.cpu().numpy() for x in r.render_persp(c2w, CAM_W, CAM_H, CAM_F, fast=fast, return_depth=True)]
                slabs = [[x.cpu().numpy() for x in r.render_persp(c2w, CAM_W, CAM_H, CAM_F, fast=fast,
                                                                   rows=(a, b - a), return_depth=True)]
                         for a, b in ((0, 7), (7, 8), (8, CAM_H))]
            for i in range(3):
                assert np.array_equal(_bits(np.concatenate([s[i] for s in slabs])), _bits(full[i])), (fast, i)
            rgb_e, depth_e, acc_e, _ = _render(r, o, d, v, fast, True)
            assert np.array_equal(_bits(full[0].reshape(-1, 3)), _bits(rgb_e))
            assert np.array_equal(_bits(full[2].reshape(-1)), _bits(acc_e[:, 0]))
            want = (depth_e[:, 0] * axis).astype(f32)
            ulp = np.abs(_bits(full[1].reshape(-1)).astype(np.int64) - _bits(want).astype(np.int64))
            assert ulp.max() <= 1, (fast, int(ulp.max()))
            assert (acc_e > 0).sum() > 50
        # the autograd edge of render_persp: a depth gradient reaches the march through the camera-axis factor, so it
        # equals the explicit rays' backward with g_depth * factor (up to the order of the atomics)
        tree = r.tree
        D = tree.data_dim
        rs = np.random.RandomState(6)
        gz, ga = rs.normal(size=CAM_H * CAM_W).astype(f32), rs.normal(size=CAM_H * CAM_W).astype(f32)
        tree.data.requires_grad_(True)
        tree.data.grad = None
        _, depth, acc = r.render_persp(c2w, CAM_W, CAM_H, CAM_F, return_depth=True)
        ((depth.reshape(-1) * torch.from_numpy(gz).cuda()).sum() + (acc.reshape(-1) * torch.from_numpy(ga).cuda()).sum()
         ).backward()
        got = tree.data.grad.reshape(-1, D)[: tree.n_internal * tree.N ** 3].cpu().numpy()
        tree.data.grad = None
        tree.data.requires_grad_(False)
        want = _c_backward(r, o, d, v, None, (gz * axis).astype(f32), ga)
        assert not got[:, :D - 1].any() and np.array_equal(got[:, -1] != 0, want[:, -1] != 0)
        assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max() and np.abs(want).max() > 0


@pytest.mark.gpu
def test_cli_evaluation_write_disp(tmp_path):
    """`python -m octree.evaluation ... --write_disp DIR` writes disp_{i:04d}.png per test view, of the image's shape,
    holding save_img of disparity(depth, acc) of the same render; --write_images keeps writing the colour images"""
    import json
    import torch
    from PIL import Image
    from tests.test_octree_momentum import _cli, _scene
    from plenoctree_b200.octree import N3Tree, VolumeRenderer, disparity
    common = _scene(tmp_path)
    out = tmp_path / "disp"
    _cli("octree.evaluation", common + ["--input", str(tmp_path / "tree.npz"), "--write_disp", str(out),
                                        "--write_images", str(tmp_path / "img")])
    assert sorted(os.listdir(out)) == ["disp_0000.png", "disp_0001.png"]
    assert sorted(os.listdir(tmp_path / "img")) == ["0000.png", "0001.png"]
    # the test cameras as the Blender loader reads them
    meta = json.load(open(tmp_path / "scene" / "transforms_test.json"))
    focal = 0.5 * 32 / np.tan(0.5 * float(meta["camera_angle_x"]))
    r = VolumeRenderer(N3Tree.load(str(tmp_path / "tree.npz"), map_location="cuda"), step_size=1e-3)
    hit = 0
    for i, frame in enumerate(meta["frames"]):
        im = np.asarray(Image.open(str(out / f"disp_{i:04d}.png")))
        assert im.shape == (32, 32) and im.dtype == np.uint8
        with torch.no_grad():
            _, depth, acc = r.render_persp(np.asarray(frame["transform_matrix"], dtype=f32), 32, 32, focal, fast=True,
                                           return_depth=True)
        disp = disparity(depth, acc)[..., 0].cpu().numpy()
        want = (np.clip(disp, 0.0, 1.0) * 255.0).astype(np.uint8)
        assert np.array_equal(im, want), (i, int((im != want).sum()))
        hit += int((disp < 1e10).sum())
    assert hit > 100

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

import numpy as np
import pytest

from oracle import octree_oracle as OO
from tests.support.octree_refs import (GRAD_ALLOW, RGB_ALLOW, SENSITIVITY, SQ_ALLOW, TRAIN_ALLOW, U24, _check_grad,
                                       _first, _layout, _rows, _safe_fast_rays, bwd64, fwd64)
from tests.support.octree_scenes import (CAM_F, CAM_H, CAM_W, NAMES, SPECS, STOP, _cameras, _fill, _to_world,
                                         _unit_rand, assert_device_tree_build_matches, device_tree, f32, f64, world)
from tests.support.records import record

# SGD: data - lr * g is one fused, correctly rounded operation, within 2^-24 * (|data| + |lr g|) of fp64  [0.998]

N_SINGLE = 32               # single-ray launches per ray set


_record = functools.partial(record, "parity_octree_march.json")


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


def _renderer(name, step, bg):
    from plenoctree_b200.octree import VolumeRenderer
    return VolumeRenderer(device_tree(name), step_size=step, background_brightness=bg)


def _forward(r, o, d, v, fast, counters=None):
    import torch
    from plenoctree_b200.octree import Rays
    with torch.no_grad():
        return r.forward(Rays(torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(v)), fast=fast,
                         counters=counters)


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

"""Forward-facing (LLFF) scenes on the PlenOctree path: NDC rays in the octree renderer, its backward, depth, compressed
trees, the fused training pass and extraction's grid-weight mask, and the CLIs that select them.

- The NDC transform (oracle/octree_ndc_oracle.py) is the reference's convert_to_ndc at near = 1, then the direction
  normalised for the march, the SH view direction left as the world one.  The first test pins the transform on the
  executed reference's NDC rays (tests/golden/ref_llff.npz); the GPU tests hold the kernels to it and to
  test_octree_march.py's / test_grid_weights.py's fp64 references, with exact leaf and voxel paths.
- The end-to-end test runs the CLI chain on a synthetic LLFF scene: nerf_sh.train, octree.extraction --z_min/--z_max,
  octree.optimization, octree.evaluation, all in NDC.  The raw tree must render the held-out views within PSNR_BOUND
  of the model's own render of them.  Two negative controls check the two svox assumptions of the transform: NDC view
  directions in place of world ones, and no NDC transform at all, must each miss that bound.
"""
import functools
import os
import types

import numpy as np
import pytest

from oracle import octree_ndc_oracle as ON
from oracle import octree_oracle as OO
from tests.support.records import record

f32, f64 = np.float32, np.float64
U24 = 2.0 ** -24
NDC_RAY_ULPS = 0        # kernel NDC rays against the float32 oracle: same operations, same order, same roundings
# raw tree against the NeRF-SH model on the held-out views of the end-to-end scene, dB (measured on an H100 80 GB HBM3
# at a 700 W power limit: see _record's llff_end_to_end; the two negative controls sit near 10 dB)
PSNR_BOUND = 18.0


_record = functools.partial(record, "parity_octree_ndc.json", echo=True)


def _ulps(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return int(np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64)).max())


# ---------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------
def _ref_world_rays(w, h, focal, c2w):
    """the world rays of the reference's generate_rays (nerf_sh/nerf/utils.py:545-587) in its float32 operations"""
    x, y = np.meshgrid(np.arange(w, dtype=f32), np.arange(h, dtype=f32), indexing="xy")
    cd = np.stack([(x - w * 0.5) / focal, -(y - h * 0.5) / focal, -np.ones_like(x)], axis=-1)
    d = np.matmul(c2w[:, None, None, :3, :3], cd[None, ..., None])[..., 0]
    o = np.broadcast_to(c2w[:, None, None, :3, -1], d.shape)
    return o.reshape(-1, 3), d.reshape(-1, 3), (d / np.linalg.norm(d, axis=-1, keepdims=True)).reshape(-1, 3)


def test_oracle_ndc_matches_executed_reference(golden_dir):
    """the oracle's convert_to_ndc on the reference's world rays reproduces the NDC rays its LLFF loader handed out:
    the views of both splits and the spiral path of the forward-facing scene (the `ring` scene is spherified: no NDC),
    and free rays"""
    z = np.load(os.path.join(golden_dir, "ref_llff.npz"))
    worst, n = 0, 0
    for split in ("train", "test"):
        k = f"fwd_{split}_"
        h, w, _ = (int(x) for x in z[k + "hw_n"])
        f = z[k + "focal"]
        sets = [(z[k + "camtoworlds"], "rays_")]
        if split == "test":
            sets.append((z[k + "render_poses"][::15], "render_rays_"))
        for c2w, key in sets:
            o, d, v = _ref_world_rays(w, h, f, c2w)
            no, nd = ON.convert_to_ndc(o, d, f, w, h)
            for got, c in ((no, "o"), (nd, "d"), (v, "v")):
                worst = max(worst, _ulps(got, z[k + key + c].reshape(-1, 3)))
            n += o.shape[0]
    no, nd = ON.convert_to_ndc(z["ndc_in_o"], z["ndc_in_d"], f32(21.5), 16, 12)
    worst = max(worst, _ulps(no, z["ndc_o_1.0"]), _ulps(nd, z["ndc_d_1.0"]))
    assert n > 1000 and worst <= 1, worst
    # the march's direction is the normalised NDC direction; the view direction passes through
    o, d, v = ON.ndc_rays(z["ndc_in_o"], z["ndc_in_d"], z["ndc_in_d"], f32(21.5), 16, 12)
    assert np.allclose(np.linalg.norm(d.astype(f64), axis=1), 1.0, atol=1e-6) and np.array_equal(v, z["ndc_in_d"])


def test_z_crop_matches_reference_filtering():
    """--z_min / --z_max: the points step 1 refines with and auto_scale's box equal the reference's, which crops zz
    before the meshgrid (octree/extraction.py:257-260,298-301)"""
    import torch
    from plenoctree_b200.octree import extraction as E
    reso = 16
    offset = torch.tensor([0.5, 0.45, 0.55], dtype=torch.float32)
    scale = torch.tensor([0.5, 0.6, 0.4], dtype=torch.float32)
    xx, yy, zz = E._axes(reso, offset, scale, "cpu")
    sig = torch.from_numpy(np.random.RandomState(4).uniform(0, 10, reso ** 3).astype(f32))
    full = sig.reshape(reso, reso, reso)
    alpha = 0.5
    thresh = -np.log(1.0 - alpha) / (2.0 / reso)
    for z_min, z_max in ((None, None), (-0.3, None), (None, 0.7), (-0.9, 0.35), (0.2, 0.1)):
        args = types.SimpleNamespace(z_min=z_min, z_max=z_max)
        zr = zz
        if z_min is not None:
            zr = zr[zr >= z_min]
        if z_max is not None:
            zr = zr[zr <= z_max]
        grid = torch.stack(torch.meshgrid(xx, yy, zr, indexing="ij")).reshape(3, -1).T
        keep = E.z_keep(args, zz)
        sub = full if keep is None else full[:, :, keep]
        assert sub.shape[2] == zr.numel()
        want = grid[sub.reshape(-1) >= 5.0]
        got = E.grid_points(full >= 5.0, keep, xx, yy, zz)
        assert torch.equal(got, want), (z_min, z_max)
        occ = grid[sub.reshape(-1) >= thresh]
        if occ.shape[0] == 0:
            continue
        lc, uc = occ.min(dim=0)[0] - 0.5 / reso, occ.max(dim=0)[0] + 0.5 / reso
        center, radius = E._bbox_of_dense(sig, alpha, reso, offset, scale, keep)
        np.testing.assert_allclose(center, ((lc + uc) * 0.5).tolist(), rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(radius, ((uc - lc) * 0.5).tolist(), rtol=1e-6, atol=1e-7)


class _Chosen(Exception):
    pass


CONDITIONS = [("/data/cfg/llff", False, True), ("/data/cfg/llff", True, False), ("/data/cfg/blender", False, False),
              (None, False, False)]


@pytest.mark.parametrize("config,spherify,ndc", CONDITIONS)
def test_ndc_condition_per_cli(monkeypatch, config, spherify, ndc):
    """extraction's weight mask, optimization and evaluation all march in NDC exactly when 'llff' is in --config and
    --spherify is off (the reference's optimization tests 'llff' alone)"""
    import torch
    from plenoctree_b200.octree import evaluation as EV, extraction as E, optimization as OPT
    from plenoctree_b200.octree.renderer import NDCConfig, scene_ndc
    w, h, focal = 16, 12, 20.5
    want = NDCConfig(w, h, focal) if ndc else None
    assert scene_ndc(types.SimpleNamespace(config=config, spherify=spherify), w, h, focal) == want
    seen = []

    class Renderer:
        def __init__(self, tree, step_size=1e-3, background_brightness=1.0, ndc=None):
            seen.append(ndc)
            raise _Chosen

    def weights(*a, **kw):
        seen.append(kw.get("ndc"))
        raise _Chosen

    monkeypatch.setattr(EV, "VolumeRenderer", Renderer)
    monkeypatch.setattr(OPT, "VolumeRenderer", Renderer)
    monkeypatch.setattr(E, "calculate_grid_weights", weights)
    monkeypatch.setattr(E, "_grid_sigmas", lambda nerf, reso, off, sc: torch.zeros(reso ** 3))
    ds = types.SimpleNamespace(w=w, h=h, focal=focal, size=1)
    with pytest.raises(_Chosen):
        EV.eval_octree(None, ds, types.SimpleNamespace(config=config, spherify=spherify, renderer_step_size=1e-3,
                                                       no_early_stop=False))
    gt = [torch.zeros((h, w, 3))]
    with pytest.raises(_Chosen):
        OPT.optimize(OPT.default_args(config=config, spherify=spherify), None, [np.eye(4)], gt, [np.eye(4)], gt, focal)
    tree = types.SimpleNamespace(offset=torch.full((3,), 0.5), invradius=torch.full((3,), 0.5), device="cpu")
    with pytest.raises(_Chosen):
        E.step1(E.default_args(init_grid_depth=2, config=config, spherify=spherify), tree, None, ds)
    assert seen == [want] * 3


# ---------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------
NDC_W, NDC_H, NDC_F = 32, 24, 27.0


def _rot(ax, ay):
    cx, sx, cy, sy = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay)
    return np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])


def ndc_cameras():
    """forward-facing cameras near the origin looking down -z (recentred LLFF poses)"""
    out = []
    for ax, ay, t in ((0.0, 0.0, (0.0, 0.0, 0.0)), (0.08, -0.12, (0.21, -0.13, 0.05)),
                      (-0.15, 0.1, (-0.3, 0.17, -0.08))):
        c2w = np.eye(4, dtype=f32)
        c2w[:3, :3] = _rot(ax, ay)
        c2w[:3, 3] = t
        out.append(c2w)
    return out


@functools.lru_cache(maxsize=None)
def device_tree(name):
    """a device copy of test_octree_march's tree `name` of this module's own (that module's SGD test steps its copy)"""
    from tests.support.octree_scenes import to_device_tree
    from tests.support.octree_scenes import world
    return to_device_tree(world(name)["otree"])


def _renderer(tree, step, bg, ndc=True):
    from plenoctree_b200.octree import NDCConfig, VolumeRenderer
    return VolumeRenderer(tree, step_size=step, background_brightness=bg,
                          ndc=NDCConfig(NDC_W, NDC_H, NDC_F) if ndc else None)


def _t(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.mark.gpu
def test_ndc_ray_kernel_matches_oracle():
    """pob_ndc_rays on camera slabs and on explicit rays (non-unit directions, arbitrary view directions)"""
    from plenoctree_b200.octree.renderer import make_camera
    r = _renderer(device_tree("n2_d8_sh16"), 1e-3, 1.0)
    worst, rs = 0, np.random.RandomState(8)
    for c2w in ndc_cameras():
        want = ON.ndc_persp_rays(c2w, NDC_W, NDC_H, NDC_F)
        cam = make_camera(c2w, NDC_W, NDC_H, NDC_F)
        for row0, nrows in ((0, NDC_H), (5, 7), (NDC_H - 1, 1)):
            got = r._ndc_rays(None, cam, row0, nrows)
            sl = slice(row0 * NDC_W, (row0 + nrows) * NDC_W)
            for g, wnt in zip(got, want):
                worst = max(worst, _ulps(g.cpu().numpy(), wnt[sl]))
        o, d, _ = OO.persp_rays(c2w, NDC_W, NDC_H, NDC_F)
        d = (d * rs.uniform(0.3, 3.0, (d.shape[0], 1))).astype(f32)
        v = rs.normal(size=d.shape).astype(f32)
        got = r._ndc_rays((_t(o), _t(d), _t(v)), None, 0, 0)
        for g, wnt in zip(got, ON.ndc_rays(o, d, v, NDC_F, NDC_W, NDC_H)):
            worst = max(worst, _ulps(g.cpu().numpy(), wnt))
    _record("ndc_rays", {"max_ulps": worst, "allow": NDC_RAY_ULPS})
    assert worst <= NDC_RAY_ULPS, worst


def _march_names():
    from tests.support.octree_scenes import NAMES
    return NAMES


@pytest.mark.gpu
@pytest.mark.parametrize("name", _march_names())
def test_render_backward_depth_on_ndc_rays(name):
    """render_persp / forward in NDC: the oracle's leaf path (visit and hit counters), rgb and the gradient within
    test_octree_march.py's fp64 bars; depth and acc bit-identical to the explicit-ray entry point on the NDC rays"""
    import torch
    from plenoctree_b200.octree import Rays
    from tests.support.octree_refs import GRAD_ALLOW, RGB_ALLOW, _check_grad, bwd64, fwd64
    from tests.support.octree_scenes import world
    otree = world(name)["otree"]
    tree = device_tree(name)
    step, bg = 1e-3, 1.0
    r, plain = _renderer(tree, step, bg), _renderer(tree, step, bg, ndc=False)
    rec, hits = {}, 0
    for i, c2w in enumerate(ndc_cameras()):
        o, d, v = ON.ndc_persp_rays(c2w, NDC_W, NDC_H, NDC_F)
        vis = OO.march_visits(otree, o, d, v, step, bg)
        f = fwd64(otree, vis, v, bg)
        cnt = torch.zeros(2, dtype=torch.int64, device="cuda")
        with torch.no_grad():
            img = r.render_persp(c2w, NDC_W, NDC_H, NDC_F, counters=cnt)
            ow, dw, vw = OO.persp_rays(c2w, NDC_W, NDC_H, NDC_F)
            fwd = r.forward(Rays(_t(ow), _t(dw), _t(vw)))
            full = r.render_persp(c2w, NDC_W, NDC_H, NDC_F, return_depth=True)
            want = plain.forward(Rays(_t(o), _t(d), _t(v)), return_depth=True)
            slab = r.render_persp(c2w, NDC_W, NDC_H, NDC_F, rows=(7, 9), return_depth=True)
        cnt = cnt.cpu().numpy()
        assert cnt[0] == vis["visits"].sum() and cnt[1] == vis["hits"].sum(), (i, cnt)
        hits += int(cnt[1])
        err = np.abs(img.cpu().numpy().reshape(-1, 3).astype(f64) - f["rgb"]) / (U24 * f["U"])
        assert err.max() <= RGB_ALLOW, (i, float(err.max()))
        assert torch.equal(fwd, img.reshape(-1, 3))
        for k in range(3):
            assert torch.equal(full[k].reshape(want[k].shape), want[k]), k
            assert torch.equal(slab[k], full[k][7:16]), k
        g = np.random.RandomState(5 + i).normal(size=(o.shape[0], 3)).astype(f32)
        uniq, grad, unit = bwd64(otree, vis, f, g.astype(f64), np.zeros_like(f["U"]), bg)
        tree.data.requires_grad_(True)
        tree.data.grad = None
        (r.render_persp(c2w, NDC_W, NDC_H, NDC_F) * _t(g.reshape(NDC_H, NDC_W, 3))).sum().backward()
        got = tree.data.grad.reshape(-1, otree.data_dim)[: otree.n_internal * otree.N ** 3].cpu().numpy()
        tree.data.grad = None
        tree.data.requires_grad_(False)
        rec[f"camera{i}"] = dict(rgb_err_units=float(err.max()), visits=int(cnt[0]), hits=int(cnt[1]),
                                 grad_err_units=_check_grad(name, otree, got, uniq, grad, unit, GRAD_ALLOW, "ndc"))
    _record(f"render_{name}", dict(rec, rgb_allow=RGB_ALLOW, grad_allow=GRAD_ALLOW))
    assert hits > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name,i", [("n2_d8_sh16", 1), ("chain_d26_rgba", 0)])
def test_compressed_tree_renders_ndc_bit_identical_to_decompressed(name, i):
    import torch
    from plenoctree_b200.octree import Rays
    from tests.support.octree_scenes import _pair
    q, ref = _pair(name, i)
    rq, rf = _renderer(q, 1e-3, 1.0), _renderer(ref, 1e-3, 1.0)
    contributing = 0
    for c2w in ndc_cameras():
        ow, dw, vw = OO.persp_rays(c2w, NDC_W, NDC_H, NDC_F)
        with torch.no_grad():
            for fast in (False, True):
                cq, cf = (torch.zeros(2, dtype=torch.int64, device="cuda") for _ in range(2))
                a = rq.render_persp(c2w, NDC_W, NDC_H, NDC_F, fast=fast, counters=cq, return_depth=True)
                b = rf.render_persp(c2w, NDC_W, NDC_H, NDC_F, fast=fast, counters=cf, return_depth=True)
                for x, y in zip(a, b):
                    assert torch.equal(x, y), fast
                assert torch.equal(cq, cf)
                assert torch.equal(rq.forward(Rays(_t(ow), _t(dw), _t(vw)), fast=fast), b[0].reshape(-1, 3))
                contributing += int(cq[1])
    assert contributing > 100


@pytest.mark.gpu
@pytest.mark.parametrize("name", _march_names())
def test_train_pass_ndc_matches_fp64(name):
    """the fused NDC training pass: its image equals render_persp in NDC bit for bit; its gradient is exactly 0 off
    the oracle's leaf path and within test_octree_march.py's training bar on it; the squared error within its bar"""
    import torch
    from tests.support.octree_refs import RGB_ALLOW, SQ_ALLOW, TRAIN_ALLOW, _check_grad, bwd64, fwd64
    from tests.support.octree_scenes import world
    otree = world(name)["otree"]
    tree = device_tree(name)
    step = 1e-3
    r = _renderer(tree, step, 1.0)
    rec = {}
    for i, c2w in enumerate(ndc_cameras()):
        o, d, v = ON.ndc_persp_rays(c2w, NDC_W, NDC_H, NDC_F)
        vis = OO.march_visits(otree, o, d, v, step, 1.0)
        gt = np.random.RandomState(4 + i).uniform(0, 1, size=(NDC_H, NDC_W, 3)).astype(f32)
        tree.grad = None
        sq, img = r.train_persp(c2w, torch.from_numpy(gt), NDC_W, NDC_H, NDC_F, want_image=True)
        got = tree.grad_buffer().reshape(-1, otree.data_dim)[: otree.n_internal * otree.N ** 3].cpu().numpy()
        with torch.no_grad():
            assert torch.equal(img, r.render_persp(c2w, NDC_W, NDC_H, NDC_F))
        im = img.cpu().numpy().reshape(-1, 3).astype(f64)
        f = fwd64(otree, vis, v, 1.0)
        scale = f64(f32(1.0 / (NDC_H * NDC_W * 3)))
        gt = gt.reshape(-1, 3).astype(f64)
        inside = (im >= 0) & (im <= 1)
        diff = np.clip(f["rgb"], 0, 1) - gt
        g = np.where(inside, scale * 2.0 * diff, 0.0)
        gerr = np.where(inside, 2.0 * scale * RGB_ALLOW * f["U"], 0.0)
        uniq, grad, unit = bwd64(otree, vis, f, g, gerr, 1.0)
        sq_unit = U24 * float((2 * np.abs(diff) * f["U"] + 16 * diff ** 2).sum())
        sq_err = abs(float(sq.item()) - float((diff ** 2).sum())) / sq_unit
        rec[f"camera{i}"] = dict(grad_err_units=_check_grad(name, otree, got, uniq, grad, unit, TRAIN_ALLOW, "train"),
                                 sq_err_units=sq_err, touched_leaves=int(uniq.size))
        assert sq_err <= SQ_ALLOW, sq_err
        tree.grad = None
    _record(f"train_{name}", dict(rec, train_allow=TRAIN_ALLOW, sq_allow=SQ_ALLOW))


def _grid_ndc_march(reso, cams):
    """test_grid_weights.march with the cameras' NDC rays"""
    from tests.support.grid_weights import STEP, geometry, merge, per_voxel, shade64, sigma_host
    off, inv = geometry()
    parts, visits = [], 0
    for c2w in cams:
        o, d, _ = ON.ndc_persp_rays(c2w, NDC_W, NDC_H, NDC_F)
        vis = OO.grid_march_visits(reso, o, d, off, inv, STEP)
        s = shade64(vis, sigma_host(vis["voxel"], reso))
        h = s["hit"]
        parts.append(per_voxel(vis["voxel"][h], s["w"][h], s["unit"][h], s["pre"][h]))
        visits += int(vis["ray"].size)
    return merge(parts), visits


@pytest.mark.gpu
@pytest.mark.parametrize("reso", [96, 512])
def test_grid_weights_ndc_exact_path_and_values(reso):
    """pob_grid_weight_render_ndc (all cameras in one launch) and calculate_grid_weights(ndc=...): the voxels hit are
    the oracle's, the per-voxel maximum weight within test_grid_weights.py's fp64 bar"""
    import torch
    from plenoctree_b200.octree.extraction import calculate_grid_weights
    from plenoctree_b200.octree.renderer import NDCConfig
    from tests.support.grid_weights import STEP, WEIGHT_ALLOW, check_launch, device_sigma, geometry, take
    from tests.support.grid_weights import cam_rows
    from plenoctree_b200 import _lib
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    import ctypes
    cams = ndc_cameras()
    ref, visits = _grid_ndc_march(reso, cams)
    off, inv = geometry()
    n = reso ** 3
    wmax = torch.zeros(n, dtype=torch.float32, device="cuda")
    hit = torch.zeros(n, dtype=torch.uint8, device="cuda")
    rows = torch.from_numpy(cam_rows([(c, NDC_W, NDC_H, NDC_F) for c in cams])).cuda()
    o = _lib.OctreeOpts()
    o.step_size, o.background_brightness, o.sigma_thresh, o.stop_thresh = STEP, 1.0, 0.0, 0.0
    nd = _lib.Ndc(NDC_W, NDC_H, NDC_F)
    check(lib.pob_grid_weight_render_ndc(ptr(device_sigma(reso)), reso, ptr(rows), len(cams), NDC_W, NDC_H,
                                         (ctypes.c_float * 3)(*map(float, off)), (ctypes.c_float * 3)(*map(float, inv)),
                                         ctypes.byref(o), ctypes.byref(nd), ptr(wmax), ptr(hit), stream_ptr()))
    torch.cuda.synchronize()
    kw, vw, kh = take(wmax, hit)
    worst, margin, masked = check_launch(ref, kw, vw, kh, "ndc")
    assert kh.size > 500 and masked > 50
    ds = types.SimpleNamespace(camtoworlds=np.stack(cams), w=NDC_W, h=NDC_H, focal=NDC_F)
    gw = calculate_grid_weights(ds, device_sigma(reso), reso, torch.from_numpy(inv), torch.from_numpy(off),
                                step_size=STEP, ndc=NDCConfig(NDC_W, NDC_H, NDC_F)).reshape(-1)
    assert torch.equal(gw.nonzero().reshape(-1).cpu(), torch.from_numpy(kw))
    assert np.array_equal(gw[gw != 0].cpu().numpy().view(np.int32), vw.view(np.int32))
    _record(f"grid_{reso}", dict(weight_err_units=worst, allow=WEIGHT_ALLOW, mask_margin_voxels=margin,
                                 masked_voxels=masked, hit_voxels=int(kh.size), visits=visits))


# ---------------------------------------------------------------------------------------------------------
# end to end: nerf_sh.train -> octree.extraction --z_min/--z_max -> octree.optimization -> octree.evaluation
# ---------------------------------------------------------------------------------------------------------
def _psnr(a, b):
    return float(-10.0 * np.log10(float(((a.clamp(0, 1) - b.clamp(0, 1)) ** 2).mean())))


def _scene(o, d, v):
    """uint8 image of a forward-facing scene in the recentred LLFF world frame: a checkered card at z = -2 in front of a
    striped wall at z = -5, both opaque, with a view-dependent tint that follows the world view direction's x (so that
    the SH colours the model learns depend on the view direction)"""
    o, d, v = (np.asarray(a, f64) for a in (o, d, v))
    t_card = (-2.0 - o[..., 2]) / d[..., 2]
    p = o + t_card[..., None] * d
    card = (np.abs(p[..., 0]) < 0.6) & (np.abs(p[..., 1]) < 0.4)
    t = np.where(card, t_card, (-5.0 - o[..., 2]) / d[..., 2])
    p = o + t[..., None] * d
    checker = (np.floor(p[..., 0] / 0.2) + np.floor(p[..., 1] / 0.2)) % 2
    stripes = 0.5 + 0.5 * np.sin(4.0 * p[..., 0])
    rgb = np.where(card[..., None], np.stack([0.2 + 0.6 * checker, 0.7 - 0.4 * checker, 0.3 + 0.0 * checker], -1),
                   np.stack([0.3 + 0.4 * stripes, 0.5 + 0.0 * stripes, 0.8 - 0.5 * stripes], -1))
    rgb = rgb + 0.5 * v[..., :1] * np.array([1.0, -0.6, 0.4])
    return (np.clip(rgb, 0.0, 1.0) * 255 + 0.5).astype(np.uint8)


@pytest.mark.gpu
def test_llff_end_to_end(tmp_path):
    """the CLI chain in NDC on a synthetic LLFF scene: the raw tree renders the held-out views like the model (and not
    without the NDC transform or with NDC view directions); optimisation raises the evaluated PSNR of the tree.

    The tree's box spans x, y in [-2.5, 2.5]: NDC x and y reach past +-1 wherever a camera sees beyond the frustum of
    the reference pose (the average camera), and the scene's cameras move and turn enough for that.  A tree confined
    to [-1, 1]^3 leaves that content out and renders a third of those pixels as background."""
    import torch
    from plenoctree_b200.nerf import datasets as D, flags as F
    from plenoctree_b200.nerf.models import Rays
    from plenoctree_b200.nerf.rays import generate_rays
    from plenoctree_b200.nerf.utils import render_image
    from plenoctree_b200.nerf_sh import train as TR
    from plenoctree_b200.octree import N3Tree, VolumeRenderer, evaluation as EV, extraction as EX
    from plenoctree_b200.octree import Rays as TreeRays
    from plenoctree_b200.octree import optimization as OPT
    from plenoctree_b200.octree.renderer import make_camera, scene_ndc
    from tests.golden.make_golden import synthetic_llff, write_llff_scene
    n, h, w = 24, 30, 40
    images, pb = synthetic_llff(21, n, h, w, 36.0)
    data_dir, train_dir = str(tmp_path / "scene"), str(tmp_path / "ckpt")
    write_llff_scene(data_dir, images, pb)
    largs = types.SimpleNamespace(data_dir=data_dir, factor=0, spherify=False, llffhold=4, batch_size=1024,
                                  image_batching=True, dataset="llff", render_path=False, white_bkgd=True)
    i_test = np.arange(n)[::4]
    for split, idx in (("test", i_test), ("train", np.setdiff1d(np.arange(n), i_test))):
        ds = D.get_dataset(split, largs, device="cpu")
        world = generate_rays(w, h, ds.focal, ds.camtoworlds)
        for j, k in enumerate(idx):
            images[k] = _scene(world.origins[j], world.directions[j], world.viewdirs[j])
    write_llff_scene(data_dir, images, pb)
    (tmp_path / "llff.yaml").write_text(
        "dataset: llff\nfactor: 0\nllffhold: 4\nspherify: false\nnear: 0.0\nfar: 1.0\nlindisp: false\n"
        "num_coarse_samples: 64\nnum_fine_samples: 128\nuse_viewdirs: false\nwhite_bkgd: true\nbatch_size: 1024\n"
        "sh_deg: 3\nrandomized: true\nmax_steps: 1000\n")
    EX._define_cli_flags()
    OPT._define_cli_flags()
    EV._define_cli_flags()
    F.define_flags()
    FLAGS = F.FLAGS
    if not FLAGS.is_parsed():
        FLAGS.mark_as_parsed()
    new = dict(train_dir=train_dir, data_dir=data_dir, config=str(tmp_path / "llff"), save_every=1000, print_every=100,
               render_every=0, sparsity_npoints=0, lr_init=2e-3, lr_final=2e-4, chunk=4096, noise_std=None,
               image_batching=True, is_jaxnerf_ckpt=True, init_grid_depth=7, samples_per_cell=8,
               masking_mode="weight", weight_thresh=1e-3, renderer_step_size=1e-3, radius="2.5 2.5 1",
               center="0 0 0",
               z_min=-0.98, z_max=0.98, eval=False, output=str(tmp_path / "tree.npz"), input=str(tmp_path / "tree.npz"),
               render_interval=0, val_interval=1, num_epochs=4, lr=1e4, continue_on_decrease=True, nosave=False,
               write_vid=None, write_images=None, write_disp=None, split_train=None, no_early_stop=True)
    yaml_keys = ["dataset", "factor", "llffhold", "spherify", "near", "far", "lindisp", "num_coarse_samples",
                 "num_fine_samples", "use_viewdirs", "white_bkgd", "batch_size", "sh_deg", "randomized", "max_steps"]
    old = {k: getattr(FLAGS, k) for k in list(new) + yaml_keys}
    try:
        for k, v in new.items():
            setattr(FLAGS, k, v)
        model, state = TR.main(None)
        assert state.step == 1000
        EX.main(None)
        tree = N3Tree.load(FLAGS.output, map_location="cuda")
        test = D.get_dataset("test", FLAGS, device="cuda")
        ndc = scene_ndc(FLAGS, test.w, test.h, test.focal)
        assert ndc is not None
        r = VolumeRenderer(tree, step_size=FLAGS.renderer_step_size, ndc=ndc)
        plain = VolumeRenderer(tree, step_size=FLAGS.renderer_step_size)
        psnr = {"ndc": [], "ndc_viewdirs": [], "world_rays": [], "gt": []}
        with torch.no_grad():
            for j in range(test.size):
                c2w = test.camtoworlds[j]
                nerf_img = render_image(model, Rays(*[x[j] for x in test.rays_np]))[0]
                img = r.render_persp(c2w, test.w, test.h, test.focal)
                psnr["ndc"].append(_psnr(img, nerf_img))
                psnr["gt"].append(_psnr(img, torch.from_numpy(test.images[j]).cuda()))
                o, d, _ = r._ndc_rays(None, make_camera(c2w, test.w, test.h, test.focal), 0, test.h)
                bad = plain.forward(TreeRays(o, d, d)).reshape(img.shape)
                psnr["ndc_viewdirs"].append(_psnr(bad, nerf_img))
                psnr["world_rays"].append(_psnr(plain.render_persp(c2w, test.w, test.h, test.focal), nerf_img))
        mean = {k: float(np.mean(v)) for k, v in psnr.items()}
        _record("llff_raw_tree", dict(psnr_vs_nerf=mean))
        p_raw, _ = EV.main(None)
        FLAGS.output = str(tmp_path / "tree_opt.npz")
        OPT.main(None)
        FLAGS.input = FLAGS.output
        p_opt, _ = EV.main(None)
        _record("llff_end_to_end", dict(psnr_vs_nerf=mean, eval_psnr_raw=p_raw, eval_psnr_optimized=p_opt))
        assert mean["ndc"] >= PSNR_BOUND, mean
        assert mean["ndc_viewdirs"] < PSNR_BOUND and mean["world_rays"] < PSNR_BOUND, mean
        assert p_opt > p_raw, (p_raw, p_opt)
    finally:
        for k, v in old.items():
            setattr(FLAGS, k, v)

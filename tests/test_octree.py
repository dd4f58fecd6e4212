"""PlenOctree side (SURVEY §8 rows a13-middle, a15): oracle self-checks on CPU, and GPU parity of the CUDA
octree kernels (csrc/octree.cu) against the oracle through the C ABI.

svox is absent from the reference tree (parity unpinned, see oracle/octree_oracle.py); what is pinned:
  * the oracle's backward equals the numerical derivative of its forward, and a uniform medium gives the closed form;
  * the CUDA kernels equal the oracle (tree topology and leaf lookup bit-exact; colours / gradients within the
    float32 tolerances written below).
"""
import functools
import os

import numpy as np
import pytest

from oracle import octree_oracle as OO
from tests.support.octree_scenes import assert_device_tree_build_matches, look_at_pose, make_tree, to_device_tree
from tests.support.records import record


# float32 march, identical operation order, differing only in expf ulps and the order of the K-term dot products
TOL_RGB = 2e-5        # absolute, colours in [0,1]
TOL_GRAD_REL = 2e-4   # relative to the largest gradient entry


_record = functools.partial(record, "parity_octree.json")


def random_rays(seed, n, radius=1.3):
    rs = np.random.RandomState(seed)
    o = rs.normal(size=(n, 3))
    o = (o / np.linalg.norm(o, axis=1, keepdims=True) * 3.0).astype(np.float32)
    tgt = rs.uniform(-0.7 * radius, 0.7 * radius, size=(n, 3)).astype(np.float32)
    d = tgt - o
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    d[: n // 8] *= -1.0  # some rays miss the volume
    return o, d, d.copy()


# ---------------------------------------------------------------------------------------------------------
# CPU: the oracle checks itself
# ---------------------------------------------------------------------------------------------------------
def test_oracle_uniform_medium_closed_form():
    tree = OO.N3Tree(N=2, data_dim=4, depth_limit=4, radius=1.0, center=(0, 0, 0), data_format="RGBA")
    tree.data[0, ..., :3] = np.array([0.3, -0.2, 1.1], dtype=np.float32)
    tree.data[0, ..., 3] = 1.7
    o = np.array([[-3.0, 0.2, 0.1]], dtype=np.float32)
    d = np.array([[1.0, 0.0, 0.0]], dtype=np.float32)
    step = 1e-3
    rgb, visits, hits = OO.volume_render(tree, o, d, d, step_size=step, return_steps=True)
    # world path length 2 (cube side) = 1 in tree units.  Each visit advances by (distance to the cell exit +
    # step_size); the overshoot shortens the next cell's segment, so only the LAST visit's step_size adds to the
    # integrated length.  delta_scale = 1/|d * invradius| = 2 converts tree units back to world units.
    length = 2.0 + step * 2.0
    T = np.exp(-1.7 * length)
    col = 1.0 / (1.0 + np.exp(-np.array([0.3, -0.2, 1.1])))
    want = (1.0 - T) * col + T * 1.0
    assert visits[0] == 2 and hits[0] == 2
    np.testing.assert_allclose(rgb[0], want, atol=2e-5)


@pytest.mark.parametrize("fmt", ["RGBA", "SH9"])
def test_oracle_backward_is_derivative_of_forward(fmt):
    tree = make_tree(3, 2, fmt, density=0.5)
    o, d, v = random_rays(4, 24)
    rs = np.random.RandomState(5)
    g = rs.normal(size=(24, 3)).astype(np.float32)
    grad = OO.volume_render_backward(tree, o, d, v, g, step_size=1e-3)
    n = tree.n_internal
    flat = tree.data[:n].reshape(-1)
    gflat = grad.reshape(-1)
    nz = np.nonzero(np.abs(gflat) > 0.05 * np.abs(gflat).max())[0]
    assert nz.size > 10
    picks = nz[rs.permutation(nz.size)[:12]]
    eps = 2e-2
    for p in picks:
        keep = flat[p]
        flat[p] = keep + eps
        fp = (OO.volume_render(tree, o, d, v, step_size=1e-3).astype(np.float64) * g).sum()
        flat[p] = keep - eps
        fm = (OO.volume_render(tree, o, d, v, step_size=1e-3).astype(np.float64) * g).sum()
        flat[p] = keep
        num = (fp - fm) / (2 * eps)
        assert abs(num - gflat[p]) <= 0.03 * abs(gflat[p]) + 1e-4, (p, num, gflat[p])


def test_oracle_tree_build_and_io(tmp_path):
    rs = np.random.RandomState(0)
    L = 3
    reso = 2 ** (L + 1)
    mask = rs.rand(reso, reso, reso) < 0.1
    tree, grid = OO.build_tree_from_grid(mask, L, 1.5, [0, 0, 0], 49, "SH16", refine_chunk=100)
    assert tree.max_depth == L
    node, ijk, cube, _ = tree.query(grid)
    assert (tree.parent_depth[node, 1] == L).all() and (cube == reso).all()
    # every internal node's parent link is consistent with child offsets
    n = tree.n_internal
    pk = tree.parent_depth[1:n, 0].astype(np.int64)
    assert (tree.child.reshape(-1)[pk] + pk // 8 == np.arange(1, n)).all()
    lv = tree.leaves()
    deep = lv[tree.leaf_depths(lv) == L]
    u = rs.rand(deep.shape[0], 4, 3).astype(np.float32)
    pts = tree.sample(deep, 4, u).reshape(-1, 3)
    n2, i2, _, _ = tree.query(pts)
    assert (n2.reshape(-1, 4) == deep[:, :1]).all() and (i2.reshape(-1, 4, 3) == deep[:, None, 1:]).all()
    st = tree.state()
    np.savez(tmp_path / "t.npz", **st)
    z = np.load(tmp_path / "t.npz")
    for k in ("data", "child", "parent_depth", "n_internal", "n_free", "depth_limit", "geom_resize_fact",
              "invradius3", "offset", "data_dim", "data_format"):
        assert k in z.files
    assert z["data"].dtype == np.float16 and z["data"].shape == (n, 2, 2, 2, 49)


def test_oracle_grid_weight_single_voxel():
    reso = 8
    grid = np.zeros((reso, reso, reso), dtype=np.float32)
    grid[4, 4, 4] = 5.0
    off = np.array([0.5, 0.5, 0.5], dtype=np.float32)
    inv = np.array([0.5, 0.5, 0.5], dtype=np.float32)  # radius 1, centre 0
    c = (4 + 0.5) / reso * 2 - 1
    o = np.array([[-3.0, c, c]], dtype=np.float32)
    d = np.array([[1.0, 0.0, 0.0]], dtype=np.float32)
    gw = OO.grid_weight_render(grid, o, d, off, inv, step_size=1e-4)
    # the ray enters voxel 4 already step_size past its face, so (exit distance + step_size) is one cell exactly
    want = 1.0 - np.exp(-5.0 * (2.0 / reso))
    assert abs(gw[4, 4, 4] - want) < 1e-5
    assert (np.delete(gw.reshape(-1), (4 * 8 + 4) * 8 + 4) == 0).all()


def test_oracle_forward_agrees_with_reference_compositing_quadrature():
    """Ties the (unpinned) octree oracle to reference arithmetic that IS restated line by line elsewhere: the tree's
    piecewise-constant field, sampled densely along each ray and composited with the reference's
    volumetric_rendering (nerf_sh/nerf/model_utils.py:176-222) and eval_sh (nerf_sh/nerf/sh.py:54-109, golden-pinned),
    must converge to what the per-leaf exact march renders (same sigmoid-of-SH colour, same white background)."""
    import torch
    from oracle import nerf_sh_oracle as O
    tree = make_tree(5, 3, "SH9", density=0.4, sigma_scale=4.0)
    o, d, v = random_rays(6, 48)
    o, d, v = o[8:], d[8:], v[8:]                       # keep the rays that hit the volume
    want = OO.volume_render(tree, o, d, v, step_size=1e-6)
    n = 8192
    # entry / exit of the bounding box in world units along the (unit) direction
    ot, dt, ds, invd, tmin, tmax = OO._setup(tree.offset, tree.invradius, o, d)
    z = (tmin[:, None] + (tmax - tmin)[:, None] * (np.arange(n, dtype=np.float64)[None, :] + 0.5) / n) * ds[:, None]
    pts = o[:, None, :] + z[..., None] * d[:, None, :]
    node, ijk, _, _ = tree.query(pts.reshape(-1, 3).astype(np.float32))
    val = tree.data[node, ijk[:, 0], ijk[:, 1], ijk[:, 2]].reshape(len(o), n, -1)
    sigma = torch.from_numpy(val[..., -1:].copy())
    sigma[:, -1] = 0.0                                  # the reference gives the last sample an infinite interval
    sh = torch.from_numpy(val[..., :-1].reshape(len(o), n, 3, 9).copy())
    rgb = torch.sigmoid(O.eval_sh(2, sh, torch.from_numpy(v)[:, None, :]))
    comp, _, _, _ = O.volumetric_rendering(rgb.double(), sigma.double(), torch.from_numpy(z), torch.from_numpy(d).double(), True)
    err = np.abs(comp.numpy() - want)
    psnr = -10 * np.log10((err ** 2).mean())
    # measured: 1024 samples/ray 1.7e-3 (65 dB), 8192 samples/ray 2.7e-4 (82.7 dB): first-order convergence
    assert err.max() < 1e-3 and psnr > 70, (err.max(), psnr)
    assert np.abs(want - 1.0).max() > 0.2               # not an empty scene


# ---------------------------------------------------------------------------------------------------------
# GPU parity
# ---------------------------------------------------------------------------------------------------------


def test_extraction_sequence_matches_executed_reference(golden_dir):
    """octree/extraction.py's own control flow — auto_scale, step1 (sigma mask), step2, relu — was EXECUTED
    (tests/golden/make_golden.py ref_extraction) with the reference's torch NeRF-SH twin and an svox stand-in
    backed by this oracle's N3Tree.  The oracle pieces the GPU tests use as the expected value
    (`build_tree_from_grid`, leaf order, `sample`, the cell mean + relu) must reproduce that run: same topology,
    same leaf data; the package's bounding-box helper must reproduce auto_scale."""
    import torch
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.octree import extraction as E
    z = np.load(os.path.join(golden_dir, "ref_extraction.npz"))
    sh_deg, L, S = int(z["sh_deg"]), int(z["init_grid_depth"]), int(z["samples_per_cell"])
    flat_f = O.init_flat_params(sh_deg, int(z["seed"]) + 1, bias_scale=0.05)            # fine MLP: what eval_points_raw uses
    assert abs(float(O.init_flat_params(sh_deg, int(z["seed"]), bias_scale=0.05).astype(np.float64).sum())
               - float(z["flat_c_checksum"])) < 1e-6
    params = O.unflatten(flat_f, sh_deg)
    center, radius = z["center"].astype(np.float32), z["radius"].astype(np.float32)

    def sigma_grid(reso, off, inv):
        arr = ((np.arange(reso, dtype=np.float32) + np.float32(0.5)) / np.float32(reso)).astype(np.float32)
        ax = [((arr - off[a]) / inv[a]).astype(np.float32) for a in range(3)]
        pts = np.stack(np.meshgrid(*ax, indexing="ij"), axis=-1).reshape(-1, 3)
        with torch.no_grad():
            return O.eval_points_raw(params, torch.from_numpy(pts))[1].numpy().reshape(-1)
    # ---- auto_scale (reso = 2^L) through the package's helper ----
    inv = (np.float32(0.5) / radius).astype(np.float32)
    off = (np.float32(0.5) * (np.float32(1.0) - center / radius)).astype(np.float32)
    sig0 = sigma_grid(2 ** L, off, inv)
    c, r = E._bbox_of_dense(torch.from_numpy(sig0), float(z["scale_alpha_thresh"]), 2 ** L, torch.from_numpy(off),
                            torch.from_numpy(inv))
    assert np.allclose(c, z["autoscale_center"], atol=1e-6) and np.allclose(r, z["autoscale_radius"], atol=1e-6)
    assert not np.allclose(r, radius)                                                   # the box did shrink
    # ---- step 1: topology ----
    reso = 2 ** (L + 1)
    sig = sigma_grid(reso, off, inv)
    thresh = -np.log(1.0 - float(z["alpha_thresh"])) / (2.0 / reso)
    assert np.abs(sig - thresh).min() > 1e-4                 # no voxel close enough to the threshold to flip
    mask = sig >= thresh
    tree, _ = OO.build_tree_from_grid(mask, L, radius, center, 3 * (sh_deg + 1) ** 2 + 1, "SH16")
    n = int(z["n_internal"])
    assert tree.n_internal == n == int(z["n_after_step1"]) and 0.2 < mask.mean() < 0.5
    assert np.array_equal(tree.child[:n], z["child"]) and np.array_equal(tree.parent_depth[:n], z["parent_depth"])
    # ---- step 2: leaves at max depth in leaf order, S samples each (the recorded uniforms), mean, relu on sigma ----
    lv = tree.leaves()
    deep = np.nonzero(tree.leaf_depths(lv) == L)[0]
    assert z["uniforms"].shape == (deep.size, S, 3)
    pts = tree.sample(lv[deep], S, z["uniforms"]).reshape(-1, 3)
    with torch.no_grad():
        rgb, s = O.eval_points_raw(params, torch.from_numpy(pts))
    want = torch.cat([rgb, s], dim=-1).reshape(-1, S, tree.data_dim).mean(dim=1).numpy()
    want[:, -1] = np.maximum(want[:, -1], 0.0)
    ref = z["data"].reshape(-1, tree.data_dim)
    at = tree.pack_index(lv[deep, 0], lv[deep, 1:])
    assert np.abs(ref[at] - want).max() < 2e-5 * np.abs(want).max()
    rest = np.ones(ref.shape[0], dtype=bool)
    rest[at] = False
    assert not ref[rest].any()                                # coarser leaves and internal cells stay empty


def test_optimization_loop_matches_executed_reference(golden_dir):
    """octree/optimization.py `main` was EXECUTED (make_golden.py ref_optimization: the reference's Blender loader,
    render -> clamp -> MSE -> backward -> torch.optim.SGD per image, validation PSNR per epoch, best-model save) over
    an svox stand-in whose renderer is this oracle's march wrapped in an autograd Function.  Replaying the run with
    the oracle pieces the GPU tests use as expected values (`mse_and_grad_out`, `sgd_step`, sequential per-image
    updates) must give the same PSNR curves and the same saved tree."""
    z = np.load(os.path.join(golden_dir, "ref_optimization.npz"))
    H, W, focal, step, lr = int(z["H"]), int(z["W"]), float(z["focal"]), float(z["step_size"]), float(z["lr"])
    n = z["child"].shape[0]
    tree = OO.N3Tree(N=2, data_dim=z["data0"].shape[-1], depth_limit=4, init_reserve=n, data_format="SH4")
    tree.child, tree.parent_depth, tree.n_internal = z["child"].copy(), z["parent_depth"].copy(), n
    tree.invradius, tree.offset = z["invradius"].astype(np.float32), z["offset"].astype(np.float32)
    tree.data = z["data0"].astype(np.float32).copy()
    psnr = lambda mse: -10.0 * np.log(mse) / np.log(10.0)

    def validate():
        tot = 0.0
        for c2w, gt in zip(z["val_c2w"], z["val_gt"]):
            im = OO.volume_render(tree, *OO.persp_rays(c2w, W, H, focal), step_size=step).reshape(H, W, 3)
            tot += psnr(float(((np.clip(im, 0.0, 1.0) - gt).astype(np.float32) ** 2).mean()))
        return tot / len(z["val_c2w"])
    assert abs(validate() - float(z["initial_val_psnr"])) < 2e-4
    best, best_data = float(z["initial_val_psnr"]), None
    for ep in range(int(z["epochs"])):
        tot = 0.0
        for c2w, gt in zip(z["train_c2w"], z["train_gt"]):
            rays = OO.persp_rays(c2w, W, H, focal)
            im = OO.volume_render(tree, *rays, step_size=step)
            mse, g = OO.mse_and_grad_out(im.reshape(H, W, 3), gt)
            grad = OO.volume_render_backward(tree, *rays, g.reshape(-1, 3), step_size=step)
            tree.data = OO.sgd_step(tree.data, grad, lr)
            tot += psnr(mse)
        assert abs(tot / len(z["train_c2w"]) - float(z["train_psnr"][ep])) < 2e-4, ep
        v = validate()
        assert abs(v - float(z["val_psnr"][ep])) < 2e-4, ep
        if v > best:
            best, best_data = v, tree.data.copy()
    assert z["train_psnr"][-1] > z["train_psnr"][0] + 0.5 and best_data is not None          # it did learn
    assert np.abs(best_data - z["data_best"]).max() < 2e-5 * np.abs(z["data_best"]).max()


@pytest.mark.gpu
def test_query_and_tree_build_bit_exact():
    rs = np.random.RandomState(1)
    L = 4
    reso = 2 ** (L + 1)
    mask = rs.rand(reso, reso, reso) < 0.08
    otree, grid = OO.build_tree_from_grid(mask, L, [1.5, 1.2, 1.0], [0.1, 0.0, -0.2], 49, "SH16", refine_chunk=700)
    refines = [grid] * (L - 1) + [grid[j:j + 700] for j in range(0, grid.shape[0], 700)]
    assert_device_tree_build_matches(otree, refines, [1.5, 1.2, 1.0], [0.1, 0.0, -0.2], rs)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,depth", [("SH16", 4), ("SH25", 3), ("RGBA", 3), ("SH4", 3), ("SH9", 2), ("SH1", 2)])
def test_render_rays_matches_oracle(fmt, depth):
    import torch
    from plenoctree_b200.octree import Rays, VolumeRenderer
    otree = make_tree(10 + depth, depth, fmt)
    tree = to_device_tree(otree)
    o, d, v = random_rays(7, 333)
    r = VolumeRenderer(tree, step_size=1e-3)
    worst = 0.0
    for fast in (False, True):
        th = 1e-2 if fast else 0.0
        want = OO.volume_render(otree, o, d, v, step_size=1e-3, sigma_thresh=th, stop_thresh=th)
        with torch.no_grad():
            got = r.forward(Rays(torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(v)), fast=fast).cpu().numpy()
        err = float(np.abs(got - want).max())
        worst = max(worst, err)
        assert err < TOL_RGB, (fmt, fast, err)
    assert (np.abs(want - 1.0).max(axis=1) > 0.05).sum() > 100  # the scene is not empty
    _record(f"render_rays_{fmt}", {"max_abs_err": worst, "tol": TOL_RGB, "rays": 333})


@pytest.mark.gpu
def test_render_persp_matches_oracle_and_slabs():
    import torch
    from plenoctree_b200.octree import VolumeRenderer
    otree = make_tree(21, 4, "SH16")
    tree = to_device_tree(otree)
    c2w = look_at_pose(2)
    W, H, fx = 50, 37, 60.0
    o, d, v = OO.persp_rays(c2w, W, H, fx)
    want = OO.volume_render(otree, o, d, v, step_size=1e-4).reshape(H, W, 3)
    r = VolumeRenderer(tree, step_size=1e-4)
    with torch.no_grad():
        got = r.render_persp(torch.from_numpy(c2w), width=W, height=H, fx=fx).cpu().numpy()
        top = r.render_persp(c2w, width=W, height=H, fx=fx, rows=(0, 19)).cpu().numpy()
        bot = r.render_persp(c2w, width=W, height=H, fx=fx, rows=(19, 18)).cpu().numpy()
    err = float(np.abs(got - want).max())
    assert err < TOL_RGB, err
    assert (np.concatenate([top, bot]) == got).all()
    _record("render_persp_SH16", {"max_abs_err": err, "tol": TOL_RGB, "pixels": W * H})


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,depth", [("SH16", 3), ("SH25", 2), ("RGBA", 3)])
def test_backward_matches_oracle(fmt, depth):
    import torch
    from plenoctree_b200.octree import Rays, VolumeRenderer
    otree = make_tree(30 + depth, depth, fmt)
    tree = to_device_tree(otree)
    o, d, v = random_rays(8, 200)
    g = np.random.RandomState(9).normal(size=(200, 3)).astype(np.float32)
    want = OO.volume_render_backward(otree, o, d, v, g, step_size=1e-3)
    r = VolumeRenderer(tree, step_size=1e-3)
    params = tree.parameters()
    rgb = r.forward(Rays(torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(v)))
    (rgb * torch.from_numpy(g).cuda()).sum().backward()
    got = params[0].grad[:otree.n_internal].cpu().numpy()
    scale = np.abs(want).max()
    err = float(np.abs(got - want).max() / scale)
    assert err < TOL_GRAD_REL, (fmt, err)
    assert np.abs(want[..., -1]).max() > 0 and np.abs(want[..., 0]).max() > 0
    _record(f"backward_{fmt}", {"rel_max_err": err, "tol": TOL_GRAD_REL})


@pytest.mark.gpu
def test_fused_train_image_and_sgd_match_oracle():
    import torch
    from plenoctree_b200.octree import VolumeRenderer
    otree = make_tree(41, 3, "SH16")
    tree = to_device_tree(otree)
    c2w = look_at_pose(3)
    W, H, fx = 40, 30, 45.0
    o, d, v = OO.persp_rays(c2w, W, H, fx)
    gt = np.random.RandomState(4).uniform(0, 1, size=(H, W, 3)).astype(np.float32)
    im = OO.volume_render(otree, o, d, v, step_size=1e-3)
    mse, gout = OO.mse_and_grad_out(im.reshape(H, W, 3), gt)
    want = OO.volume_render_backward(otree, o, d, v, gout.reshape(-1, 3), step_size=1e-3)
    r = VolumeRenderer(tree, step_size=1e-3)
    # whole image in one launch, and as two row slabs accumulated into the same buffer
    for slabs in ([(0, H)], [(0, 13), (13, H - 13)]):
        tree.grad = None
        sq = torch.zeros(1, dtype=torch.float64, device="cuda")
        for rows in slabs:
            _, img = r.train_persp(c2w, torch.from_numpy(gt), W, H, fx, rows=rows, want_image=True, sq_err=sq)
        got = tree.grad_buffer()[:otree.n_internal].cpu().numpy()
        err = float(np.abs(got - want).max() / np.abs(want).max())
        assert err < TOL_GRAD_REL, err
        assert abs(float(sq.item()) / (H * W * 3) - mse) < 1e-6 * max(1.0, mse)
    _record("fused_train_SH16", {"rel_max_err": err, "mse": mse})
    # SGD: data <- data - lr * grad, grad zeroed
    before = tree.data[:otree.n_internal].cpu().numpy().copy()
    tree.sgd_step(1e3)
    after = tree.data[:otree.n_internal].cpu().numpy()
    np.testing.assert_allclose(after, OO.sgd_step(before, got, 1e3), rtol=0, atol=1e-6 * np.abs(before).max())
    assert float(tree.grad_buffer().abs().max()) == 0.0


@pytest.mark.gpu
def test_grid_weight_render_matches_oracle():
    import torch
    from plenoctree_b200.octree.extraction import calculate_grid_weights
    rs = np.random.RandomState(6)
    reso = 32
    grid = rs.uniform(0, 8, size=(reso, reso, reso)).astype(np.float32)
    grid[rs.rand(reso, reso, reso) < 0.8] = 0.0
    radius = np.array([1.4, 1.2, 1.3], dtype=np.float32)
    center = np.array([0.05, -0.1, 0.0], dtype=np.float32)
    inv = (0.5 / radius).astype(np.float32)
    off = (0.5 * (1 - center / radius)).astype(np.float32)
    W, H, fx = 28, 22, 30.0
    c2ws = np.stack([look_at_pose(s) for s in (1, 2, 3)])
    want = np.zeros_like(grid)
    for c2w in c2ws:
        o, d, _ = OO.persp_rays(c2w, W, H, fx)
        OO.grid_weight_render(grid, o, d, off, inv, step_size=1e-4, out=want)

    class DS:
        pass
    ds = DS()
    ds.w, ds.h, ds.focal, ds.camtoworlds = W, H, fx, c2ws
    got = calculate_grid_weights(ds, torch.from_numpy(grid).cuda().reshape(-1), reso, torch.from_numpy(inv).cuda(),
                                 torch.from_numpy(off).cuda(), step_size=1e-4).cpu().numpy()
    err = float(np.abs(got - want).max())
    assert err < 1e-5, err
    assert ((got > 0) == (want > 0)).all() and (want > 0).sum() > 500
    _record("grid_weight", {"max_abs_err": err, "voxels_hit": int((want > 0).sum())})


@pytest.mark.gpu
def test_extraction_end_to_end_matches_oracle(tmp_path):
    """octree.extraction on a random-init SH16 field, init_grid_depth 4 (32^3 grid): sigma sweep, weight mask,
    tree build, step-2 cell means, relu, npz — against the oracle pieces fed with the same masks and samples."""
    import torch
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200._lib import PREC_FP16X3
    from plenoctree_b200.nerf.models import NerfModel
    from plenoctree_b200.octree import N3Tree
    from plenoctree_b200.octree import extraction as E
    sh_deg = 3
    flat = O.init_flat_params(sh_deg, 20200823, bias_scale=0.05)
    flat2 = np.concatenate([flat, flat])
    nerf = NerfModel(sh_deg=sh_deg, precision=PREC_FP16X3)
    nerf.set_params(flat2)
    L = 4
    reso = 2 ** (L + 1)

    class DS:
        pass
    ds = DS()
    ds.w, ds.h, ds.focal = 24, 24, 26.0
    ds.camtoworlds = np.stack([look_at_pose(s, 4.0) for s in range(4)])
    args = E.default_args(init_grid_depth=L, samples_per_cell=4, masking_mode="weight", weight_thresh=1e-4,
                          renderer_step_size=1e-4, radius="1.5", center="0 0 0", output=str(tmp_path / "tree.npz"))
    torch.manual_seed(0)
    tree = E.extract(args, nerf, ds)
    # -- step 1 pieces against the oracle
    arr = ((np.arange(reso, dtype=np.float32) + 0.5) / reso).astype(np.float32)
    ax = ((arr - np.float32(0.5)) / np.float32(1.0 / 3.0)).astype(np.float32)
    pts = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), axis=-1).reshape(-1, 3)
    with torch.no_grad():
        _, sig_o = O.eval_points_raw(O.unflatten(flat, sh_deg), torch.from_numpy(pts))
    sig_o = sig_o.numpy().reshape(-1)
    sig_g = E._grid_sigmas(nerf, reso, [0.5] * 3, [1.0 / 3.0] * 3).cpu().numpy()
    assert np.abs(sig_g - sig_o).max() < 1e-4 * max(1.0, np.abs(sig_o).max())
    # tree topology from the GPU's own mask must equal the oracle's literal refinement sequence
    inv = np.full(3, 1.0 / 3.0, dtype=np.float32)
    off = np.full(3, 0.5, dtype=np.float32)
    gw = np.zeros((reso, reso, reso), dtype=np.float32)
    for c2w in ds.camtoworlds:
        o, d, _ = OO.persp_rays(c2w, ds.w, ds.h, ds.focal)
        OO.grid_weight_render(sig_g.reshape(reso, reso, reso), o, d, off, inv, step_size=1e-4, out=gw)
    mask = gw >= 1e-4
    assert mask.sum() > 50
    otree, _ = OO.build_tree_from_grid(mask, L, 1.5, [0, 0, 0], 49, "SH16")
    n = otree.n_internal
    assert tree.n_internal == n
    assert (tree.child.cpu().numpy() == otree.child[:n]).all()
    assert (tree.parent_depth.cpu().numpy() == otree.parent_depth[:n]).all()
    # -- step 2: finest leaves hold the mean of [raw_rgb, relu-ed raw_sigma-mean] over their samples
    lv = otree.leaves()
    deep = np.nonzero(otree.leaf_depths(lv) == L)[0]
    gen = torch.Generator(device="cuda")
    gen.manual_seed(20200823)   # step2 seeds leaf chunk c with 20200823 + c; this tree is a single chunk
    u = torch.rand((deep.size, 4, 3), device="cuda", generator=gen).cpu().numpy()
    spts = otree.sample(lv[deep], 4, u).reshape(-1, 3)
    with torch.no_grad():
        rgb_o, s_o = O.eval_points_raw(O.unflatten(flat, sh_deg), torch.from_numpy(spts))
    want = torch.cat([rgb_o, s_o], dim=-1).reshape(-1, 4, 49).mean(dim=1).numpy()
    want[:, -1] = np.maximum(want[:, -1], 0.0)
    got = tree.data.reshape(-1, 49)[torch.from_numpy(otree.pack_index(lv[deep, 0], lv[deep, 1:])).cuda()].cpu().numpy()
    err = float(np.abs(got - want).max() / np.abs(want).max())
    assert err < 2e-4, err
    # coarse leaves stay empty; file round-trips through N3Tree.load with fp16 data
    t2 = N3Tree.load(str(tmp_path / "tree.npz"))
    assert t2.n_internal == n and repr(t2.data_format) == "SH16"
    assert float((t2.data - tree.data).abs().max()) <= 1e-3 * float(tree.data.abs().max())
    _record("extraction_e2e", {"nodes": int(n), "finest_leaves": int(deep.size), "cell_mean_rel_err": err})


@pytest.mark.gpu
def test_optimization_improves_psnr():
    """octree.optimization (SGD on tree.data through the fused render+gradient kernel): fitting images rendered
    from a perturbed copy of the tree must raise the PSNR, like the reference's training loop does."""
    import torch
    from plenoctree_b200.octree import VolumeRenderer, optimization as OPT
    otree = make_tree(51, 3, "SH16")
    teacher = to_device_tree(otree)
    W, H, fx = 48, 48, 60.0
    poses = [look_at_pose(s) for s in range(6)]
    rt = VolumeRenderer(teacher, step_size=1e-3)
    with torch.no_grad():
        gts = [rt.render_persp(p, width=W, height=H, fx=fx).clamp_(0, 1) for p in poses]
    student = to_device_tree(otree)
    torch.manual_seed(1)
    with torch.no_grad():
        student.data[..., :-1] += 0.5 * torch.randn_like(student.data[..., :-1])
    # the reference's lr = 1e7 is for 800x800 images (the MSE mean divides every gradient by H*W*3, and every voxel
    # is seen by ~280x more pixels); 1e4 is the stable range for these 48x48 images
    lr = float(os.environ.get("POB_TEST_OCTREE_LR", 1e4))
    args = OPT.default_args(num_epochs=int(os.environ.get("POB_TEST_OCTREE_EPOCHS", 40)), lr=lr, val_interval=5,
                            renderer_step_size=1e-3, nosave=True, continue_on_decrease=True)
    r = VolumeRenderer(student, step_size=1e-3)
    p0 = OPT.run_test_step(r, poses, gts, H, W, fx)
    logs = []
    best, p1 = OPT.optimize(args, student, poses, gts, poses, gts, fx, log=logs.append)
    print("\n".join(logs[-6:]))
    assert p1 > p0 + 1.0, (p0, p1)
    _record("optimization", {"psnr_before": p0, "psnr_after": p1})


@pytest.mark.gpu
def test_adam_step_matches_torch_adam():
    """octree.optimization --nosgd (optimization.py:190-193): pob_octree_adam_step == torch.optim.Adam + zero_grad."""
    import torch
    otree = make_tree(71, 2, "SH9")
    tree = to_device_tree(otree)
    n = otree.n_internal
    ref = torch.nn.Parameter(tree.data[:n].clone())
    opt = torch.optim.Adam([ref], lr=0.05, eps=1e-8)
    g = torch.Generator(device="cuda").manual_seed(5)
    for _ in range(3):
        grad = torch.randn(ref.shape, device="cuda", generator=g) * (torch.rand(ref.shape, device="cuda", generator=g) < 0.3)
        tree.grad_buffer()[:n] = grad
        tree.adam_step(0.05, 1e-8)
        ref.grad = grad.clone()
        opt.step()
        assert float(tree.grad_buffer().abs().max()) == 0.0
    err = float((tree.data[:n] - ref.data).abs().max())
    assert err < 1e-5, err


def test_n3tree_host_bookkeeping_on_cpu(tmp_path):
    """The integer bookkeeping of plenoctree_b200.octree.N3Tree (refine order, chunked last level, leaf order, depths,
    corners / sample, assignment, relu, npz round trip) run on CPU tensors: the one CUDA call it makes (leaf lookup,
    pob_octree_query) is served by the oracle's query here; tests/-m gpu checks the real kernel against the same."""
    import torch
    from plenoctree_b200.octree import n3tree as NT
    rs = np.random.RandomState(1)
    L = 4
    reso = 2 ** (L + 1)
    mask = rs.rand(reso, reso, reso) < 0.08
    radius, center = [1.5, 1.2, 1.0], [0.1, 0.0, -0.2]
    otree, grid = OO.build_tree_from_grid(mask, L, radius, center, 49, "SH16", refine_chunk=700)
    t = NT.N3Tree.__new__(NT.N3Tree)                      # the constructor insists on a CUDA device
    t.device = torch.device("cpu")
    t.N, t.data_dim, t.depth_limit, t.geom_resize_fact = 2, 49, L, 1.0
    t.data_format = NT.DataFormat("SH16")
    t.invradius = torch.from_numpy(otree.invradius.copy())
    t.offset = torch.from_numpy(otree.offset.copy())
    t.data = torch.zeros((16, 2, 2, 2, 49))
    t.child = torch.zeros((16, 2, 2, 2), dtype=torch.int32)
    t.parent_depth = torch.zeros((16, 2), dtype=torch.int32)
    t.n_internal, t.n_free, t.grad, t._leaves = 1, 0, None, None

    def query_packed(points):
        o = OO.N3Tree(N=2, data_dim=49, depth_limit=L, radius=radius, center=center, data_format="SH16")
        o.child, o.n_internal = t.child.numpy(), t.n_internal
        node, ijk, _, _ = o.query(points.numpy())
        return torch.from_numpy(o.pack_index(node, ijk))
    t.query_packed = query_packed
    g = torch.from_numpy(grid)
    for _ in range(L - 1):
        t[g].refine()
    for j in range(0, g.shape[0], 700):
        t[g[j:j + 700]].refine()
    n = otree.n_internal
    assert t.n_internal == n and t.max_depth == L and t.capacity >= n
    assert (t.child[:n].numpy() == otree.child[:n]).all()
    assert (t.parent_depth[:n].numpy() == otree.parent_depth[:n]).all()
    lv = otree.leaves()
    assert (t._all_leaves().numpy() == lv).all() and (t.depths.numpy() == otree.leaf_depths(lv)).all()
    sel = np.nonzero(otree.leaf_depths(lv) == L)[0][:200]
    u = rs.rand(sel.size, 3, 3).astype(np.float32)
    got = t[torch.from_numpy(sel)].sample(3, torch.from_numpy(u)).numpy()
    np.testing.assert_allclose(got, otree.sample(lv[sel], 3, u), rtol=0, atol=1e-6)
    vals = torch.randn(sel.size, 49)
    t[torch.from_numpy(sel)] = vals
    t[:, -1:].relu_()
    flat = t.data.reshape(-1, 49)
    pk = otree.pack_index(lv[sel, 0], lv[sel, 1:])
    assert torch.equal(flat[pk][:, :-1], vals[:, :-1]) and torch.equal(flat[pk][:, -1], vals[:, -1].clamp(min=0))
    assert float(flat[:, -1].min()) >= 0.0
    t.save(str(tmp_path / "t.npz"), compress=False)
    assert t.capacity == n                                 # shrink_to_fit
    z = np.load(str(tmp_path / "t.npz"))
    assert z["data"].dtype == np.float16 and int(z["n_internal"]) == n and str(z["data_format"]) == "SH16"
    t2 = NT.N3Tree.load(str(tmp_path / "t.npz"), map_location="cpu")
    assert t2.n_internal == n and t2.N == 2 and repr(t2.data_format) == "SH16"
    assert (t2.child.numpy() == otree.child[:n]).all()
    assert float((t2.data - t.data).abs().max()) <= 2e-3 * float(t.data.abs().max())
    # a depth-limited tree refuses to refine further
    assert t[g[:10]].refine() is False


def test_camera_records_match_the_c_struct():
    """pob_camera is 16 floats: c2w[3][4] row-major, fx, fy, width, height (include/plenoctree_b200.h)."""
    import ctypes
    from plenoctree_b200 import _lib
    from plenoctree_b200.octree.renderer import camera_array, make_camera
    assert ctypes.sizeof(_lib.Camera) == 64 and ctypes.sizeof(_lib.OctreeOpts) == 16
    c2w = look_at_pose(4)
    cam = make_camera(c2w, 800, 600, 1111.0)
    rec = np.frombuffer(bytes(cam), dtype=np.float32)
    assert np.array_equal(rec[:12], c2w[:3, :4].reshape(-1)) and list(rec[12:]) == [1111.0, 1111.0, 800.0, 600.0]
    arr = camera_array(np.stack([c2w, look_at_pose(5)]), 800, 600, 1111.0, device="cpu").numpy()
    assert arr.shape == (2, 16) and np.array_equal(arr[0], rec)
    with pytest.raises(ValueError):
        make_camera(np.eye(3), 8, 8, 1.0)


def test_backward_first_pass_equals_g_dot_out():
    """svox's trace_ray_backward spends a whole march computing accum = sum_j w_j (c_j . g) + T_end * bg * sum(g);
    the CUDA kernels use g . rgb of the forward render instead.  The two are the same number."""
    tree = make_tree(8, 3, "SH16", density=0.4)
    o, d, v = random_rays(9, 64)
    g = np.random.RandomState(2).normal(size=(64, 3)).astype(np.float32)
    rgb = OO.volume_render(tree, o, d, v, step_size=1e-3)
    # accumulate pass 1 exactly like the oracle's backward does
    rgba = False
    K = 16
    oo, dd, ds, invd, tmin, tmax = OO._setup(tree.offset, tree.invradius, o, d)
    basis = OO.sh_basis(K, v)
    miss = (tmax < 0) | (tmin > tmax)
    accum = np.zeros(64, dtype=np.float64)
    light = np.ones(64, dtype=np.float32)
    t = tmin.copy()
    active = ~miss & (t < tmax)
    while active.any():
        a = np.nonzero(active)[0]
        pos = (oo[a] + t[a][:, None] * dd[a]).astype(np.float32)
        node, ijk, cube, rel = tree.query_unit(pos)
        smin, smax = OO._dda_unit(rel, invd[a])
        delta_t = (((smax - smin) / cube).astype(np.float32) + np.float32(1e-3)).astype(np.float32)
        sigma = tree.data[node, ijk[:, 0], ijk[:, 1], ijk[:, 2], -1]
        h = sigma > 0
        if h.any():
            ah = a[h]
            att = np.exp(-delta_t[h] * ds[ah] * sigma[h]).astype(np.float32)
            w = light[ah] * (1 - att)
            pre, _ = OO._leaf_color_pre(tree, basis[ah], node[h], ijk[h], K, rgba)
            accum[ah] += w * (OO._sigmoid(pre) * g[ah]).sum(axis=1)
            light[ah] *= att
        t[a] = (t[a] + delta_t).astype(np.float32)
        active = active & (t < tmax)
    accum[~miss] += light[~miss] * 1.0 * g[~miss].sum(axis=1)
    want = (g[~miss].astype(np.float64) * rgb[~miss]).sum(axis=1)
    assert np.abs(accum[~miss] - want).max() < 1e-5

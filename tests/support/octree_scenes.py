"""Octree scenes: random and production-depth trees, their device copies, cameras, ray sets and CLI scenes."""
import functools
import subprocess
import sys
import time

import numpy as np

from oracle import octree_oracle as OO
from plenoctree_b200.octree import compression as C
from tests.support.records import ROOT


def make_tree(seed, depth, data_format, density=0.35, radius=1.3, center=(0.1, -0.05, 0.0), sigma_scale=6.0):
    """random sparse tree: refine `depth` levels at random occupied voxels, random coefficients, sigma >= 0 with
    about half of the finest leaves empty (sigma = 0), coarse leaves empty."""
    rs = np.random.RandomState(seed)
    K = 1 if data_format == "RGBA" else int(data_format[2:])
    D = 4 if data_format == "RGBA" else 3 * K + 1
    reso = 2 ** (depth + 1)
    mask = rs.rand(reso, reso, reso) < density
    tree, _ = OO.build_tree_from_grid(mask, depth, radius, center, D, data_format)
    n = tree.n_internal
    tree.data[:n] = rs.normal(0, 1.0, size=tree.data[:n].shape).astype(np.float32)
    sig = rs.uniform(0, sigma_scale, size=tree.data[:n, ..., -1].shape).astype(np.float32)
    sig[rs.rand(*sig.shape) < 0.5] = 0.0
    deep = (tree.parent_depth[:n, 1] == depth)[:, None, None, None]
    tree.data[:n, ..., -1] = np.where(deep, sig, 0.0)
    return tree


def look_at_pose(seed, dist=3.5):
    rs = np.random.RandomState(seed)
    eye = rs.normal(size=3)
    eye = eye / np.linalg.norm(eye) * dist
    fwd = -eye / np.linalg.norm(eye)
    up = np.array([0.0, 0.0, 1.0])
    right = np.cross(fwd, up)
    right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    c2w = np.eye(4, dtype=np.float32)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, up, -fwd, eye
    return c2w


def to_device_tree(otree):
    import torch
    from plenoctree_b200.octree import N3Tree
    fmt = otree.data_format
    t = N3Tree(N=otree.N, data_dim=otree.data_dim, depth_limit=otree.depth_limit, init_reserve=otree.n_internal,
               radius=0.5 / otree.invradius, center=(1 - 2 * otree.offset) * (0.5 / otree.invradius),
               data_format=fmt)
    n = otree.n_internal
    t.invradius = torch.from_numpy(otree.invradius).cuda()
    t.offset = torch.from_numpy(otree.offset).cuda()
    t.data[:n] = torch.from_numpy(otree.data[:n]).cuda()
    t.child[:n] = torch.from_numpy(otree.child[:n]).cuda()
    t.parent_depth[:n] = torch.from_numpy(otree.parent_depth[:n]).cuda()
    t.n_internal = n
    t._leaves = None
    return t


def assert_device_tree_build_matches(otree, refines, radius, center, rs, query_box=2.0):
    """A device N3Tree refined by the same sequence of `tree[points].refine()` calls as the oracle tree `otree`
    (refines: float32 [n,3] world-point arrays, one call each) has the oracle's topology bit for bit; query_packed is
    bit-exact on points of [-query_box, query_box]^3 around the box centre, leaves / depths are identical and sample
    agrees."""
    import torch
    from plenoctree_b200.octree import N3Tree
    L = otree.depth_limit
    tree = N3Tree(N=otree.N, data_dim=otree.data_dim, depth_limit=L, init_reserve=16, geom_resize_fact=1.0,
                  radius=radius, center=center, data_format=otree.data_format)
    for pts in refines:
        tree[torch.from_numpy(pts).cuda()].refine()
    n = otree.n_internal
    assert tree.n_internal == n and tree.max_depth == otree.max_depth == L
    assert (tree.child[:n].cpu().numpy() == otree.child[:n]).all()
    assert (tree.parent_depth[:n].cpu().numpy() == otree.parent_depth[:n]).all()
    pts = (np.asarray(center, dtype=np.float32) + rs.uniform(-query_box, query_box, size=(5000, 3))).astype(np.float32)
    node, ijk, _, _ = otree.query(pts)
    want = otree.pack_index(node, ijk)
    got = tree.query_packed(torch.from_numpy(pts).cuda()).cpu().numpy()
    assert (got == want).all()
    # leaves / depths / sample agree with the oracle
    lv = otree.leaves()
    assert (tree._all_leaves().cpu().numpy() == lv).all()
    assert (tree.depths.cpu().numpy() == otree.leaf_depths(lv)).all()
    sel = np.nonzero(otree.leaf_depths(lv) == L)[0][:300]
    u = rs.rand(sel.size, 5, 3).astype(np.float32)
    got = tree[torch.from_numpy(sel).cuda()].sample(5, torch.from_numpy(u).cuda()).cpu().numpy()
    want = otree.sample(lv[sel], 5, u)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-6)
    return tree


f32, f64 = np.float32, np.float64


STOP = 1e-2                 # svox fast=True: sigma_thresh = stop_thresh = 1e-2


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


NAMES = list(SPECS)


def _scene(tmp_path):
    """a Blender-layout scene (the writer tests/test_pipeline.py uses) of 32x32 views of a random SH16 tree, and a
    perturbed copy of the tree as tree.npz"""
    import torch
    from plenoctree_b200.nerf import datasets as D
    from plenoctree_b200.octree import VolumeRenderer
    otree = make_tree(61, 3, "SH16")
    teacher = to_device_tree(otree)
    W, cam_x = 32, 0.6911112070083618
    focal = 0.5 * W / np.tan(0.5 * cam_x)
    poses = {"train": [look_at_pose(s) for s in range(4)], "val": [look_at_pose(s) for s in range(10, 13)],
             "test": [look_at_pose(s) for s in range(20, 22)]}
    r = VolumeRenderer(teacher, step_size=1e-3)
    with torch.no_grad():
        images = {k: [r.render_persp(p, W, W, focal).clamp_(0, 1).cpu().numpy() for p in ps] for k, ps in poses.items()}
    D.write_blender_scene(str(tmp_path / "scene"), images, poses, cam_x)
    student = to_device_tree(otree)
    torch.manual_seed(2)
    with torch.no_grad():
        student.data[..., :-1] += 0.5 * torch.randn_like(student.data[..., :-1])
    student.save(str(tmp_path / "tree.npz"), compress=False)
    (tmp_path / "cfg.yaml").write_text("dataset: blender\nfactor: 0\nwhite_bkgd: true\n")
    return ["--config", str(tmp_path / "cfg"), "--data_dir", str(tmp_path / "scene"), "--renderer_step_size", "1e-3"]


def _cli(module, argv):
    r = subprocess.run([sys.executable, "-m", module] + argv, capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    return r.stdout


def _state(otree):
    """the keys N3Tree.save writes (data in fp16, like svox) for an oracle tree"""
    n = otree.n_internal
    return {"data_dim": np.int64(otree.data_dim), "child": otree.child[:n].copy(),
            "parent_depth": otree.parent_depth[:n].copy(), "n_internal": np.int64(n), "n_free": np.int64(0),
            "invradius3": otree.invradius.astype(f32), "offset": otree.offset.astype(f32),
            "depth_limit": np.int64(otree.depth_limit), "geom_resize_fact": np.float64(1.5),
            "data": otree.data[:n].astype(np.float16), "data_format": str(otree.data_format)}


SH25_SPEC = (2, 7, "SH25", (1.0, 1.2, 0.9), (0.1, -0.05, 0.2), (-1, 1, -1))
# tree -> (bits, retain, weighted) compressions
CASES = {
    "n2_d8_sh16": [(16, 0, False), (5, 2, True)],
    "n3_d4_sh16": [(5, 0, False), (16, 2, False)],
    "n2_d7_sh25": [(5, 2, False), (16, 0, True)],
    "chain_d26_rgba": [(16, 0, False), (5, 0, True)],
}


@functools.lru_cache(maxsize=None)
def _tree(name):
    """-> oracle tree, world points of its occupied cells (test_octree_march's trees; SH25 built the same way)"""
    if name != "n2_d7_sh25":
        otree, _, pts = _build(name)
        return otree, pts
    N, L, fmt, radius, center, region = SH25_SPEC
    rs = np.random.RandomState(sum(map(ord, name)))
    otree = OO.N3Tree(N=N, data_dim=76, depth_limit=L, init_reserve=1024, geom_resize_fact=1.5, radius=radius,
                      center=center, data_format=fmt)
    pts = _to_world(otree, _shell_voxels(N, L, region, rs))
    for _ in range(L):
        otree.refine_at(pts)
    _fill(otree, rs)
    return otree, pts


@functools.lru_cache(maxsize=None)
def _compressed(name, i):
    bits, retain, weighted = CASES[name][i]
    return C.compress_tree(_state(_tree(name)[0]), bits=bits, sigma_thresh=2.0, retain=retain, weighted=weighted)


def _pair(name, i):
    """(compressed renderer, fp32 renderer of decompress_data of the same file)"""
    import torch
    from plenoctree_b200.octree import VolumeRenderer, load_tree
    otree, _ = _tree(name)
    c = _compressed(name, i)
    q = load_tree(c, map_location="cuda")
    ref = to_device_tree(otree)
    n = otree.n_internal
    ref.data[:n] = torch.from_numpy(C.decompress_data(c)).cuda()
    return q, ref

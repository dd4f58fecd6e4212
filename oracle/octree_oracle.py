"""CPU oracle for the PlenOctree side of the path (SURVEY.md §8 rows a13 middle, a15).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and the CPU legs of the bench scripts may import this module.

**Parity unpinned.**  Everything here belongs to a third-party dependency that is *absent* from
/root/reference: `svox` (PyPI, `svox>=0.2.26` in requirements.txt:14 / `>=0.2.28` in environment.yml:28,
"SVOX 0.2.22" in octree/optimization.py:238).  The reference tree holds no test, golden vector or fixture for
it.  What follows restates svox's published algorithm (svox/svox.py `N3Tree`, svox/renderer.py
`VolumeRenderer`, svox/csrc/{svox_kernel,rt_kernel}.cu of the 0.2.2x line) and is anchored on the reference's
own call sites, which fix the argument meaning and the data layout:

  octree/extraction.py:181-214   _C.grid_weight_render(sigma_grid, cam, opts, offset, invradius)
  octree/extraction.py:341-353   tree[grid].refine()            (level-by-level build, 2M-point chunks)
  octree/extraction.py:358-394   tree.depths, tree[inds].sample(S), tree[inds] = rgba   (sigma is the LAST channel)
  octree/extraction.py:503-509   tree[:, -1:].relu_(), shrink_to_fit(), save(compress=False)
  octree/compression.py:75-95    npz keys data / child / parent_depth / n_internal / n_free / depth_limit / ...
  octree/optimization.py:167-229 VolumeRenderer.render_persp(c2w, height, width, fx) fwd/bwd, SGD on tree.data
  octree/nerf/utils.py:448-498   render_persp(..., fast=not no_early_stop) for evaluation

The checks that stand in for an executable reference: the backward pass equals the autograd/finite-difference
gradient of the forward pass (tests/test_octree.py), a uniform-density tree reproduces the closed-form
transmittance, and a tree sampled from a NeRF-SH field renders to the same image as the NeRF-SH volumetric
renderer of that field up to discretisation (PSNR acceptance test).

All arithmetic is float32 numpy in the operation order of the CUDA kernels it describes; rays are processed in
lock-step (one numpy op per scalar op of the per-ray loop).
"""
import numpy as np

f32 = np.float32

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
SH_C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
         -0.4570457994644658, 1.445305721320277, -0.5900435899266435]
SH_C4 = [2.5033429417967046, -1.7701307697799304, 0.9461746957575601, -0.6690465435572892,
         0.10578554691520431, -0.6690465435572892, 0.47308734787878004, -1.7701307697799304,
         0.6258357354491761]


def sh_basis(basis_dim, d):
    """svox rt_kernel.cu `_precalc_sh_basis` (same polynomials and signs as nerf_sh/nerf/sh.py:73-108).
    d [R,3] unit view directions -> [R, basis_dim]."""
    d = np.asarray(d, dtype=f32)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    out = np.zeros((d.shape[0], 25), dtype=f32)
    out[:, 0] = SH_C0
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    out[:, 1] = f32(-SH_C1) * y
    out[:, 2] = f32(SH_C1) * z
    out[:, 3] = f32(-SH_C1) * x
    out[:, 4] = f32(SH_C2[0]) * xy
    out[:, 5] = f32(SH_C2[1]) * yz
    out[:, 6] = f32(SH_C2[2]) * (f32(2.0) * zz - xx - yy)
    out[:, 7] = f32(SH_C2[3]) * xz
    out[:, 8] = f32(SH_C2[4]) * (xx - yy)
    out[:, 9] = f32(SH_C3[0]) * y * (f32(3) * xx - yy)
    out[:, 10] = f32(SH_C3[1]) * xy * z
    out[:, 11] = f32(SH_C3[2]) * y * (f32(4) * zz - xx - yy)
    out[:, 12] = f32(SH_C3[3]) * z * (f32(2) * zz - f32(3) * xx - f32(3) * yy)
    out[:, 13] = f32(SH_C3[4]) * x * (f32(4) * zz - xx - yy)
    out[:, 14] = f32(SH_C3[5]) * z * (xx - yy)
    out[:, 15] = f32(SH_C3[6]) * x * (xx - f32(3) * yy)
    out[:, 16] = f32(SH_C4[0]) * xy * (xx - yy)
    out[:, 17] = f32(SH_C4[1]) * yz * (f32(3) * xx - yy)
    out[:, 18] = f32(SH_C4[2]) * xy * (f32(7) * zz - f32(1))
    out[:, 19] = f32(SH_C4[3]) * yz * (f32(7) * zz - f32(3))
    out[:, 20] = f32(SH_C4[4]) * (zz * (f32(35) * zz - f32(30)) + f32(3))
    out[:, 21] = f32(SH_C4[5]) * xz * (f32(7) * zz - f32(3))
    out[:, 22] = f32(SH_C4[6]) * (xx - yy) * (f32(7) * zz - f32(1))
    out[:, 23] = f32(SH_C4[7]) * xz * (xx - f32(3) * yy)
    out[:, 24] = f32(SH_C4[8]) * (xx * (xx - f32(3) * yy) - yy * (f32(3) * xx - yy))
    return out[:, :basis_dim]


# ----------------------------------------------------------------------------------------------
# N3Tree (svox/svox.py)
# ----------------------------------------------------------------------------------------------
class N3Tree:
    """svox.N3Tree restated: N^3-tree whose internal node t holds data[t, i, j, k, :] for its N^3 cells and
    child[t, i, j, k] = (index of the child node) - t, 0 for a leaf cell.  parent_depth[t] = (packed index of
    the parent cell, depth); the root node is node 0 with depth 0.  World -> tree: p * invradius + offset in
    [0,1]^3 (constructor: invradius = 0.5 / radius, offset = 0.5 * (1 - center / radius))."""

    def __init__(self, N=2, data_dim=4, depth_limit=10, init_reserve=1, geom_resize_fact=1.0, radius=0.5,
                 center=(0.5, 0.5, 0.5), data_format="RGBA"):
        self.N = int(N)
        self.data_dim = int(data_dim)
        self.depth_limit = int(depth_limit)
        self.geom_resize_fact = float(geom_resize_fact)
        radius = np.broadcast_to(np.asarray(radius, dtype=f32), (3,)).copy()
        center = np.broadcast_to(np.asarray(center, dtype=f32), (3,)).copy()
        self.invradius = (f32(0.5) / radius).astype(f32)
        self.offset = (f32(0.5) * (f32(1.0) - center / radius)).astype(f32)
        cap = max(int(init_reserve), 1)
        self.data = np.zeros((cap, N, N, N, data_dim), dtype=f32)
        self.child = np.zeros((cap, N, N, N), dtype=np.int32)
        self.parent_depth = np.zeros((cap, 2), dtype=np.int32)
        self.n_internal = 1
        self.n_free = 0
        self.data_format = data_format

    # -- geometry -------------------------------------------------------------------------------
    def world2tree(self, p):
        return (self.offset + self.invradius * np.asarray(p, dtype=f32)).astype(f32)

    def query(self, points_world):
        """svox_kernel.cu `query_single_from_root` for a batch: -> (node, i, j, k) int arrays, cube_sz, rel pos."""
        q = self.world2tree(points_world)
        return self.query_unit(q)

    def query_unit(self, q):
        N = f32(self.N)
        q = np.maximum(f32(0.0), np.minimum(f32(1.0) - f32(1e-6), q)).astype(f32)  # clamp_coord
        M = q.shape[0]
        node = np.zeros(M, dtype=np.int64)
        ijk = np.zeros((M, 3), dtype=np.int64)
        cube = np.full(M, N, dtype=f32)
        rel = q.copy()
        active = np.ones(M, dtype=bool)
        while active.any():
            a = np.nonzero(active)[0]
            r = rel[a] * N
            u = np.floor(r).astype(np.int64)
            rel[a] = (r - u.astype(f32)).astype(f32)
            ijk[a] = u
            skip = self.child[node[a], u[:, 0], u[:, 1], u[:, 2]]
            leaf = skip == 0
            active[a[leaf]] = False
            go = a[~leaf]
            cube[go] = cube[go] * N
            node[go] = node[go] + skip[~leaf]
        return node, ijk, cube, rel

    def pack_index(self, node, ijk):
        N = self.N
        return ((node * N + ijk[:, 0]) * N + ijk[:, 1]) * N + ijk[:, 2]

    # -- refinement -----------------------------------------------------------------------------
    def _reserve(self, need):
        cap = self.data.shape[0]
        if need <= cap:
            return
        new = max(need, int(cap * max(self.geom_resize_fact, 1.0)) + 1)
        N, D = self.N, self.data_dim
        for name, shape, dt in (("data", (new, N, N, N, D), f32), ("child", (new, N, N, N), np.int32),
                                ("parent_depth", (new, 2), np.int32)):
            arr = np.zeros(shape, dtype=dt)
            arr[:cap] = getattr(self, name)
            setattr(self, name, arr)

    def refine_at(self, points_world):
        """`tree[points].refine()` (octree/extraction.py:343-352): the distinct leaves holding the points, in
        sorted (node, i, j, k) order (N3TreeView._unique_node_key = torch.unique(dim=0)), each become an
        internal node appended at the end; leaves already at depth_limit are skipped (N3Tree.refine)."""
        node, ijk, _, _ = self.query(points_world)
        key = np.unique(self.pack_index(node, ijk))
        N3 = self.N ** 3
        knode = key // N3
        depths = self.parent_depth[knode, 1]
        key = key[depths < self.depth_limit]
        n_new = key.shape[0]
        if n_new == 0:
            return False
        filled = self.n_internal
        self._reserve(filled + n_new)
        knode = key // N3
        new_idx = np.arange(filled, filled + n_new, dtype=np.int64)
        self.child.reshape(-1)[key] = (new_idx - knode).astype(np.int32)
        self.data[filled:filled + n_new] = self.data.reshape(-1, self.data_dim)[key][:, None, None, None, :]
        self.parent_depth[filled:filled + n_new, 0] = key.astype(np.int32)
        self.parent_depth[filled:filled + n_new, 1] = self.parent_depth[knode, 1] + 1
        self.n_internal += n_new
        return True

    # -- leaves ---------------------------------------------------------------------------------
    def leaves(self):
        """N3Tree._all_leaves: (child[:n_internal] == 0).nonzero() — lexicographic (node, i, j, k)."""
        return np.argwhere(self.child[:self.n_internal] == 0)

    @property
    def max_depth(self):
        return int(self.parent_depth[:self.n_internal, 1].max())

    def leaf_depths(self, leaves):
        return self.parent_depth[leaves[:, 0], 1]

    def sample(self, leaves, n_samples, uniforms):
        """N3TreeView.sample (octree/extraction.py:370): corners + U[0,1) * lengths in world coordinates;
        `uniforms` [n, S, 3] replaces torch.rand."""
        depth = self.leaf_depths(leaves).astype(f32)
        corn_unit = self._corners_exact(leaves)
        corn = ((corn_unit - self.offset) / self.invradius).astype(f32)
        length = (np.power(np.float64(self.N), -depth.astype(np.float64) - 1.0).astype(f32)[:, None]
                  / self.invradius).astype(f32)   # N^-(depth+1); exact for N = 2
        return (corn[:, None, :] + uniforms.astype(f32) * length[:, None, :]).astype(f32)

    def _corners_exact(self, leaves):
        """N3Tree._calc_corners: lower corner of each leaf in [0,1]^3, walking up the parents (leaf digit has
        weight 1, its parent cell N, ...); exact in fp32 for depth < 23."""
        N = self.N
        node = leaves[:, 0].copy()
        coord = leaves[:, 1:4].astype(np.int64)
        mult = np.ones(leaves.shape[0], dtype=np.int64)
        while True:
            up = node > 0
            if not up.any():
                break
            pk = self.parent_depth[node[up], 0].astype(np.int64)
            pijk = np.stack([(pk // (N * N)) % N, (pk // N) % N, pk % N], axis=1)
            mult[up] = mult[up] * N
            coord[up] = coord[up] + pijk * mult[up][:, None]
            node[up] = pk // (N ** 3)
        depth = self.leaf_depths(leaves).astype(np.int64)
        res = (N ** (depth + 1)).astype(np.float64)
        return (coord / res[:, None]).astype(f32)

    # -- io ---------------------------------------------------------------------------------------
    def shrink_to_fit(self):
        n = self.n_internal
        self.data = self.data[:n].copy()
        self.child = self.child[:n].copy()
        self.parent_depth = self.parent_depth[:n].copy()

    def state(self):
        """N3Tree.save payload (keys consumed by octree/compression.py:75-95 and N3Tree.load); data is stored
        as float16 like svox does ("save CPU memory")."""
        n = self.n_internal
        d = {
            "data_dim": np.int64(self.data_dim),
            "child": self.child[:n],
            "parent_depth": self.parent_depth[:n],
            "n_internal": np.int64(self.n_internal),
            "n_free": np.int64(self.n_free),
            "invradius3": self.invradius,
            "offset": self.offset,
            "depth_limit": np.int64(self.depth_limit),
            "geom_resize_fact": np.float64(self.geom_resize_fact),
            "data": self.data[:n].astype(np.float16),
        }
        if self.data_format is not None:
            d["data_format"] = str(self.data_format)
        return d


# ----------------------------------------------------------------------------------------------
# Rays
# ----------------------------------------------------------------------------------------------
def persp_rays(c2w, width, height, fx, fy=None):
    """svox rt_kernel.cu `render_image_kernel` (what VolumeRenderer.render_persp launches; call sites
    octree/optimization.py:178,202): pixel (ix, iy) -> dir = normalize([(ix - w/2)/fx, -(iy - h/2)/fy, -1]),
    rotated by c2w[:3,:3]; origin = c2w[:3,3]; vdir = dir (no +0.5 pixel centre, README.md:184).
    Returns origins, dirs, vdirs [h*w, 3], row-major pixels."""
    fy = fx if fy is None else fy
    c2w = np.asarray(c2w, dtype=f32)
    ix, iy = np.meshgrid(np.arange(width, dtype=f32), np.arange(height, dtype=f32), indexing="xy")
    d = np.stack([(ix - f32(0.5) * f32(width)) / f32(fx), -(iy - f32(0.5) * f32(height)) / f32(fy),
                  np.full_like(ix, -1.0)], axis=-1).reshape(-1, 3).astype(f32)
    nrm = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]).astype(f32)
    d = (d / nrm[:, None]).astype(f32)
    R = c2w[:3, :3]
    out = np.zeros_like(d)
    for a in range(3):
        out[:, a] = R[a, 0] * d[:, 0] + R[a, 1] * d[:, 1] + R[a, 2] * d[:, 2]
    o = np.broadcast_to(c2w[:3, 3], out.shape).astype(f32).copy()
    return o, out, out.copy()


def _dda_unit(cen, invdir):
    """rt_kernel.cu `_dda_unit`: intersect the unit cube, -> (tmin, tmax)."""
    tmin = np.zeros(cen.shape[0], dtype=f32)
    tmax = np.full(cen.shape[0], 1e9, dtype=f32)
    for i in range(3):
        t1 = (-cen[:, i] * invdir[:, i]).astype(f32)
        t2 = (t1 + invdir[:, i]).astype(f32)
        tmin = np.maximum(tmin, np.minimum(t1, t2))
        tmax = np.minimum(tmax, np.maximum(t1, t2))
    return tmin, tmax


def _setup(offset, invradius, origins, dirs):
    """transform_coord + _get_delta_scale + invdir (rt_kernel.cu trace_ray prologue)."""
    o = (offset + invradius * np.asarray(origins, dtype=f32)).astype(f32)
    d = (np.asarray(dirs, dtype=f32) * invradius).astype(f32)
    nrm = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]).astype(f32)
    delta_scale = (f32(1.0) / nrm).astype(f32)
    d = (d * delta_scale[:, None]).astype(f32)
    invdir = (f32(1.0) / (d + f32(1e-9))).astype(f32)
    tmin, tmax = _dda_unit(o, invdir)
    return o, d, delta_scale, invdir, tmin, tmax


def _sigmoid(x):
    return (f32(1.0) / (f32(1.0) + np.exp(-x).astype(f32))).astype(f32)


def _leaf_color_pre(tree, basis, node, ijk, basis_dim, rgba):
    """pre-sigmoid colour of the leaves for each ray: sum_k basis[k] * val[c*K + k]  (trace_ray inner loop)."""
    val = tree.data[node, ijk[:, 0], ijk[:, 1], ijk[:, 2]]
    if rgba:
        return val[:, :3].astype(f32), val
    K = basis_dim
    pre = np.zeros((node.shape[0], 3), dtype=f32)
    for c in range(3):
        acc = np.zeros(node.shape[0], dtype=f32)
        for k in range(K):
            acc = (acc + basis[:, k] * val[:, c * K + k]).astype(f32)
        pre[:, c] = acc
    return pre, val


def volume_render(tree, origins, dirs, vdirs, step_size=1e-3, background_brightness=1.0, sigma_thresh=0.0,
                  stop_thresh=0.0, return_steps=False, _record=None):
    """rt_kernel.cu `trace_ray` (forward of svox.VolumeRenderer; octree/optimization.py:178,202,
    octree/nerf/utils.py:472).  fast=True in svox sets sigma_thresh = stop_thresh = 1e-2.
    -> rgb [R,3] (and the number of leaf visits / contributing visits per ray).
    `_record` (a dict, see march_visits) receives every visit of the march as it happens."""
    rgba = tree.data_format is None or str(tree.data_format).upper().startswith("RGBA")
    K = 1 if rgba else (tree.data_dim - 1) // 3
    R = np.asarray(origins).shape[0]
    o, d, delta_scale, invdir, tmin, tmax = _setup(tree.offset, tree.invradius, origins, dirs)
    basis = sh_basis(K, vdirs) if not rgba else None
    out = np.zeros((R, 3), dtype=f32)
    miss = (tmax < 0) | (tmin > tmax)
    out[miss] = f32(background_brightness)
    light = np.ones(R, dtype=f32)
    t = tmin.copy()
    active = ~miss & (t < tmax)
    done_full = np.zeros(R, dtype=bool)
    visits = np.zeros(R, dtype=np.int64)
    hits = np.zeros(R, dtype=np.int64)
    while active.any():
        a = np.nonzero(active)[0]
        pos = (o[a] + t[a][:, None] * d[a]).astype(f32)
        node, ijk, cube, rel = tree.query_unit(pos)
        smin, smax = _dda_unit(rel, invdir[a])
        t_sub = ((smax - smin) / cube).astype(f32)
        delta_t = (t_sub + f32(step_size)).astype(f32)
        sigma = tree.data[node, ijk[:, 0], ijk[:, 1], ijk[:, 2], tree.data_dim - 1]
        visits[a] += 1
        if _record is not None:
            _record["steps"].append((a, tree.pack_index(node, ijk), delta_t))
        h = sigma > f32(sigma_thresh)
        if h.any():
            ah = a[h]
            hits[ah] += 1
            att = np.exp(-delta_t[h] * delta_scale[ah] * sigma[h]).astype(f32)
            weight = (light[ah] * (f32(1.0) - att)).astype(f32)
            pre, _ = _leaf_color_pre(tree, None if rgba else basis[ah], node[h], ijk[h], K, rgba)
            out[ah] = (out[ah] + weight[:, None] * _sigmoid(pre)).astype(f32)
            light[ah] = (light[ah] * att).astype(f32)
            full = light[ah] <= f32(stop_thresh)
            if full.any():
                af = ah[full]
                scale = (f32(1.0) / (f32(1.0) - light[af])).astype(f32)
                out[af] = (out[af] * scale[:, None]).astype(f32)
                done_full[af] = True
        t[a] = (t[a] + delta_t).astype(f32)
        active = active & ~done_full & (t < tmax)
    bg = ~miss & ~done_full
    out[bg] = (out[bg] + light[bg][:, None] * f32(background_brightness)).astype(f32)
    if _record is not None:
        _record.update(delta_scale=delta_scale, miss=miss, stopped=done_full)
    if return_steps:
        return out, visits, hits
    return out


def march_visits(tree, origins, dirs, vdirs, step_size=1e-3, background_brightness=1.0, sigma_thresh=0.0,
                 stop_thresh=0.0):
    """The leaf visits of `volume_render`'s float32 march (the same march, recorded as it runs), ray by ray in march
    order: dict of
        ray [V] int64, leaf [V] int64 (packed leaf index), delta_t [V] float32   one entry per visit
        delta_scale [R] float32, miss [R] bool (the ray misses the box), stopped [R] bool (early termination)
        rgb [R,3], visits [R], hits [R]                                          volume_render's return values
    A ray's march depends on the tree data only through early termination (stop_thresh > 0)."""
    rec = {"steps": []}
    rgb, visits, hits = volume_render(tree, origins, dirs, vdirs, step_size, background_brightness, sigma_thresh,
                                      stop_thresh, return_steps=True, _record=rec)
    steps = rec.pop("steps")
    if steps:
        ray, leaf, dt = (np.concatenate([s[i] for s in steps]) for i in range(3))
    else:
        ray, leaf, dt = np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, f32)
    order = np.argsort(ray, kind="stable")           # iterations were appended in march order
    rec.update(ray=ray[order].astype(np.int64), leaf=leaf[order].astype(np.int64), delta_t=dt[order].astype(f32),
               rgb=rgb, visits=visits, hits=hits)
    return rec


def volume_render_backward(tree, origins, dirs, vdirs, grad_out, step_size=1e-3, background_brightness=1.0):
    """rt_kernel.cu `trace_ray_backward` (two passes per ray: pass 1 accumulates sum_j w_j c_j . g and scatters
    the colour gradients, pass 2 scatters the density gradients
        d/dsigma_i = delta_i * delta_scale * (c_i . g * T_{i+1} - sum_{j>i} w_j c_j . g - T_end * bg * sum g) ).
    -> grad w.r.t. tree.data (same shape as tree.data[:n_internal])."""
    rgba = tree.data_format is None or str(tree.data_format).upper().startswith("RGBA")
    D = tree.data_dim
    K = 1 if rgba else (D - 1) // 3
    R = np.asarray(origins).shape[0]
    grad_out = np.asarray(grad_out, dtype=f32)
    o, d, delta_scale, invdir, tmin, tmax = _setup(tree.offset, tree.invradius, origins, dirs)
    basis = sh_basis(K, vdirs) if not rgba else np.ones((R, 1), dtype=f32)
    grad = np.zeros((tree.n_internal * tree.N ** 3, D), dtype=np.float64)
    miss = (tmax < 0) | (tmin > tmax)
    accum = np.zeros(R, dtype=f32)
    for pas in (1, 2):
        light = np.ones(R, dtype=f32)
        t = tmin.copy()
        active = ~miss & (t < tmax)
        while active.any():
            a = np.nonzero(active)[0]
            pos = (o[a] + t[a][:, None] * d[a]).astype(f32)
            node, ijk, cube, rel = tree.query_unit(pos)
            smin, smax = _dda_unit(rel, invdir[a])
            delta_t = (((smax - smin) / cube).astype(f32) + f32(step_size)).astype(f32)
            sigma = tree.data[node, ijk[:, 0], ijk[:, 1], ijk[:, 2], D - 1]
            h = sigma > f32(0.0)
            if h.any():
                ah = a[h]
                flat = tree.pack_index(node[h], ijk[h])
                att = np.exp(-delta_t[h] * delta_scale[ah] * sigma[h]).astype(f32)
                weight = (light[ah] * (f32(1.0) - att)).astype(f32)
                pre, _ = _leaf_color_pre(tree, None if rgba else basis[ah], node[h], ijk[h], K, rgba)
                sig = _sigmoid(pre)
                total = (sig * grad_out[ah]).sum(axis=1).astype(f32)
                if pas == 1:
                    tmp2 = (weight[:, None] * sig * (f32(1.0) - sig) * grad_out[ah]).astype(f32)
                    for c in range(3):
                        for k in range(K):
                            np.add.at(grad[:, c * K + k], flat, (basis[ah, k] * tmp2[:, c]).astype(np.float64))
                    light[ah] = (light[ah] * att).astype(f32)
                    accum[ah] = (accum[ah] + weight * total).astype(f32)
                else:
                    light[ah] = (light[ah] * att).astype(f32)
                    accum[ah] = (accum[ah] - weight * total).astype(f32)
                    gs = (delta_t[h] * delta_scale[ah] * (total * light[ah] - accum[ah])).astype(f32)
                    np.add.at(grad[:, D - 1], flat, gs.astype(np.float64))
            t[a] = (t[a] + delta_t).astype(f32)
            active = active & (t < tmax)
        if pas == 1:
            hit = ~miss
            accum[hit] = (accum[hit] + light[hit] * f32(background_brightness) * grad_out[hit].sum(axis=1)).astype(f32)
    return grad.reshape(tree.n_internal, tree.N, tree.N, tree.N, D)


def mse_and_grad_out(im, gt):
    """octree/optimization.py:203-204: mse = mean((clamp(im, 0, 1) - gt)^2) and d mse / d im."""
    im = np.asarray(im, dtype=f32)
    gt = np.asarray(gt, dtype=f32)
    c = np.clip(im, 0.0, 1.0)
    diff = (c - gt).astype(f32)
    mse = float((diff.astype(np.float64) ** 2).mean())
    inside = (im >= 0.0) & (im <= 1.0)
    g = np.where(inside, f32(2.0) * diff / f32(im.size), f32(0.0)).astype(f32)
    return mse, g


def sgd_step(data, grad, lr):
    """torch.optim.SGD(lr, momentum=0) (octree/optimization.py:187-189,208): data <- data - lr * grad."""
    return (data - f32(lr) * grad.astype(f32)).astype(f32)


# ----------------------------------------------------------------------------------------------
# Dense-grid weight render (extraction masking_mode == "weight")
# ----------------------------------------------------------------------------------------------
def grid_weight_render(sigma_grid, origins, dirs, offset, invradius, step_size=1e-3, sigma_thresh=0.0,
                       stop_thresh=0.0, out=None):
    """svox rt_kernel.cu `grid_trace_ray` behind `_C.grid_weight_render` (octree/extraction.py:181-214):
    march every ray through the dense sigma grid [reso,reso,reso] exactly like trace_ray marches the tree
    (cell exit by _dda_unit, + step_size) and keep, per voxel, the maximum compositing weight
    light * (1 - exp(-delta_t * delta_scale * sigma)) any ray gave it."""
    grid = np.asarray(sigma_grid, dtype=f32)
    reso = grid.shape[0]
    gw = np.zeros_like(grid) if out is None else out
    R = np.asarray(origins).shape[0]
    o, d, delta_scale, invdir, tmin, tmax = _setup(np.asarray(offset, dtype=f32), np.asarray(invradius, dtype=f32),
                                                   origins, dirs)
    miss = (tmax < 0) | (tmin > tmax)
    light = np.ones(R, dtype=f32)
    t = tmin.copy()
    active = ~miss & (t < tmax)
    stopped = np.zeros(R, dtype=bool)
    while active.any():
        a = np.nonzero(active)[0]
        pos = (o[a] + t[a][:, None] * d[a]).astype(f32)
        pos = np.maximum(f32(0.0), np.minimum(f32(1.0) - f32(1e-6), pos)).astype(f32)
        pos = (pos * f32(reso)).astype(f32)
        u = np.floor(pos).astype(np.int64)
        rel = (pos - u.astype(f32)).astype(f32)
        smin, smax = _dda_unit(rel, invdir[a])
        delta_t = (((smax - smin) / f32(reso)).astype(f32) + f32(step_size)).astype(f32)
        sigma = grid[u[:, 0], u[:, 1], u[:, 2]]
        h = sigma > f32(sigma_thresh)
        if h.any():
            ah = a[h]
            att = np.exp(-delta_t[h] * delta_scale[ah] * sigma[h]).astype(f32)
            weight = (light[ah] * (f32(1.0) - att)).astype(f32)
            light[ah] = (light[ah] * att).astype(f32)
            np.maximum.at(gw, (u[h, 0], u[h, 1], u[h, 2]), weight)
            stopped[ah[light[ah] <= f32(stop_thresh)]] = True
        t[a] = (t[a] + delta_t).astype(f32)
        active = active & ~stopped & (t < tmax)
    return gw


def grid_march_visits(reso, origins, dirs, offset, invradius, step_size=1e-3):
    """The voxel visits of `grid_weight_render`'s float32 march (same setup, clamp to 1 - 1e-6, floor and
    _dda_unit), ray by ray in march order, as if no ray stopped early: dict of
        ray [V] int64, voxel [V] int64 (flat x-major index), delta_t [V] float32   one entry per visit
        delta_scale [R] float32, miss [R] bool (the ray misses the box)
    The positions depend on the ray geometry alone.  sigma selects the hits (sigma > sigma_thresh) and ends a ray
    early through stop_thresh (with stop_thresh = 0 only once its light is exactly 0), so one list serves any grid."""
    R = np.asarray(origins).shape[0]
    o, d, delta_scale, invdir, tmin, tmax = _setup(np.asarray(offset, dtype=f32), np.asarray(invradius, dtype=f32),
                                                   origins, dirs)
    miss = (tmax < 0) | (tmin > tmax)
    t = tmin.copy()
    active = ~miss & (t < tmax)
    steps = []
    while active.any():
        a = np.nonzero(active)[0]
        pos = (o[a] + t[a][:, None] * d[a]).astype(f32)
        pos = np.maximum(f32(0.0), np.minimum(f32(1.0) - f32(1e-6), pos)).astype(f32)
        pos = (pos * f32(reso)).astype(f32)
        u = np.floor(pos).astype(np.int64)
        rel = (pos - u.astype(f32)).astype(f32)
        smin, smax = _dda_unit(rel, invdir[a])
        delta_t = (((smax - smin) / f32(reso)).astype(f32) + f32(step_size)).astype(f32)
        steps.append((a, (u[:, 0] * reso + u[:, 1]) * reso + u[:, 2], delta_t))
        t[a] = (t[a] + delta_t).astype(f32)
        active[a] = t[a] < tmax[a]
    # every active ray takes one step per iteration and a ray that leaves never returns, so iteration k holds
    # visit k of each of its rays: scatter straight into ray-major order
    count = np.zeros(R, dtype=np.int64)
    for a, _, _ in steps:
        count[a] += 1
    first = np.cumsum(count) - count
    V = int(count.sum())
    ray, vox, dt = np.empty(V, np.int64), np.empty(V, np.int64), np.empty(V, f32)
    for k, (a, v, dtk) in enumerate(steps):
        at = first[a] + k
        ray[at], vox[at], dt[at] = a, v, dtk
    return dict(ray=ray, voxel=vox, delta_t=dt, delta_scale=delta_scale, miss=miss)


def build_tree_from_grid(mask, init_grid_depth, radius, center, data_dim, data_format, refine_chunk=2000000):
    """octree/extraction.py:330-353 restated literally: the voxel centres of the masked init grid
    (reso = 2^(init_grid_depth+1), x-major like torch.meshgrid(...).reshape(3,-1).T) refine the tree
    init_grid_depth times; the last level in chunks of `refine_chunk` points."""
    reso = 2 ** (init_grid_depth + 1)
    tree = N3Tree(N=2, data_dim=data_dim, depth_limit=init_grid_depth, init_reserve=1024, geom_resize_fact=1.5,
                  radius=radius, center=center, data_format=data_format)
    arr = ((np.arange(reso, dtype=f32) + f32(0.5)) / f32(reso)).astype(f32)
    xx = ((arr - tree.offset[0]) / tree.invradius[0]).astype(f32)
    yy = ((arr - tree.offset[1]) / tree.invradius[1]).astype(f32)
    zz = ((arr - tree.offset[2]) / tree.invradius[2]).astype(f32)
    idx = np.argwhere(np.asarray(mask).reshape(reso, reso, reso))
    grid = np.stack([xx[idx[:, 0]], yy[idx[:, 1]], zz[idx[:, 2]]], axis=1).astype(f32)
    for _ in range(init_grid_depth - 1):
        tree.refine_at(grid)
    if grid.shape[0] <= refine_chunk:
        tree.refine_at(grid)
    else:
        for j in range(0, grid.shape[0], refine_chunk):
            tree.refine_at(grid[j:j + refine_chunk])
    return tree, grid

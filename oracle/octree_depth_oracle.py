"""CPU oracle for depth and opacity of the octree march (pob_octree_render_depth / pob_octree_render_depth_backward).
TEST INFRASTRUCTURE ONLY, like oracle/octree_oracle.py, on which it builds.

svox has no depth output; the definitions are this project's (include/plenoctree_b200.h).  Over the contributing
visits i of a ray (sigma_i > sigma_thresh), visit i starting at t_i with step delta_t_i and weight
w_i = T_i (1 - exp(-delta_t_i * delta_scale * sigma_i)):
    acc = sum_i w_i,   depth = sum_i w_i z_i,   z_i = (t_i + delta_t_i / 2) * delta_scale
(a parameter along the ray's direction vector); early termination rescales both by 1 / (1 - T) like the colour, and a
ray that misses the box has depth = acc = 0.

The march is octree_oracle.volume_render's own (recorded by march_visits, whose rgb is volume_render's return value,
so the colour is that function's bit for bit); depth and acc are shaded from its visit list in float32 in
volume_render's operation order, t_i rebuilt as the march steps it: t_0 = tmin, t_{k+1} = fl(t_k + delta_t_k).
"""
import numpy as np

from oracle import octree_oracle as OO

f32 = np.float32


def _visit_t(tree, origins, dirs, vis):
    """float32 entry t of every visit of the list (ray-major, march order) and each visit's index within its ray"""
    _, _, _, _, tmin, _ = OO._setup(tree.offset, tree.invradius, origins, dirs)
    ray, R = vis["ray"], vis["miss"].shape[0]
    k = np.arange(ray.size) - np.searchsorted(ray, np.arange(R))[ray]
    t = np.zeros(ray.size, dtype=f32)
    cur = tmin.astype(f32).copy()
    for step in range(int(k.max()) + 1 if k.size else 0):
        sel = np.nonzero(k == step)[0]
        t[sel] = cur[ray[sel]]
        cur[ray[sel]] = (cur[ray[sel]] + vis["delta_t"][sel]).astype(f32)
    return t, k


def mid_depth(t, delta_t, delta_scale):
    """z of a visit: the midpoint of its segment, (t + delta_t / 2) * delta_scale, in float32"""
    return ((t + f32(0.5) * delta_t).astype(f32) * delta_scale).astype(f32)


def volume_render_depth(tree, origins, dirs, vdirs, step_size=1e-3, background_brightness=1.0, sigma_thresh=0.0,
                        stop_thresh=0.0, return_steps=False):
    """-> rgb [R,3] (octree_oracle.volume_render's), depth [R], acc [R] (and visits, hits per ray)"""
    vis = OO.march_visits(tree, origins, dirs, vdirs, step_size, background_brightness, sigma_thresh, stop_thresh)
    ray, R = vis["ray"], vis["miss"].shape[0]
    t, k = _visit_t(tree, origins, dirs, vis)
    sigma = tree.data.reshape(-1, tree.data_dim)[vis["leaf"], -1]
    depth = np.zeros(R, dtype=f32)
    acc = np.zeros(R, dtype=f32)
    light = np.ones(R, dtype=f32)
    for step in range(int(k.max()) + 1 if k.size else 0):
        sel = np.nonzero((k == step) & (sigma > f32(sigma_thresh)))[0]
        a, dt = ray[sel], vis["delta_t"][sel]
        att = np.exp(-dt * vis["delta_scale"][a] * sigma[sel]).astype(f32)
        weight = (light[a] * (f32(1.0) - att)).astype(f32)
        depth[a] = (depth[a] + weight * mid_depth(t[sel], dt, vis["delta_scale"][a])).astype(f32)
        acc[a] = (acc[a] + weight).astype(f32)
        light[a] = (light[a] * att).astype(f32)
    st = vis["stopped"]                       # the list of a stopped ray ends at the visit that stopped it
    scale = (f32(1.0) / (f32(1.0) - light[st])).astype(f32)
    depth[st] = (depth[st] * scale).astype(f32)
    acc[st] = (acc[st] * scale).astype(f32)
    if return_steps:
        return vis["rgb"], depth, acc, vis["visits"], vis["hits"]
    return vis["rgb"], depth, acc


def volume_render_depth_backward(tree, origins, dirs, vdirs, grad_out, step_size=1e-3, background_brightness=1.0,
                                 grad_depth=None, grad_acc=None):
    """gradient w.r.t. tree.data of <grad_out, rgb> + <grad_depth, depth> + <grad_acc, acc> (thresholds ignored, as in
    octree_oracle.volume_render_backward, which gives the colour part).  Depth and acc reach sigma only: per ray,
    accum = sum_j w_j tot_j with tot_j = z_j grad_depth + grad_acc, and each contributing visit peels its term off,
        d/dsigma_i += delta_t_i * delta_scale * (tot_i * T_{i+1} - sum_{j>i} w_j tot_j)."""
    grad = OO.volume_render_backward(tree, origins, dirs, vdirs, grad_out, step_size, background_brightness)
    if grad_depth is None and grad_acc is None:
        return grad
    vis = OO.march_visits(tree, origins, dirs, vdirs, step_size, background_brightness)
    ray, R = vis["ray"], vis["miss"].shape[0]
    gz = np.zeros(R, f32) if grad_depth is None else np.asarray(grad_depth, dtype=f32).reshape(R)
    ga = np.zeros(R, f32) if grad_acc is None else np.asarray(grad_acc, dtype=f32).reshape(R)
    t, k = _visit_t(tree, origins, dirs, vis)
    sigma = tree.data.reshape(-1, tree.data_dim)[vis["leaf"], -1]
    hit = sigma > f32(0.0)
    ds = vis["delta_scale"][ray]
    att = np.exp(-vis["delta_t"] * ds * sigma).astype(f32)
    tot = (mid_depth(t, vis["delta_t"], ds) * gz[ray] + ga[ray]).astype(f32)
    flat = grad.reshape(-1, tree.data_dim)
    n_steps = int(k.max()) + 1 if k.size else 0
    for pas in (1, 2):                        # pass 1: accum = sum_j w_j tot_j; pass 2: the sigma gradients
        light = np.ones(R, dtype=f32)
        if pas == 1:
            accum = np.zeros(R, dtype=f32)
        for step in range(n_steps):
            sel = np.nonzero((k == step) & hit)[0]
            a = ray[sel]
            weight = (light[a] * (f32(1.0) - att[sel])).astype(f32)
            light[a] = (light[a] * att[sel]).astype(f32)
            if pas == 1:
                accum[a] = (accum[a] + weight * tot[sel]).astype(f32)
            else:
                accum[a] = (accum[a] - weight * tot[sel]).astype(f32)
                gs = (vis["delta_t"][sel] * ds[sel] * (tot[sel] * light[a] - accum[a])).astype(f32)
                np.add.at(flat[:, -1], vis["leaf"][sel], gs.astype(np.float64))
    return grad

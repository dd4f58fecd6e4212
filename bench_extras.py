"""Extra measurements appended to bench.py's JSON line (keys `strong`, `tt_sh25`, `c4_extraction`, `c5_octree_opt`).

The contract line of bench.py is BASELINE configs[1] under weak scaling.  The driver only runs `bench.py --gpus N`,
so the other configurations BASELINE names are timed here, after the main region, on the same ranks:

  strong         configs[1] under the REFERENCE's batch semantics: the 4096-ray batch is global and split over the
                 ranks (nerf_sh/nerf/datasets.py:80, utils.py:518-522); every rank still draws its own 10,000
                 sparsity points (nerf_sh/train.py:77-83).  The step is replayed from a CUDA graph.
  tt_sh25        configs[2]: SH25, nerf_sh/config/tt (near/far 0/4, sparsity radius 5 / length 0.2), synthetic
                 1920x1080 poses, global batch 4096, same strong-scaling split.
  c4_extraction  configs[3]: octree.extraction at 512^3 from a random-init SH16 field, x-slabs over the ranks: the
                 sigma sweep, the sigma+SH sweep, the slab all-gather, the grid-weight render over 100 cameras, the
                 tree build and step 2 at samples_per_cell 256 (octree/extraction.py:288-394), timed per stage.
  c5_octree_opt  configs[4]: octree.optimization on a 256^3-equivalent SH16 tree, ray-parallel (row slabs per rank,
                 gradient exchange per image, replicated SGD: the reference's sequential per-image updates).
  render_eval    nerf_sh.eval's render loop: 800x800 test-mode frames through utils.render_image, chunks split over
                 the ranks.

Every timing: CUDA events on the launching stream, barrier + synchronize on both sides, max over ranks.
"""
import math
import time

import numpy as np
import torch
import torch.distributed as dist

F_SH16 = (1007104.0, 2 * 471296.0, 1007104.0)     # fwd, dgrad, wgrad FLOP per MLP-sample (SURVEY.md 8d)
F_SH25 = (1020928.0, 2 * 478208.0, 1020928.0)
F_SIGMA_ONLY = 982528.0


def _world():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def _rank():
    return dist.get_rank() if _world() > 1 else 0


def timed_ms(fn, dev, reps=1):
    """max over ranks of the device time of `reps` calls of fn()."""
    if _world() > 1:
        dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(reps):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
    if _world() > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        dist.barrier()
    return float(ms) / reps


def strong_scaling(dev, peak_tflops, steps=30, tt=False, global_batch=4096, nsp=10000):
    """global batch split over the ranks, graph-replayed steps; also times the same global batch on one rank alone
    (no collectives, every rank does it at once) so that the efficiency is self-contained."""
    from plenoctree_b200.nerf import train as T
    from plenoctree_b200.nerf.models import NerfModel
    from plenoctree_b200.nerf.rays import random_rays_np
    world, rank = _world(), _rank()
    sh_deg = 4 if tt else 3
    near, far = (0.0, 4.0) if tt else (2.0, 6.0)
    sp_len, sp_rad = (0.2, 5.0) if tt else (0.05, 1.5)
    fl = F_SH25 if tt else F_SH16
    per = global_batch // world
    model = NerfModel(sh_deg=sh_deg, num_coarse_samples=64, num_fine_samples=128, near=near, far=far, white_bkgd=True,
                      max_rays=global_batch, sparsity_npoints=nsp, device=dev)
    model.init_params(20200823)
    state = T.TrainState(model)
    nb = 64
    kw = dict(w=1920, h=1080, focal=1166.0, radius=2.5) if tt else {}
    o, d, vd, px = random_rays_np(nb * global_batch, 4242 + 7919 * rank, **kw)
    pool = torch.from_numpy(np.concatenate([o, d, vd, px], axis=1)).to(dev)
    lr = 5e-4
    out = {}

    def run(n_rays, collective):
        g = T.GraphedTrainStep(model, state, n_rays, sparsity_length=sp_len, sparsity_radius=sp_rad,
                               collective=collective)
        def one(i):
            b = (i * 37) % (nb * global_batch // n_rays)
            g.step(pool[b * n_rays:(b + 1) * n_rays], lr)
        for i in range(5):
            one(i)
        return timed_ms(one, dev, reps=steps)

    ms_n = run(per, True)
    flop = (global_batch * 256 + world * nsp) * sum(fl)
    out.update({"value": global_batch / ms_n * 1e3, "unit": "rays/s", "ms_per_step": ms_n, "n_gpus": world,
                "global_batch": global_batch, "rays_per_gpu": per, "sparsity_points_per_gpu": nsp,
                "sh_deg": sh_deg, "graph_replay": True,
                "tflops_algorithmic": flop / (ms_n * 1e-3) / 1e12,
                "frac_of_tensor_peak": flop / (ms_n * 1e-3) / 1e12 / (peak_tflops * world)})
    if world > 1:
        ms_1 = run(global_batch, False)
        out["ms_per_step_one_gpu_same_batch"] = ms_1
        out["efficiency_vs_n1"] = ms_1 / (world * ms_n)
    return out


def render_eval(dev, frames=2, hw=800):
    """a14 / nerf_sh.eval: full test-mode frames (randomized False, 64 + 128 samples) through utils.render_image;
    every chunk is split over the ranks and all-gathered (nerf_sh/nerf/utils.py:331-381, 701-706)."""
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf.utils import generate_rays, pose_spherical, render_image
    world = _world()
    model = NerfModel(sh_deg=3, num_coarse_samples=64, num_fine_samples=128, max_rays=8192, device=dev)
    model.init_params(20200823)
    focal = 0.5 * hw / math.tan(0.5 * 0.6911112070083618)
    rs = np.random.RandomState(20200823)
    poses = np.stack([pose_spherical(rs.uniform(-180, 180), rs.uniform(-90, 0), 4.0) for _ in range(frames)])
    rays = generate_rays(hw, hw, focal, poses)
    frames_dev = [Rays(*[torch.from_numpy(np.ascontiguousarray(r[i])).to(dev) for r in rays]) for i in range(frames)]
    chunk = 8192 * world

    def one(i):
        render_image(model, frames_dev[i % frames], chunk=chunk)
    one(0)
    ms = timed_ms(one, dev, reps=frames)
    flop = hw * hw * 256 * F_SH16[0]
    return {"n_gpus": world, "image": f"{hw}x{hw}", "ms_per_frame": ms, "value": hw * hw / ms * 1e3, "unit": "rays/s",
            "chunk_rays": chunk, "tflops_algorithmic": flop / (ms * 1e-3) / 1e12}


class _SynthCams:
    """100 spherical poses at radius 4, 800x800, the Blender focal (SURVEY.md 8d)."""

    def __init__(self, n=100, w=800, h=800):
        from plenoctree_b200.nerf.rays import pose_spherical
        rs = np.random.RandomState(20200823)
        self.w, self.h = w, h
        self.focal = 0.5 * w / math.tan(0.5 * 0.6911112070083618)
        self.camtoworlds = np.stack([pose_spherical(rs.uniform(-180, 180), rs.uniform(-90, 0), 4.0) for _ in range(n)])
        self.size = n


def c4_extraction(dev, peak_tflops, depth=8, samples_per_cell=256, keep_fraction=0.02):
    """octree.extraction at 2^(depth+1) cubed on a random-init SH16 field, stage by stage."""
    from plenoctree_b200 import ops
    from plenoctree_b200.nerf.models import NerfModel
    from plenoctree_b200.octree import extraction as E
    from plenoctree_b200.octree.n3tree import N3Tree
    world, rank = _world(), _rank()
    reso = 2 ** (depth + 1)
    nerf = NerfModel(sh_deg=3, num_coarse_samples=64, num_fine_samples=128, max_rays=4096, device=dev)
    nerf.init_params(20200823)
    radius, center = [1.5] * 3, [0.0] * 3
    tree = N3Tree(N=2, data_dim=49, init_refine=0, init_reserve=2200000, geom_resize_fact=1.0, depth_limit=depth,
                  radius=radius, center=center, data_format="SH16", map_location=dev)
    offset, scale = tree.offset.tolist(), tree.invradius.tolist()
    x0, nx = ops.grid_slab(reso, rank, world)
    res = {"grid": reso, "n_gpus": world, "points": reso ** 3}
    hold = {}

    def sweep_sigma(_):
        hold["sig"] = ops.eval_grid(nerf._blob(False), 3, reso, offset, scale, x0=x0, nx=nx, want_rgb=False,
                                    precision=nerf.precision, device=dev)[1]
    sweep_sigma(0)
    ms = timed_ms(sweep_sigma, dev, reps=2)
    res["sigma_sweep_ms"] = ms
    res["sigma_sweep_tflops"] = reso ** 3 * F_SIGMA_ONLY / (ms * 1e-3) / 1e12
    res["sigma_sweep_frac_of_tensor_peak"] = res["sigma_sweep_tflops"] / (peak_tflops * world)

    def sweep_raw(_):
        hold["raw"] = None
        hold["raw"] = ops.eval_grid(nerf._blob(False), 3, reso, offset, scale, x0=x0, nx=nx, want_rgb=True,
                                    precision=nerf.precision, device=dev)
    sweep_raw(0)                      # first call pays the cudaMalloc of the 26 GB / world output
    ms = timed_ms(sweep_raw, dev, reps=1)
    hold["raw"] = None
    res["sigma_sh_sweep_ms"] = ms
    res["sigma_sh_sweep_tflops"] = reso ** 3 * F_SH16[0] / (ms * 1e-3) / 1e12
    res["sigma_sh_sweep_output_gb"] = reso ** 3 * 196 / 1e9

    if world > 1:
        def gather(_):
            full = torch.empty(reso ** 3, dtype=torch.float32, device=dev)
            dist.all_gather_into_tensor(full, hold["sig"].contiguous())
            hold["full"] = full
        res["slab_allgather_ms"] = timed_ms(gather, dev)
        sig = hold["full"]
    else:
        res["slab_allgather_ms"] = 0.0
        sig = hold["sig"]
    cams = _SynthCams()

    def weights(_):
        hold["w"] = E.calculate_grid_weights(cams, sig, reso, tree.invradius, tree.offset, step_size=1e-4)
    res["grid_weights_100_cameras_ms"] = timed_ms(weights, dev)
    if world > 4:
        # Tree build and step 2 are host-driven (torch bookkeeping, caching-allocator traffic): with 8 processes that
        # hold a peer-mapped NCCL communicator they took 58 s + 71 s on the 8-GPU box (4 GPUs: 10 s + 0.73 s; 1 GPU:
        # 0.09 s + 2.6 s) — a host / driver effect, not a kernel one (DESIGN.md section 7).  The bench line stays bounded.
        res["tree_build_and_step2"] = "skipped at more than 4 ranks"
        res["total_ms"] = res["sigma_sweep_ms"] + res["slab_allgather_ms"] + res["grid_weights_100_cameras_ms"]
        return res
    # a random-init field has no surfaces: keep the `keep_fraction` heaviest voxels (a synthetic scene keeps ~2.7 %)
    w = hold["w"].reshape(-1)
    k = int(keep_fraction * w.numel())
    thresh = torch.topk(w[:: max(1, w.numel() // 4000000)], max(1, int(keep_fraction * min(w.numel(), 4000000))))[0][-1]
    mask = (w >= thresh).reshape(reso, reso, reso)
    res["occupied_voxels"] = int(mask.sum())
    t0 = time.perf_counter()
    idx = torch.nonzero(mask)
    xx, yy, zz = E._axes(reso, tree.offset, tree.invradius, dev)
    grid = torch.stack([xx[idx[:, 0]], yy[idx[:, 1]], zz[idx[:, 2]]], dim=1).contiguous()
    for _ in range(depth - 1):
        tree[grid].refine()
    for j in range(0, grid.shape[0], 2000000):
        tree[grid[j:j + 2000000]].refine()
    torch.cuda.synchronize()
    res["tree_build_ms"] = (time.perf_counter() - t0) * 1e3
    res["tree_nodes"] = int(tree.n_internal)
    res["leaves_at_max_depth"] = int((tree.depths == tree.max_depth).sum())
    args = E.default_args(samples_per_cell=samples_per_cell, init_grid_depth=depth)

    def s2(_):
        E.step2(args, tree, nerf)
    ms = timed_ms(s2, dev)
    res["step2_ms"] = ms
    res["step2_samples_per_cell"] = samples_per_cell
    res["step2_tflops"] = res["leaves_at_max_depth"] * samples_per_cell * F_SH16[0] / (ms * 1e-3) / 1e12
    res["total_ms"] = (res["sigma_sweep_ms"] + res["slab_allgather_ms"] + res["grid_weights_100_cameras_ms"] +
                       res["tree_build_ms"] + res["step2_ms"])
    del k
    return res


def c5_octree_opt(dev, depth=7, images=12, hw=800):
    """octree.optimization, ray-parallel: render + clamp-MSE gradient + scatter on this rank's pixel rows, gradient
    exchange, replicated SGD step — the reference's per-image update (octree/optimization.py:195-229)."""
    import os
    import sys
    root = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.join(root, "scripts"))
    from bench_octree import build_tree
    from plenoctree_b200.nerf.rays import pose_spherical
    from plenoctree_b200.octree import VolumeRenderer
    from plenoctree_b200.octree.optimization import exchange_gradients, row_slab
    world, rank = _world(), _rank()
    tree, n_occ, _ = build_tree(depth, dev)
    H = W = hw
    focal = 0.5 * W / math.tan(0.5 * 0.6911112070083618)
    rs = np.random.RandomState(20200823)
    poses = [pose_spherical(rs.uniform(-180, 180), rs.uniform(-90, 0), 4.0) for _ in range(8)]
    r = VolumeRenderer(tree, step_size=1e-4)
    r0, nr = row_slab(H, rank, world)
    with torch.no_grad():
        gts = [(r.render_persp(p, W, H, focal, rows=(r0, nr)) + 0.05 * torch.randn((nr, W, 3), device=dev)).clamp_(0, 1)
               for p in poses]
    sq = torch.zeros(1, dtype=torch.float64, device=dev)
    out = {"n_gpus": world, "tree": f"{2 ** (depth + 1)}^3-equivalent SH16", "nodes": int(tree.n_internal),
           "occupied_voxels": int(n_occ), "image": f"{H}x{W}",
           "dense_gradient_mb": tree.n_internal * 8 * tree.data_dim * 4 / 1e6}
    for mode in (("sparse", "dense") if world > 1 else ("dense",)):
        info = {}

        def image(i):
            r.train_persp(poses[i % 8], gts[i % 8], W, H, focal, rows=(r0, nr), sq_err=sq)
            if world > 1:
                info.update(exchange_gradients(tree, sparse=(mode == "sparse")) or {})
            tree.sgd_step(1e-3)
        for i in range(3):
            image(i)
        ms = timed_ms(image, dev, reps=images)
        out[f"ms_per_image_{mode}"] = ms
        if mode == "sparse":
            out["sparse_exchange"] = info
    best = min(v for k, v in out.items() if k.startswith("ms_per_image"))
    out["value"] = 1e3 / best
    out["unit"] = "images/s"
    out["rays_per_s"] = H * W / best * 1e3
    return out

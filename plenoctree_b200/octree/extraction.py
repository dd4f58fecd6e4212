"""Host-side mirror of `octree/extraction.py` (NeRF-SH -> PlenOctree conversion) over the CUDA library.

    reference                                        here
    calculate_grid_weights   extraction.py:181-214   calculate_grid_weights  (all cameras in one launch)
    auto_scale               extraction.py:244-286   auto_scale              (pob_eval_grid: no host grid)
    step1                    extraction.py:288-353   step1
    step2                    extraction.py:355-394   step2                   (pob_eval_cells_mean epilogue)
    main                     extraction.py:425-516   extract                 (flags arrive as an args namespace)

`args` carries the reference's flag names (extraction.py:66-176, octree/nerf/utils.py:60-253); `default_args()`
returns the reference defaults.  `nerf` is plenoctree_b200.nerf.models.NerfModel; `dataset` needs .w .h .focal
.camtoworlds [n,4,4] (and .size), like octree/nerf/datasets.py.  A vanilla NeRF (use_viewdirs) is projected to SH
in step2 (projection.py: projection_samples directions per block of leaves); SG is outside the scope of this path
and raises NotImplementedError.

Forward-facing (LLFF) scenes: the tree lives in NDC, where the model was trained, and the weight mask marches the
training cameras' rays in NDC when renderer.scene_ndc says so ('llff' in --config and not --spherify).  --z_min /
--z_max drop the grid's z slices outside [z_min, z_max] as the reference does (extraction.py:257-260,298-301).  The
reference's weight mask cannot take a cropped grid (its reshape to reso^3 fails); here the dropped slices are empty
space to the weight render: they neither occlude the rest of the grid nor enter the tree.  NDC x and y go past +-1
wherever a camera sees beyond the frustum of the reference pose, so the box (--radius / --center) must reach that far
in x and y or the tree leaves that content out (DESIGN.md §8).
"""
import ctypes
import os
import types

import numpy as np
import torch

from .. import _lib, ops
from .._lib import check, lib, ptr, stream_ptr
from .n3tree import N3Tree
from .renderer import camera_array, scene_ndc


def default_args(**kw):
    a = types.SimpleNamespace(
        output="./tree.npz", center="0 0 0", radius="1.5", alpha_thresh=0.01, max_refine_prop=0.5, z_min=None,
        z_max=None, tree_branch_n=2, init_grid_depth=8, samples_per_cell=8, is_jaxnerf_ckpt=False,
        masking_mode="weight", weight_thresh=0.001, projection_samples=10000, bbox_from_data=False,
        data_bbox_scale=1.0, autoscale=False, bbox_cube=False, bbox_scale=1.0, scale_alpha_thresh=0.01, eval=True,
        chunk=81920, renderer_step_size=1e-4, sh_deg=3, sg_dim=-1, use_viewdirs=False, num_rgb_channels=3,
        config="", spherify=False, no_early_stop=False)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _rank_world():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def _grid_sigmas(nerf, reso, offset, scale):
    """the chunked eval_points_raw loop over the dense grid (extraction.py:262-274 / 308-320) as one sweep whose
    voxel centres are generated in the kernel; returns sigma [reso^3] x-major.  With torch.distributed initialised
    every rank sweeps its x-slab (SURVEY §8e: voxel slabs, no collective in the sweep) and the slabs are all-gathered
    once so that every rank can build the (replicated) tree."""
    import torch.distributed as dist
    rank, world = _rank_world()
    x0, nx = ops.grid_slab(reso, rank, world)
    _, sig = ops.eval_grid(nerf._blob(False), nerf.sh_deg, reso, offset, scale, x0=x0, nx=nx, want_rgb=False,
                           precision=nerf.precision, device=nerf.device, posenc=nerf.posenc,
                           net_activation=nerf.net_act_code)
    if world == 1:
        return sig
    slabs = [ops.grid_slab(reso, r, world) for r in range(world)]
    if len({n for _, n in slabs}) == 1:
        full = torch.empty(reso * reso * reso, dtype=torch.float32, device=nerf.device)
        dist.all_gather_into_tensor(full, sig.contiguous())
        return full
    parts = [torch.empty(n * reso * reso, dtype=torch.float32, device=nerf.device) for _, n in slabs]
    dist.all_gather(parts, sig.contiguous())
    return torch.cat(parts)


def calculate_grid_weights(dataset, sigmas, reso, invradius, offset, step_size=1e-4, cam_chunk=4096, ndc=None):
    """extraction.py:181-214.  One launch marches the rays of every training camera through the grid and keeps the
    per-voxel maximum weight directly (atomic max); the reference renders one weight grid per camera and reduces
    with torch.max.  ndc (renderer.NDCConfig): the rays are marched in NDC (extraction.py:187-193)."""
    dev = sigmas.device
    grid = sigmas.reshape(reso, reso, reso).contiguous().float()
    wmax = torch.zeros_like(grid)
    c2ws = np.asarray(dataset.camtoworlds, dtype=np.float32)
    rank, world = _rank_world()
    c2ws = c2ws[rank::world]        # cameras are dealt to the ranks; the per-voxel maxima are joined below
    cams = camera_array(c2ws, dataset.w, dataset.h, dataset.focal, device=dev)
    o = _lib.OctreeOpts()
    o.step_size = float(step_size)
    o.background_brightness = 1.0
    o.sigma_thresh = 0.0
    o.stop_thresh = 0.0
    off = (ctypes.c_float * 3)(*[float(v) for v in offset.detach().cpu().numpy().reshape(3)])
    inv = (ctypes.c_float * 3)(*[float(v) for v in invradius.detach().cpu().numpy().reshape(3)])
    ndc_args = () if ndc is None else (ctypes.byref(_lib.Ndc(*map(float, ndc))),)
    fn = lib.pob_grid_weight_render if ndc is None else lib.pob_grid_weight_render_ndc
    for c0 in range(0, cams.shape[0], cam_chunk):
        sub = cams[c0:c0 + cam_chunk].contiguous()
        check(fn(ptr(grid), reso, ptr(sub), sub.shape[0], int(dataset.w), int(dataset.h), off, inv, ctypes.byref(o),
                 *ndc_args, ptr(wmax), None, stream_ptr()))
    if world > 1:
        import torch.distributed as dist
        dist.all_reduce(wmax, op=dist.ReduceOp.MAX)
    return wmax


def _axes(reso, offset, scale, dev):
    arr = (torch.arange(0, reso, dtype=torch.float32, device=dev) + 0.5) / reso
    return [(arr - offset[a]) / scale[a] for a in range(3)]


def z_keep(args, zz):
    """the z slices the grid keeps: zz >= z_min and zz <= z_max, the reference's zz[zz >= args.z_min] / zz[zz <=
    args.z_max] (extraction.py:257-260,298-301) as a mask over zz [reso]; None when neither flag is set"""
    z_min, z_max = getattr(args, "z_min", None), getattr(args, "z_max", None)
    if z_min is None and z_max is None:
        return None
    keep = torch.ones_like(zz, dtype=torch.bool)
    if z_min is not None:
        keep &= zz >= z_min
    if z_max is not None:
        keep &= zz <= z_max
    return keep


def auto_scale(args, center, radius, nerf):
    """extraction.py:244-286: bounding box of the voxels whose sigma passes scale_alpha_thresh (inside the z crop)."""
    reso = 2 ** args.init_grid_depth
    radius = torch.tensor(radius, dtype=torch.float32)
    center = torch.tensor(center, dtype=torch.float32)
    scale = 0.5 / radius
    offset = 0.5 * (1.0 - center / radius)
    sigmas = _grid_sigmas(nerf, reso, offset.tolist(), scale.tolist())
    keep = z_keep(args, _axes(reso, offset, scale, sigmas.device)[2])
    return _bbox_of_dense(sigmas, args.scale_alpha_thresh, reso, offset, scale, keep)


def _bbox_of_dense(sigmas, alpha_thresh, reso, offset, scale, keep=None):
    """centre and half-extent of the box around the voxel centres whose sigma reaches the alpha threshold, grown by
    half a grid step (extraction.py:276-286: the margin is 0.5 / reso in WORLD units, as in the reference).
    sigmas: [reso^3] x-major; offset / scale: the grid's world -> [0,1]^3 transform (torch float32 [3]); keep: the z
    slices of the crop (z_keep) or None."""
    approx_delta = 2.0 / reso
    sigma_thresh = -np.log(1.0 - alpha_thresh) / approx_delta
    mask = (sigmas >= sigma_thresh).reshape(reso, reso, reso)
    if keep is not None:
        mask = mask & keep
    xx, yy, zz = _axes(reso, offset.to(sigmas.device), scale.to(sigmas.device), sigmas.device)
    lc, uc = [], []
    for a, ax in enumerate((xx, yy, zz)):
        occ = mask.any(dim=tuple(d for d in range(3) if d != a))
        vals = ax[occ]
        lc.append(float(vals.min()) - 0.5 / reso)
        uc.append(float(vals.max()) + 0.5 / reso)
    lc, uc = np.asarray(lc, dtype=np.float32), np.asarray(uc, dtype=np.float32)
    return ((lc + uc) * 0.5).tolist(), ((uc - lc) * 0.5).tolist()


def step1(args, tree, nerf, dataset, refine_chunk=2000000):
    """extraction.py:288-353: dense sigma grid -> mask (sigma or weight) -> level-by-level refinement."""
    reso = 2 ** (args.init_grid_depth + 1)
    offset, scale = tree.offset, tree.invradius
    approx_delta = 2.0 / reso
    sigma_thresh = -np.log(1.0 - args.alpha_thresh) / approx_delta
    sigmas = _grid_sigmas(nerf, reso, offset.tolist(), scale.tolist())
    xx, yy, zz = _axes(reso, offset, scale, tree.device)
    keep = z_keep(args, zz)
    if args.masking_mode == "sigma":
        mask = sigmas >= sigma_thresh
    elif args.masking_mode == "weight":
        if keep is not None:            # the cropped slices are not part of the grid: empty space to the rays
            sigmas = sigmas.reshape(reso, reso, reso).masked_fill(~keep, 0.0).reshape(-1)
        grid_weights = calculate_grid_weights(dataset, sigmas, reso, tree.invradius, tree.offset,
                                              step_size=args.renderer_step_size,
                                              ndc=scene_ndc(args, dataset.w, dataset.h, dataset.focal))
        mask = grid_weights.reshape(-1) >= args.weight_thresh
        del grid_weights
    else:
        raise ValueError
    del sigmas
    grid = grid_points(mask.reshape(reso, reso, reso), keep, xx, yy, zz)
    del mask
    for _ in range(args.init_grid_depth - 1):
        tree[grid].refine()
    if grid.shape[0] <= refine_chunk:
        tree[grid].refine()
    else:
        for j in range(0, grid.shape[0], refine_chunk):
            tree[grid[j:j + refine_chunk]].refine()
    assert tree.max_depth == args.init_grid_depth
    return grid


def grid_points(mask, keep, xx, yy, zz):
    """the voxel centres of mask [reso]^3 inside the z crop (keep, or None), in x-major order: grid[mask] of the
    reference's (cropped) meshgrid"""
    if keep is not None:
        mask = mask & keep
    idx = torch.nonzero(mask)
    return torch.stack([xx[idx[:, 0]], yy[idx[:, 1]], zz[idx[:, 2]]], dim=1).contiguous()


def step2(args, tree, nerf, cells_per_launch=None):
    """extraction.py:355-394 (SH data formats): S uniform samples per finest leaf, mean of [raw_rgb, raw_sigma].
    The per-cell mean is taken in the MLP kernel's epilogue (pob_eval_cells_mean); launches cover
    `cells_per_launch` leaves (default: 2^22 points) instead of chunk // S = 320.
    A vanilla NeRF (args.use_viewdirs, nerf a projection.VanillaNerf) is projected to SH instead: each block of
    projection.CELLS_PER_BLOCK leaves takes its own set of projection_samples directions (extraction.py:217-241), and
    `cells_per_launch` (default: projection.blocks_per_launch) must be a multiple of the block."""
    rgba_tree = tree.data_format.format == 0
    import torch.distributed as dist
    S = int(args.samples_per_cell)
    leaf_ind = torch.where(tree.depths == tree.max_depth)[0]
    if args.use_viewdirs:
        from . import projection as P
        if rgba_tree:
            raise NotImplementedError("a vanilla NeRF is projected to an SH tree: sh_deg 1-4 expected")
        D = int(args.projection_samples)
        if cells_per_launch is None:
            cells_per_launch = P.blocks_per_launch(S, D, args.sh_deg) * P.CELLS_PER_BLOCK
        if cells_per_launch % P.CELLS_PER_BLOCK:
            raise ValueError(f"cells_per_launch must be a multiple of {P.CELLS_PER_BLOCK} (one direction set each)")
    elif cells_per_launch is None:
        cells_per_launch = max(1, (1 << 22) // S)
    rank, world = _rank_world()
    n = int(leaf_ind.shape[0])
    out = torch.zeros((n, tree.data_dim), dtype=torch.float32, device=tree.device)
    gen = torch.Generator(device=tree.device)
    # every rank takes a contiguous block of leaf chunks (no collective inside); each chunk draws its sample
    # positions from its own seed, so the tree does not depend on the number of ranks.  The blocks are all-gathered.
    n_chunks = (n + cells_per_launch - 1) // cells_per_launch
    per_rank = (n_chunks + world - 1) // world
    c_lo, c_hi = min(n_chunks, rank * per_rank), min(n_chunks, (rank + 1) * per_rank)
    for cid in range(c_lo, c_hi):
        i = cid * cells_per_launch
        chunk_inds = leaf_ind[i:i + cells_per_launch]
        gen.manual_seed(20200823 + cid)
        u = torch.rand((chunk_inds.shape[0], S, 3), device=tree.device, generator=gen)
        points = tree[chunk_inds].sample(S, uniforms=u)
        if args.use_viewdirs:
            out[i:i + cells_per_launch] = P.project_leaves(nerf, args.sh_deg, D, points, S, i // P.CELLS_PER_BLOCK)
        elif not rgba_tree:
            out[i:i + cells_per_launch] = ops.eval_cells_mean(nerf._blob(False), nerf.sh_deg, points.contiguous(), S,
                                                              precision=nerf.precision, posenc=nerf.posenc,
                                                              net_activation=nerf.net_act_code)
        else:
            # RGBA trees (extraction.py:378-390): sigma = mean, rgb = alpha-weighted mean with alpha of a 2/reso step
            rgb, sigma = nerf.eval_points_raw(points.reshape(-1, 3).contiguous())
            rgb = rgb.reshape(-1, S, tree.data_dim - 1)
            sigma = sigma.reshape(-1, S, 1)
            approx_delta = 2.0 / (2 ** (args.init_grid_depth + 1))
            alpha = 1.0 - torch.exp(-approx_delta * sigma)
            msum = alpha.sum(dim=1)
            rgb_avg = (rgb * alpha).sum(dim=1) / msum
            rgb_avg[msum[..., 0] < 1e-3] = 0
            out[i:i + cells_per_launch] = torch.cat([rgb_avg, sigma.mean(dim=1)], dim=-1)
    if world > 1:
        rows = per_rank * cells_per_launch            # rows of one rank's block (the last block may be short)
        mine = torch.zeros((rows, tree.data_dim), dtype=torch.float32, device=tree.device)
        lo, hi = min(n, c_lo * cells_per_launch), min(n, c_hi * cells_per_launch)
        mine[:hi - lo] = out[lo:hi]
        full = torch.empty((world * rows, tree.data_dim), dtype=torch.float32, device=tree.device)
        dist.all_gather_into_tensor(full, mine)
        out = full[:n]
    tree[leaf_ind] = out


def extract(args, nerf, dataset):
    """extraction.py:425-509 without file/flag plumbing: returns the N3Tree (saved to args.output if set)."""
    if args.sg_dim > 0:
        raise NotImplementedError("SG trees are outside the scope of this path")
    data_format = f"SH{(args.sh_deg + 1) ** 2}" if args.sh_deg > 0 else None
    if getattr(args, "bbox_from_data", False):            # extraction.py:458-462 (NSVF bbox.txt)
        assert getattr(dataset, "bbox", None) is not None  # Dataset must be NSVF
        center = ((dataset.bbox[:3] + dataset.bbox[3:6]) * 0.5).tolist()
        radius = ((dataset.bbox[3:6] - dataset.bbox[:3]) * 0.5 * args.data_bbox_scale).tolist()
    else:
        center = list(map(float, str(args.center).split()))
        if len(center) == 1:
            center *= 3
        radius = list(map(float, str(args.radius).split()))
        if len(radius) == 1:
            radius *= 3
    if args.autoscale:
        center, radius = auto_scale(args, center, radius, nerf)
    radius = [r * args.bbox_scale for r in radius]
    if args.bbox_cube:
        radius = [max(radius)] * 3
    num_rgb_channels = args.num_rgb_channels
    if args.sh_deg >= 0:
        num_rgb_channels *= (args.sh_deg + 1) ** 2
    data_dim = 1 + num_rgb_channels
    tree = N3Tree(N=args.tree_branch_n, data_dim=data_dim, init_refine=0, init_reserve=500000, geom_resize_fact=1.0,
                  depth_limit=args.init_grid_depth, radius=radius, center=center, data_format=data_format,
                  map_location=nerf.device)
    step1(args, tree, nerf, dataset)
    step2(args, tree, nerf)
    tree[:, -1:].relu_()
    tree.shrink_to_fit()
    if args.output and _rank_world()[0] == 0:   # the tree is replicated: rank 0 writes it
        tree.save(args.output, compress=False)
    return tree


# ---- `python -m plenoctree_b200.octree.extraction` (octree/extraction.py:60-176,425-516) ---------------------------------
def _define_cli_flags():
    from ..nerf import flags as F
    F.define_flags(octree=True)
    F.define({
        "output": ("string", "./tree.npz", "Output file"),
        "center": ("string", "0 0 0", "Center of volume in x y z OR single number"),
        "radius": ("string", "1.5", "1/2 side length of volume"),
        "alpha_thresh": ("float", 0.01, "Alpha threshold to keep a voxel in initial sigma thresholding"),
        "max_refine_prop": ("float", 0.5, "Max proportion of cells to refine"),
        "z_min": ("float", None, "Discard z axis points below this value, for NDC use"),
        "z_max": ("float", None, "Discard z axis points above this value, for NDC use"),
        "tree_branch_n": ("integer", 2, "Tree branch factor (2=octree)"),
        "init_grid_depth": ("integer", 8, "Initial evaluation grid (2^{x+1} voxel grid)"),
        "samples_per_cell": ("integer", 8, "Samples per cell in step 2 (3D antialiasing)"),
        "is_jaxnerf_ckpt": ("bool", False, "Whether the ckpt is from jaxnerf or not."),
        "masking_mode": ("string", "weight", "How to calculate mask when building the octree (sigma | weight)"),
        "weight_thresh": ("float", 0.001, "Weight threshold to keep a voxel"),
        "projection_samples": ("integer", 10000, "Number of rays to sample for SH projection."),
        "bbox_from_data": ("bool", False, "Use bounding box from dataset if possible"),
        "data_bbox_scale": ("float", 1.0, "Scaling factor to apply to the bounding box from dataset"),
        "autoscale": ("bool", False, "Automatic scaling, after bbox_from_data"),
        "bbox_cube": ("bool", False, "Force bbox to be a cube"),
        "bbox_scale": ("float", 1.0, "Scaling factor to apply to the bounding box at the end"),
        "scale_alpha_thresh": ("float", 0.01, "Alpha threshold for autoscale"),
        "eval": ("bool", True, "Evaluate after building the octree"),
    })
    return F


def load_nerf(FLAGS, device):
    """models.get_model_state(FLAGS, restore=True) of the octree side (octree/nerf/models.py:38-49): torch *.ckpt, or
    a flax-format checkpoint_<step> with --is_jaxnerf_ckpt.  With --use_viewdirs the vanilla model of the SH
    projection (projection.VanillaNerf)."""
    from ..nerf import checkpoints, models
    if FLAGS.use_viewdirs:
        from .projection import VanillaNerf
        posenc = (FLAGS.min_deg_point, FLAGS.max_deg_point, bool(FLAGS.legacy_posenc_order))
        mlps = checkpoints.restore_vanilla(FLAGS.train_dir, FLAGS.is_jaxnerf_ckpt, posenc, FLAGS.deg_view)
        if mlps is None:
            raise ValueError(f"no checkpoint found in {FLAGS.train_dir}")
        return VanillaNerf(mlps, posenc, FLAGS.deg_view, FLAGS.num_fine_samples, device=device)
    margs = type("A", (), dict(sh_deg=FLAGS.sh_deg, sigma_activation=FLAGS.sigma_activation,
                               net_activation=FLAGS.net_activation,
                               min_deg_point=FLAGS.min_deg_point, max_deg_point=FLAGS.max_deg_point,
                               legacy_posenc_order=FLAGS.legacy_posenc_order,
                               num_coarse_samples=FLAGS.num_coarse_samples,
                               num_fine_samples=FLAGS.num_fine_samples, near=FLAGS.near, far=FLAGS.far,
                               white_bkgd=FLAGS.white_bkgd, lindisp=FLAGS.lindisp, batch_size=min(FLAGS.chunk, 8192),
                               sparsity_npoints=0, train_dir=None))
    nerf, _ = models.get_model_state(margs, device=device, restore=False)
    ok = (checkpoints.restore_model_state_from_jaxnerf(FLAGS.train_dir, nerf) if FLAGS.is_jaxnerf_ckpt
          else checkpoints.restore_model_state(FLAGS.train_dir, nerf))
    if not ok:
        raise ValueError(f"no checkpoint found in {FLAGS.train_dir}")
    return nerf


def main(unused_argv):
    from ..nerf import datasets
    F = _define_cli_flags()
    FLAGS = F.FLAGS
    F.update_flags(FLAGS)
    if FLAGS.use_viewdirs:
        F.check_projection_scope(FLAGS)
    else:
        F.check_model_scope(FLAGS)
    torch.manual_seed(20200823)
    from .._dist import dist_finish, dist_init
    rank, _, dev = dist_init()       # under torchrun: NCCL group, this rank's GPU (x-slabs / leaf blocks / cameras)
    nerf = load_nerf(FLAGS, dev)
    assert FLAGS.data_dir  # Dataset is required now (extraction.py:455)
    dataset = datasets.get_dataset("train", FLAGS, device=dev)
    base_dir = os.path.dirname(FLAGS.output)
    if base_dir:
        os.makedirs(base_dir, exist_ok=True)
    tree = extract(FLAGS, nerf, dataset)
    if rank == 0:
        print(tree)
        if FLAGS.eval:
            from .evaluation import eval_octree
            test = datasets.get_dataset("test", FLAGS, device=dev)
            from ..nerf.lpips import load_lpips
            extra = {}
            psnr, ssim = eval_octree(tree, test, FLAGS, lpips_fn=load_lpips(dev), metrics=extra)
            print("Average PSNR", psnr, "SSIM", ssim, "LPIPS", extra["lpips"])
    dist_finish()
    return tree


if __name__ == "__main__":
    from absl import app
    _define_cli_flags()
    app.run(main)

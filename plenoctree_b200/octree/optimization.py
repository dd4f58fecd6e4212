"""Host-side mirror of `octree/optimization.py` (direct PlenOctree fine-tuning on the training images).

    reference                                             here
    run_test_step          optimization.py:191-209        run_test_step
    epoch loop             optimization.py:213-243        optimize  (SGD path: one fused launch per image +
                                                          pob_octree_sgd_step, or pob_octree_sgd_momentum_step
                                                          with --sgd_momentum / --sgd_nesterov; no autograd graph)
    --render_interval      optimization.py:163-164,202-205  run_test_step(vis_dir, i, render_interval)
    svox.N3Tree.load/save  optimization.py:168,245-248    plenoctree_b200.octree.N3Tree

Multi-GPU (SURVEY §8e, C5): every image's pixel rows are split over the ranks, each rank scatters into its own
dense gradient buffer, and the touched rows are exchanged (exchange_gradients: compacted indices + values, all-gathered)
before the replicated SGD update.  Both optimiser branches of the reference are fused with zero_grad: SGD (`--sgd`, all shipped configs) and Adam (`--nosgd`).
Forward-facing scenes train in NDC under renderer.scene_ndc's condition, the one extraction and evaluation use.
"""
import math
import os
import types

import numpy as np
import torch

from .n3tree import N3Tree
from .renderer import VolumeRenderer, scene_ndc


def default_args(**kw):
    a = types.SimpleNamespace(input="./tree.npz", output="./tree_opt.npz", render_interval=0, val_interval=2,
                              num_epochs=80, sgd=True, lr=1e7, sgd_momentum=0.0, sgd_nesterov=False,
                              nosave=False, continue_on_decrease=False, renderer_step_size=1e-4)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _rank_world():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def row_slab(height, rank, world):
    base, rem = divmod(height, world)
    r0 = rank * base + min(rank, rem)
    return r0, base + (1 if rank < rem else 0)


def exchange_gradients(tree, sparse=True):
    """Sum the ranks' gradient buffers before the replicated update (SURVEY.md 8e, C5).

    dense : one NCCL all-reduce over the whole buffer (n_internal * N^3 * data_dim floats: 160 MB for a 256^3 tree,
            1.28 GB at 512^3), whatever the image touched.
    sparse: an image's row slab only reaches the leaves its rays cross, so each rank compacts the rows of its
            buffer that received a gradient (indices + values), the ranks all-gather those lists (padded to the
            longest) and add the other ranks' rows into their own buffers.  One host read of the row counts per image.
            With 4 ranks (256^3-equivalent tree, 800x800 images; bench_extras c5_octree_opt) the four row slabs of one
            image touch 41 k / 317 k / 369 k / 44 k of the tree's 926 k rows — 83 % of all rows between them — so the
            padded lists (75 MB per rank) outweigh the 181 MB all-reduce.  A per-image gradient is dense over the
            visible leaves; the default stays dense.
    Returns a small dict describing what was exchanged."""
    import torch.distributed as dist
    rank, world = _rank_world()
    if world == 1:
        return None
    g = tree.grad_buffer()[:tree.n_internal]
    if not sparse:
        dist.all_reduce(g)
        return {"mode": "dense", "bytes_per_rank": g.numel() * 4}
    D = g.shape[-1]
    rows = g.view(-1, D)
    idx = torch.nonzero((rows != 0).any(dim=1)).squeeze(1)
    k = torch.tensor([idx.numel()], dtype=torch.int64, device=g.device)
    ks = torch.empty(world, dtype=torch.int64, device=g.device)
    dist.all_gather_into_tensor(ks, k)
    ks = ks.tolist()
    kmax = max(ks)
    if kmax == 0:
        return {"mode": "sparse", "touched_rows": ks, "bytes_per_rank": 0}
    send_i = torch.zeros(kmax, dtype=torch.int64, device=g.device)
    send_v = torch.zeros((kmax, D), dtype=g.dtype, device=g.device)
    send_i[:idx.numel()] = idx
    send_v[:idx.numel()] = rows[idx]
    all_i = torch.empty(world * kmax, dtype=torch.int64, device=g.device)
    all_v = torch.empty((world * kmax, D), dtype=g.dtype, device=g.device)
    dist.all_gather_into_tensor(all_i, send_i)
    dist.all_gather_into_tensor(all_v, send_v)
    for r in range(world):
        if r != rank and ks[r] > 0:
            rows.index_add_(0, all_i[r * kmax:r * kmax + ks[r]], all_v[r * kmax:r * kmax + ks[r]])
    return {"mode": "sparse", "touched_rows": ks, "rows_total": int(rows.shape[0]),
            "bytes_per_rank": kmax * (D * 4 + 8)}


def render_dir(input_path):
    """optimization.py:163: where --render_interval writes its validation images."""
    return os.path.splitext(input_path)[0] + "_render"


def render_vis_name(vis_dir, i, j):
    """optimization.py:205: validation view j at validation i (0 = before training, epoch + 1 after it)."""
    return f"{vis_dir}/{i:04}_{j:04}.png"


def render_vis_image(im_gt, im):
    """optimization.py:203-204: [ground truth | clamped render] side by side, scaled by 255 and truncated to uint8."""
    return (torch.cat((im_gt.to(im.device), im), dim=1) * 255).cpu().numpy().astype(np.uint8)


def run_test_step(r, test_c2w, test_gt, H, W, focal, vis_dir=None, i=0, render_interval=0):
    """optimization.py:191-209: mean PSNR of full-quality renders (fast=False) over the validation images.  With
    vis_dir and render_interval K > 0, every K-th view is also written as a [gt | render] PNG."""
    from PIL import Image
    tpsnr = 0.0
    with torch.no_grad():
        for j, (c2w, im_gt) in enumerate(zip(test_c2w, test_gt)):
            im = r.render_persp(c2w, height=H, width=W, fx=focal, fast=False).clamp_(0.0, 1.0)
            mse = ((im - im_gt.to(im.device)) ** 2).mean()
            tpsnr += -10.0 * math.log10(float(mse))
            if vis_dir is not None and render_interval > 0 and j % render_interval == 0:
                Image.fromarray(render_vis_image(im_gt, im)).save(render_vis_name(vis_dir, i, j), "PNG")
    return tpsnr / max(len(test_c2w), 1)


def train_epoch(tree, r, train_c2w, train_gt, H, W, focal, lr, adam_eps=None, momentum=0.0, nesterov=False):
    """one pass over the training images (optimization.py:216-229); returns the mean train PSNR."""
    import torch.distributed as dist
    rank, world = _rank_world()
    rows = row_slab(H, rank, world)
    sq = torch.zeros(len(train_c2w), dtype=torch.float64, device=tree.device)
    for j, (c2w, im_gt) in enumerate(zip(train_c2w, train_gt)):
        r.train_persp(c2w, im_gt, W, H, focal, rows=rows if world > 1 else None, sq_err=sq[j:j + 1])
        if world > 1:
            exchange_gradients(tree, sparse=False)   # dense wins: one image touches most visible leaves (see below)
        if adam_eps is None:
            tree.sgd_step(lr, momentum, nesterov)     # after the exchange: every rank's momentum buffer stays equal
        else:
            tree.adam_step(lr, adam_eps)
    if world > 1:
        dist.all_reduce(sq)
    mse = (sq / float(H * W * 3)).cpu().numpy()
    return float(np.mean(-10.0 * np.log10(mse)))


def optimize(args, tree, train_c2w, train_gt, test_c2w, test_gt, focal, log=print):
    """optimization.py:134-248 without dataset/flag plumbing.  train_gt/test_gt: [n,H,W,3] float tensors."""
    adam_eps = None if args.sgd else 1e-8      # optimization.py:190-193 (1e-4 only for fp16 trees)
    momentum, nesterov = float(args.sgd_momentum), bool(args.sgd_nesterov)
    if args.sgd:
        N3Tree.check_sgd_options(momentum, nesterov)     # torch.optim.SGD raises when it is built, before any render
    H, W = int(train_gt[0].shape[0]), int(train_gt[0].shape[1])
    rank, _ = _rank_world()
    if rank != 0:                       # every rank renders / trains the same replicated tree; rank 0 talks and saves
        log = lambda *a, **k: None      # noqa: E731
    K = int(getattr(args, "render_interval", 0) or 0)
    vis_dir = None
    if K > 0 and rank == 0:
        vis_dir = render_dir(args.input)
        os.makedirs(vis_dir, exist_ok=True)
    r = VolumeRenderer(tree, step_size=args.renderer_step_size, ndc=scene_ndc(args, W, H, focal))
    best_validation_psnr = run_test_step(r, test_c2w, test_gt, H, W, focal, vis_dir, 0, K)
    log(f"** initial val psnr {best_validation_psnr}")
    best_t = None
    for i in range(args.num_epochs):
        tpsnr = train_epoch(tree, r, train_c2w, train_gt, H, W, focal, args.lr, adam_eps, momentum, nesterov)
        log(f"** train_psnr {tpsnr}")
        if i % args.val_interval == args.val_interval - 1 or i == args.num_epochs - 1:
            validation_psnr = run_test_step(r, test_c2w, test_gt, H, W, focal, vis_dir, i + 1, K)
            log(f"** val psnr {validation_psnr} best {best_validation_psnr}")
            if validation_psnr > best_validation_psnr:
                best_validation_psnr = validation_psnr
                best_t = tree.clone()
            elif not args.continue_on_decrease:
                log("Stop since overfitting")
                break
    if not args.nosave and best_t is not None and args.output and rank == 0:
        best_t.save(args.output, compress=False)
    return best_t, best_validation_psnr


# ---- `python -m plenoctree_b200.octree.optimization` (octree/optimization.py:56-133,134-248) -----------------------------
def _define_cli_flags():
    from ..nerf import flags as F
    F.define_flags(octree=True)
    F.define({
        "input": ("string", "./tree.npz", "Input octree npz from extraction.py"),
        "output": ("string", "./tree_opt.npz", "Output octree npz"),
        "render_interval": ("integer", 0, "render interval"),
        "val_interval": ("integer", 2, "validation interval"),
        "num_epochs": ("integer", 80, "epochs to train for"),
        "sgd": ("bool", True, "use SGD optimizer instead of Adam"),
        "lr": ("float", 1e7, "optimizer step size"),
        "sgd_momentum": ("float", 0.0, "sgd momentum"),
        "sgd_nesterov": ("bool", False, "sgd nesterov momentum?"),
        "write_vid": ("string", None, "If specified, writes rendered video to given path (*.mp4)"),
        "split_train": ("bool", None, "If specified, splits train set instead of loading val set"),
        "split_holdout_prop": ("float", 0.2, "Proportion of images to hold out if split_train is set"),
        "nosave": ("bool", False, "If set, does not save (for speed)"),
        "continue_on_decrease": ("bool", False, "If set, continues training even if validation PSNR decreases"),
    })
    return F


def _cli_main(argv):
    main(argv)          # absl exits with main's return value; the command line exits 0 on success


def main(unused_argv):
    from ..nerf import datasets
    F = _define_cli_flags()
    FLAGS = F.FLAGS
    F.update_flags(FLAGS)
    if FLAGS.write_vid:
        raise NotImplementedError("write_vid (mp4 output) is outside the scope of this path")
    torch.manual_seed(20200823)
    np.random.seed(20200823)
    from .._dist import dist_finish, dist_init
    _, _, dev = dist_init()          # under torchrun: NCCL group, this rank's GPU (rows of every image are split)

    def get_data(stage):
        ds = datasets.get_dataset(stage, FLAGS, device=dev)
        return ds.focal, [c for c in ds.camtoworlds], [torch.from_numpy(im).to(dev) for im in ds.images]

    focal, train_c2w, train_gt = get_data("train")
    if FLAGS.split_train:
        test_sz = int(len(train_c2w) * FLAGS.split_holdout_prop)
        perm = torch.randperm(len(train_c2w)).tolist()
        test_c2w, test_gt = [train_c2w[i] for i in perm[:test_sz]], [train_gt[i] for i in perm[:test_sz]]
        train_c2w, train_gt = [train_c2w[i] for i in perm[test_sz:]], [train_gt[i] for i in perm[test_sz:]]
    else:
        test_focal, test_c2w, test_gt = get_data("val")
        assert focal == test_focal
    tree = N3Tree.load(FLAGS.input, map_location=dev)
    res = optimize(FLAGS, tree, train_c2w, train_gt, test_c2w, test_gt, focal)
    dist_finish()
    return res


if __name__ == "__main__":
    from absl import app
    _define_cli_flags()
    app.run(_cli_main)

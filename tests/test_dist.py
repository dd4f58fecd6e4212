"""Host-side multi-process logic on CPU: world_size-2 gloo rendezvous on 127.0.0.1."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from plenoctree_b200.nerf.train import allreduce_gradients, shard_batch
        from plenoctree_b200.ops import grid_slab
        # [grads | stats] bucket: rank r contributes (r+1) everywhere
        gbuf = torch.full((1000 + 8,), float(rank + 1))
        w = allreduce_gradients(gbuf)
        ok = (w == world) and torch.allclose(gbuf, torch.full_like(gbuf, 3.0))
        mean = gbuf / w            # what Adam (grad_mult = 1/world) and the stats see
        ok = ok and torch.allclose(mean, torch.full_like(mean, 1.5))
        lo, hi = shard_batch(4096, rank, world)
        ok = ok and (hi - lo == 2048) and lo == rank * 2048
        x0, nx = grid_slab(512, rank, world)
        ok = ok and (x0, nx) == (rank * 256, 256)
        # octree gradient exchange (C5): the touched-row (sparse) exchange must give the dense all-reduce's sums
        from plenoctree_b200.octree.optimization import exchange_gradients

        class FakeTree:
            n_internal = 40

            def __init__(self, seed):
                gen = torch.Generator().manual_seed(seed)
                self.g = torch.zeros(48, 2, 2, 2, 5)
                rows = torch.randperm(40 * 8, generator=gen)[:60 + 30 * seed]        # rank-dependent touched rows
                self.g.view(-1, 5)[rows] = torch.randn(rows.numel(), 5, generator=gen)

            def grad_buffer(self):
                return self.g
        want = FakeTree(0).g[:40] + FakeTree(1).g[:40]
        for sparse in (False, True):
            t = FakeTree(rank)
            info = exchange_gradients(t, sparse=sparse)
            ok = ok and info["mode"] == ("sparse" if sparse else "dense") and torch.allclose(t.g[:40], want, atol=1e-6)
            ok = ok and not t.g[40:].any()
        empty = FakeTree(rank)
        empty.g.zero_()
        ok = ok and exchange_gradients(empty, sparse=True)["bytes_per_rank"] == 0
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_two_rank_gradient_bucket_and_sharding():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]


def test_single_process_is_identity():
    from plenoctree_b200.nerf.train import allreduce_gradients, shard_batch
    from plenoctree_b200.ops import grid_slab
    g = torch.arange(10.0)
    assert allreduce_gradients(g) == 1 and torch.equal(g, torch.arange(10.0))
    with pytest.raises(ValueError):
        shard_batch(1000, 0, 3)
    assert [grid_slab(10, r, 3) for r in range(3)] == [(0, 4), (4, 3), (7, 3)]


def test_octree_row_slabs_cover_image():
    from plenoctree_b200.octree.optimization import row_slab
    for H, world in ((800, 8), (37, 4), (5, 8), (1080, 3)):
        slabs = [row_slab(H, r, world) for r in range(world)]
        assert slabs[0][0] == 0 and sum(n for _, n in slabs) == H
        for (a, n), (b, _) in zip(slabs, slabs[1:]):
            assert a + n == b


def _octree_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    # both ranks share cuda:0 (one-GPU box), so the collective is gloo on device tensors; on a multi-GPU box the
    # same code runs one rank per GPU over NCCL (scripts/bench_octree_dist.py)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import numpy as np
        from tests.support.octree_scenes import look_at_pose, make_tree, to_device_tree
        from plenoctree_b200.octree import VolumeRenderer, optimization as OPT
        torch.cuda.set_device(0)
        otree = make_tree(61, 3, "SH16")
        tree = to_device_tree(otree)
        W, H, fx = 40, 33, 50.0
        poses = [look_at_pose(s) for s in range(3)]
        gts = [torch.from_numpy(np.random.RandomState(s).uniform(0, 1, size=(H, W, 3)).astype(np.float32)) for s in range(3)]
        r = VolumeRenderer(tree, step_size=1e-3)
        psnr = OPT.train_epoch(tree, r, poses, gts, H, W, fx, 2e3)
        q.put((rank, float(psnr), tree.data[:otree.n_internal].cpu().numpy()))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_octree_epoch_two_ranks_equals_one_rank():
    """C5 ray-parallel (SURVEY §8e): pixel-row slabs per rank + one all-reduce of the dense gradient per image must
    reproduce the single-process epoch (same SGD sequence) up to fp32 summation order."""
    import numpy as np
    from tests.support.octree_scenes import look_at_pose, make_tree, to_device_tree
    from plenoctree_b200.octree import VolumeRenderer, optimization as OPT
    otree = make_tree(61, 3, "SH16")
    tree = to_device_tree(otree)
    W, H, fx = 40, 33, 50.0
    poses = [look_at_pose(s) for s in range(3)]
    gts = [torch.from_numpy(np.random.RandomState(s).uniform(0, 1, size=(H, W, 3)).astype(np.float32)) for s in range(3)]
    psnr1 = OPT.train_epoch(tree, VolumeRenderer(tree, step_size=1e-3), poses, gts, H, W, fx, 2e3)
    want = tree.data[:otree.n_internal].cpu().numpy()
    assert np.abs(want - otree.data[:otree.n_internal]).max() > 1e-3   # the epoch changed the tree
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_octree_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for rank, psnr2, data in res:
        assert abs(psnr2 - psnr1) < 1e-3, (rank, psnr1, psnr2)
        assert np.abs(data - want).max() <= 1e-4 * np.abs(want).max(), rank


def _extract_tree(cells_per_launch):
    import numpy as np
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf.models import NerfModel
    from plenoctree_b200.octree import N3Tree, extraction as E
    sh_deg = 3
    flat = O.init_flat_params(sh_deg, 20200823, bias_scale=0.05)
    nerf = NerfModel(sh_deg=sh_deg)
    nerf.set_params(np.concatenate([flat, flat]))
    args = E.default_args(init_grid_depth=4, samples_per_cell=4, masking_mode="sigma", alpha_thresh=1e-4, output=None)
    tree = N3Tree(N=2, data_dim=49, init_reserve=4096, geom_resize_fact=1.0, depth_limit=4, radius=[1.5] * 3,
                  center=[0.0] * 3, data_format="SH16")
    E.step1(args, tree, nerf, None)
    E.step2(args, tree, nerf, cells_per_launch=cells_per_launch)
    n = tree.n_internal
    return tree.child[:n].cpu().numpy(), tree.data[:n].cpu().numpy()


def _extract_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)   # both ranks share cuda:0 (see _octree_worker)
    try:
        torch.cuda.set_device(0)
        child, data = _extract_tree(500)
        q.put((rank, child, data))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_extraction_two_ranks_equals_one_rank():
    """C4 sharding (SURVEY §8e): x-slabs of the grid sweep and leaf chunks of step 2 split over ranks must give the
    same tree as one process (per-chunk sample seeds make step 2 independent of the world size)."""
    import numpy as np
    child1, data1 = _extract_tree(500)
    assert child1.shape[0] > 100 and np.abs(data1).max() > 0
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + os.getpid() % 2000
    procs = [ctx.Process(target=_extract_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for rank, child, data in res:
        assert np.array_equal(child, child1), rank
        # identical sample positions; the per-cell mean is accumulated with float atomics (order-dependent rounding)
        assert np.abs(data - data1).max() <= 1e-5 * np.abs(data1).max(), rank


def _render_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)     # both ranks share cuda:0 (see _octree_worker)
    try:
        import numpy as np
        from plenoctree_b200.nerf.models import NerfModel, Rays
        from plenoctree_b200.nerf.utils import generate_rays, pose_spherical, render_image
        torch.cuda.set_device(0)
        model = NerfModel(sh_deg=3, max_rays=512)
        model.init_params(7)
        rays = generate_rays(37, 29, 40.0, np.stack([pose_spherical(30.0, -40.0, 4.0)]))
        rgb, disp, acc = render_image(model, Rays(rays.origins[0], rays.directions[0], rays.viewdirs[0]), chunk=700)
        q.put((rank, rgb.cpu().numpy(), disp.cpu().numpy(), acc.cpu().numpy()))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_render_image_two_ranks_equals_one_rank():
    """a14 (nerf_sh/nerf/utils.py:331-381, 701-706): every chunk of an image is split over the ranks and all-gathered;
    rays are independent, so two ranks must return exactly the single-process image (ragged last chunk included)."""
    import numpy as np
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf.utils import generate_rays, pose_spherical, render_image
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 977) % 2000
    procs = [ctx.Process(target=_render_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
    model = NerfModel(sh_deg=3, max_rays=512)
    model.init_params(7)
    rays = generate_rays(37, 29, 40.0, np.stack([pose_spherical(30.0, -40.0, 4.0)]))
    rgb, disp, acc = render_image(model, Rays(rays.origins[0], rays.directions[0], rays.viewdirs[0]), chunk=700)
    for _, r_rgb, r_disp, r_acc in res:
        assert np.array_equal(r_rgb, rgb.cpu().numpy())
        assert np.array_equal(r_disp, disp.cpu().numpy()) and np.array_equal(r_acc, acc.cpu().numpy())

"""octree.optimization with torch.optim.SGD's momentum / Nesterov (`--sgd_momentum`, `--sgd_nesterov`), validation
renders (`--render_interval`) and octree.evaluation's `--write_vid`.

- CPU: a numpy restatement of the update (fp32, the buffer formed with two roundings like torch) equals
  torch.optim.SGD; replaying the executed reference run (tests/golden/ref_optimization_momentum.npz, made by
  tests/golden/make_golden_momentum.py) with it reproduces the reference's PSNR curves and best tree; the package's
  render_interval writer rebuilds every image the reference wrote, name and bytes, from the render it came from.
- GPU: octree_sgd_momentum_kernel against fp64 on the production-depth trees of tests/test_octree_march.py; optimize()
  on the golden scene against the executed reference; the two CLIs end to end.
"""
import functools
import os

import numpy as np
import pytest

from oracle import octree_oracle as OO
from tests.support.octree_scenes import _cli, _scene
from tests.support.records import record

f32, f64 = np.float32, np.float64
U24 = 2.0 ** -24
RUNS = {"momentum": False, "nesterov": True}           # golden run name -> nesterov


def sgd_momentum_step(data, grad, buf, lr, momentum, nesterov):
    """torch.optim.SGD(lr, momentum, dampening=0, nesterov) on fp32 arrays: buf <- mu*buf + g (two roundings, torch's
    buf.mul_(mu).add_(g)); d = nesterov ? g + mu*buf : buf; data <- data - lr*d.  -> (data, buf)"""
    mu = f32(momentum)
    grad = np.asarray(grad, dtype=f32)
    b = (mu * np.asarray(buf, dtype=f32)).astype(f32) + grad
    d = (grad + (mu * b).astype(f32)).astype(f32) if nesterov else b
    return (np.asarray(data, dtype=f32) - (f32(lr) * d).astype(f32)).astype(f32), b.astype(f32)


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "ref_optimization.npz")), \
        np.load(os.path.join(golden_dir, "ref_optimization_momentum.npz"))


def _golden_tree(z):
    n = z["child"].shape[0]
    tree = OO.N3Tree(N=2, data_dim=z["data0"].shape[-1], depth_limit=4, init_reserve=n, data_format="SH4")
    tree.child, tree.parent_depth, tree.n_internal = z["child"].copy(), z["parent_depth"].copy(), n
    tree.invradius, tree.offset = z["invradius"].astype(f32), z["offset"].astype(f32)
    tree.data = z["data0"].astype(f32).copy()
    return tree


_record = functools.partial(record, "parity_octree_momentum.json")


def _psnr(mse):
    return -10.0 * np.log(mse) / np.log(10.0)


# ---------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nesterov", [False, True])
def test_numpy_step_matches_torch_sgd(nesterov):
    """the restatement against torch.optim.SGD itself: buffer bit for bit, data to fp32 rounding (torch may fuse)"""
    import torch
    rs = np.random.RandomState(3)
    data = rs.normal(size=4000).astype(f32)
    p = torch.nn.Parameter(torch.from_numpy(data.copy()))
    opt = torch.optim.SGD([p], lr=0.3, momentum=0.9, nesterov=nesterov)
    buf = np.zeros_like(data)
    for _ in range(4):
        # (zeros are +0: torch's first step clones a -0 gradient, fl(mu*0 + -0) is +0)
        g = np.where(rs.rand(*data.shape) > 0.3, rs.normal(size=data.shape), 0.0).astype(f32)
        p.grad = torch.from_numpy(g.copy())
        opt.step()
        data, buf = sgd_momentum_step(data, g, buf, 0.3, 0.9, nesterov)
        tb = opt.state[p]["momentum_buffer"].numpy()
        assert np.array_equal(tb.view(np.int32), buf.view(np.int32))
        np.testing.assert_allclose(p.detach().numpy(), data, rtol=0, atol=4 * U24 * (np.abs(data).max() + 1.0))


def test_nesterov_and_momentum_errors_match_torch():
    import torch
    from plenoctree_b200.octree import N3Tree, optimization as OPT
    p = [torch.nn.Parameter(torch.zeros(3))]
    for momentum, nesterov in ((0.0, True), (-0.5, False)):
        with pytest.raises(ValueError) as want:
            torch.optim.SGD(p, lr=1.0, momentum=momentum, nesterov=nesterov)
        with pytest.raises(ValueError) as got:
            N3Tree.check_sgd_options(momentum, nesterov)
        assert str(got.value) == str(want.value)
        # optimize() raises it before touching the tree or rendering, as the reference does when it builds SGD
        args = OPT.default_args(sgd_momentum=momentum, sgd_nesterov=nesterov)
        with pytest.raises(ValueError) as got:
            OPT.optimize(args, None, [], [], [], [], 1.0)
        assert str(got.value) == str(want.value)
    assert N3Tree.check_sgd_options(0.9, True) == 0.9


def _replay(zs, lr, momentum, nesterov):
    """the reference run re-executed with the oracle march and sgd_momentum_step -> (initial val psnr, train psnrs,
    val psnrs, best data, [(validation i, view j, clamped render)])"""
    H, W, focal, step = int(zs["H"]), int(zs["W"]), float(zs["focal"]), float(zs["step_size"])
    tree = _golden_tree(zs)
    buf = np.zeros_like(tree.data)
    renders = []

    def validate(i):
        tot = 0.0
        for j, (c2w, gt) in enumerate(zip(zs["val_c2w"], zs["val_gt"])):
            im = np.clip(OO.volume_render(tree, *OO.persp_rays(c2w, W, H, focal), step_size=step).reshape(H, W, 3), 0, 1)
            renders.append((i, j, im))
            tot += _psnr(float(((im - gt).astype(f32) ** 2).mean()))
        return tot / len(zs["val_c2w"])
    init = validate(0)
    best, best_data, train, val = init, None, [], []
    for ep in range(int(zs["epochs"])):
        tot = 0.0
        for c2w, gt in zip(zs["train_c2w"], zs["train_gt"]):
            rays = OO.persp_rays(c2w, W, H, focal)
            im = OO.volume_render(tree, *rays, step_size=step)
            mse, g = OO.mse_and_grad_out(im.reshape(H, W, 3), gt)
            grad = OO.volume_render_backward(tree, *rays, g.reshape(-1, 3), step_size=step)
            tree.data, buf = sgd_momentum_step(tree.data, grad, buf, lr, momentum, nesterov)
            tot += _psnr(mse)
        train.append(tot / len(zs["train_c2w"]))
        val.append(validate(ep + 1))
        if val[-1] > best:
            best, best_data = val[-1], tree.data.copy()
    return init, train, val, best_data, renders


@pytest.mark.parametrize("run", list(RUNS))
def test_momentum_loop_matches_executed_reference(golden_dir, run):
    """octree/optimization.py `main` was EXECUTED with --sgd_momentum 0.9 (and --sgd_nesterov): replaying it with the
    oracle pieces and sgd_momentum_step gives the reference's PSNR curves and saved tree."""
    zs, zm = _golden(golden_dir)
    assert list(zm[f"{run}_flags"]) == ["--sgd_momentum", "0.9", "--sgd_nesterov" if RUNS[run] else "--nosgd_nesterov"]
    init, train, val, best_data, _ = _replay(zs, float(zm["lr"]), float(zm["momentum"]), RUNS[run])
    assert abs(init - float(zm[f"{run}_initial_val_psnr"])) < 2e-4
    np.testing.assert_allclose(train, zm[f"{run}_train_psnr"], rtol=0, atol=2e-4)
    np.testing.assert_allclose(val, zm[f"{run}_val_psnr"], rtol=0, atol=2e-4)
    assert zm[f"{run}_train_psnr"][-1] > zm[f"{run}_train_psnr"][0] + 0.5 and best_data is not None    # it learns
    ref = zm[f"{run}_data_best"]
    assert np.abs(best_data - ref).max() < 2e-5 * np.abs(ref).max()


@pytest.mark.parametrize("run", list(RUNS))
def test_render_interval_images_match_the_reference_writes(golden_dir, run):
    """--render_interval 1: the reference wrote `<input stem>_render/{i:04}_{j:04}.png` for every validation view;
    the package's name and image builders, fed the render each image came from, give the same names and bytes."""
    import torch
    from plenoctree_b200.octree.optimization import render_dir, render_vis_image, render_vis_name
    zs, zm = _golden(golden_dir)
    names, images, renders = zm[f"{run}_vis_names"], zm[f"{run}_vis_images"], zm[f"{run}_vis_renders"]
    nv = len(zs["val_c2w"])
    assert len(names) == nv * (int(zs["epochs"]) + 1)
    scene = os.path.join(os.sep, "scene")
    for k, (name, image, render) in enumerate(zip(names, images, renders)):
        i, j = divmod(k, nv)
        assert os.path.relpath(render_vis_name(render_dir(os.path.join(scene, "tree.npz")), i, j), scene) == name
        got = render_vis_image(torch.from_numpy(zs["val_gt"][j]), torch.from_numpy(render).clamp_(0.0, 1.0))
        assert got.dtype == np.uint8 and got.shape == image.shape
        assert np.array_equal(got, image), (name, int((got != image).sum()))
    # the recorded renders are the replay's validation renders
    _, _, _, _, replayed = _replay(zs, float(zm["lr"]), float(zm["momentum"]), RUNS[run])
    assert len(replayed) == len(renders)
    for (i, j, im), render in zip(replayed, renders):
        assert np.abs(im - np.clip(render, 0, 1)).max() < 1e-5, (i, j)


# ---------------------------------------------------------------------------------------------------------
# GPU: the kernel against fp64
# ---------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _production_tree(name):
    from tests.support.octree_scenes import _build
    return _build(name)[0]


def _bound(data, g, b, lr, mu, nesterov):
    """fp64 expected data and the per-element bound on the kernel's error, from the kernel's own fp32 inputs.
    b' = fl(fl(mu b) + g) is off B = mu b + g by <= u (mu |b| + |B|); Nesterov's d = fma(mu, b', g) is off
    D = g + mu B by <= mu |b' - B| + u |D|; data' = fma(-lr, d, data) adds u |data - lr D|.  Against the unit
    u (|data| + lr (|g| + 2 mu |b|)) this is at most c = 2 (plain) and 2 + 3 mu (Nesterov) of it."""
    data, g, b = data.astype(f64), g.astype(f64), b.astype(f64)
    B = mu * b + g
    eb = U24 * (mu * np.abs(b) + np.abs(B))
    D, ed = (g + mu * B, mu * eb + U24 * np.abs(g + mu * B)) if nesterov else (B, eb)
    want = data - lr * D
    bound = (lr * ed + U24 * np.abs(want)) * (1.0 + 2.0 ** -20) + 2.0 ** -149
    unit = U24 * (np.abs(data) + lr * (np.abs(g) + 2.0 * mu * np.abs(b)))
    c = 2.0 + 3.0 * mu if nesterov else 2.0
    return want, bound, unit, c


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n2_d8_sh16", "n2_d9_sh4", "n3_d4_sh16", "n4_d3_sh9", "chain_d26_rgba"])
@pytest.mark.parametrize("nesterov", [False, True])
def test_momentum_kernel_matches_fp64(name, nesterov):
    import torch
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    otree = _production_tree(name)
    n = otree.n_internal * otree.N ** 3 * otree.data_dim
    if name.startswith("n3"):
        assert n % 4 != 0                                      # the scalar tail runs
    rs = np.random.RandomState(sum(map(ord, name)) + nesterov)
    pad = 37
    canary = np.float32(-1234.5)
    lr, mu = f32(0.05), f32(0.9)

    def draw():
        x = (rs.normal(size=n) * 10.0 ** rs.uniform(-3, 1, size=n)).astype(f32)
        x[rs.rand(n) < 0.3] = 0.0
        return x
    host = {"data": otree.data[:otree.n_internal].reshape(-1).astype(f32), "g": draw(), "b": draw()}
    dev = {}
    for k, v in host.items():
        t = torch.full((n + pad,), float(canary), dtype=torch.float32, device="cuda")
        t[:n] = torch.from_numpy(v).cuda()
        dev[k] = t
    worst, moved_b_only = 0.0, 0
    for step in range(3):
        if step:
            dev["g"][:n] = torch.from_numpy(draw()).cuda()
        d0, g0, b0 = (dev[k][:n].cpu().numpy() for k in ("data", "g", "b"))
        check(lib.pob_octree_sgd_momentum_step(ptr(dev["data"]), ptr(dev["g"]), ptr(dev["b"]), n, float(lr), float(mu),
                                               int(nesterov), stream_ptr()))
        torch.cuda.synchronize()
        d1, g1, b1 = (dev[k].cpu().numpy() for k in ("data", "g", "b"))
        for x in (d1, g1, b1):
            assert np.array_equal(x[n:].view(np.int32), np.full(pad, canary).view(np.int32))   # nothing past n
        d1, g1, b1 = d1[:n], g1[:n], b1[:n]
        moved = (g0 != 0) | (b0 != 0)
        assert 0 < (~moved).sum() < n
        # the buffer: numpy's two-rounding form, bit for bit
        assert np.array_equal(b1.view(np.int32), ((mu * b0).astype(f32) + g0).view(np.int32))
        # untouched where g = b = 0, and the gradient is cleared everywhere
        assert np.array_equal(d1[~moved].view(np.int32), d0[~moved].view(np.int32))
        assert not g1.any()
        want, bound, unit, c = _bound(d0, g0, b0, f64(lr), f64(mu), nesterov)
        err = np.abs(d1[moved].astype(f64) - want[moved])
        assert (err <= bound[moved]).all(), float((err / bound[moved]).max())
        assert (bound <= c * unit * (1.0 + 2.0 ** -20) + 2.0 ** -149).all()
        worst = max(worst, float((err / np.maximum(unit[moved], 1e-300)).max()))
        # momentum moves elements whose gradient is 0
        only_b = (g0 == 0) & (b0 != 0)
        moved_b_only += int((d1[only_b] != d0[only_b]).sum())
        assert (d1[only_b] != d0[only_b]).mean() > 0.5
    _record(f"kernel_{name}_{'nesterov' if nesterov else 'momentum'}", {
        "n": int(n), "err_in_unit_max": worst, "c": c, "moved_by_buffer_only": moved_b_only})


@pytest.mark.gpu
def test_sgd_step_momentum_zero_is_the_plain_kernel_and_buffer_lifetime():
    """N3Tree.sgd_step(lr, 0.0) is pob_octree_sgd_step bit for bit and allocates no buffer; with momentum the buffer
    starts at zero, persists across steps, and clone() / shrink_to_fit() drop it."""
    import torch
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    from tests.support.octree_scenes import to_device_tree
    otree = _production_tree("n3_d4_sh16")
    tree = to_device_tree(otree)
    n = otree.n_internal * otree.N ** 3 * otree.data_dim
    rs = np.random.RandomState(8)
    g = np.where(rs.rand(*tree.data.shape) > 0.3, rs.normal(size=tree.data.shape), 0.0).astype(f32)
    data = tree.data.clone()
    grad = torch.from_numpy(g).cuda()
    tree.grad_buffer().copy_(grad)
    tree.sgd_step(1e-2, 0.0)
    check(lib.pob_octree_sgd_step(ptr(data), ptr(grad), n, 1e-2, stream_ptr()))
    assert torch.equal(tree.data.view(torch.int32), data.view(torch.int32))
    assert getattr(tree, "_sgd_buf", None) is None and not tree.grad_buffer().any()
    # momentum: two steps through the tree equal two steps of the numpy restatement
    want, buf = tree.data[:otree.n_internal].cpu().numpy(), np.zeros_like(g[:otree.n_internal])
    for s in range(2):
        gs = np.roll(g, s, axis=0)
        tree.grad_buffer().copy_(torch.from_numpy(gs).cuda())
        tree.sgd_step(1e-2, 0.9, nesterov=True)
        want, buf = sgd_momentum_step(want, gs[:otree.n_internal], buf, 1e-2, 0.9, True)
    assert np.array_equal(tree._sgd_buf[:otree.n_internal].cpu().numpy().view(np.int32), buf.view(np.int32))
    np.testing.assert_allclose(tree.data[:otree.n_internal].cpu().numpy(), want, rtol=0,
                               atol=4 * U24 * (np.abs(want).max() + 1.0))
    assert tree.clone()._sgd_buf is None and tree._sgd_buf is not None
    tree.shrink_to_fit()
    assert tree._sgd_buf is None
    with pytest.raises(ValueError, match="Nesterov momentum requires a momentum"):
        tree.sgd_step(1.0, 0.0, nesterov=True)


# ---------------------------------------------------------------------------------------------------------
# GPU: end to end
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("run", list(RUNS))
def test_optimize_matches_executed_reference(golden_dir, tmp_path, run):
    """optimize() on the device, on the golden scene with the reference run's flags, against the executed reference:
    PSNR curves and best tree at the bars of the CPU replay (2e-4 dB, 2e-5 of the largest value), and the
    --render_interval PNGs (names exact, bytes within the one-LSB truncation of a render equal up to float rounding)."""
    import torch
    from PIL import Image
    from tests.support.octree_scenes import to_device_tree
    from plenoctree_b200.octree import optimization as OPT
    zs, zm = _golden(golden_dir)
    H, W, focal, step = int(zs["H"]), int(zs["W"]), float(zs["focal"]), float(zs["step_size"])
    tree = to_device_tree(_golden_tree(zs))
    to = lambda a: [torch.from_numpy(x).cuda() for x in a]       # noqa: E731
    args = OPT.default_args(input=str(tmp_path / "tree.npz"), num_epochs=int(zs["epochs"]), val_interval=1,
                            lr=float(zm["lr"]), sgd_momentum=float(zm["momentum"]), sgd_nesterov=RUNS[run],
                            continue_on_decrease=True, renderer_step_size=step, nosave=True, render_interval=1)
    logs = []
    best_t, _ = OPT.optimize(args, tree, list(zs["train_c2w"]), to(zs["train_gt"]), list(zs["val_c2w"]),
                             to(zs["val_gt"]), focal, log=logs.append)
    init = [float(l.split()[-1]) for l in logs if l.startswith("** initial val psnr")][0]
    train = [float(l.split()[-1]) for l in logs if l.startswith("** train_psnr")]
    val = [float(l.split()[3]) for l in logs if l.startswith("** val psnr")]
    d_psnr = max(abs(init - float(zm[f"{run}_initial_val_psnr"])),
                 float(np.abs(np.array(train) - zm[f"{run}_train_psnr"]).max()),
                 float(np.abs(np.array(val) - zm[f"{run}_val_psnr"]).max()))
    ref = zm[f"{run}_data_best"]
    d_data = float(np.abs(best_t.data.cpu().numpy() - ref).max() / np.abs(ref).max())
    # the PNGs: the reference's names, and its bytes up to the 8-bit truncation of renders equal to float rounding
    names = sorted(os.path.relpath(os.path.join(dp, f), str(tmp_path)) for dp, _, fs in os.walk(tmp_path) for f in fs)
    assert names == sorted(zm[f"{run}_vis_names"])
    lsb = 0
    for name, want in zip(zm[f"{run}_vis_names"], zm[f"{run}_vis_images"]):
        got = np.asarray(Image.open(str(tmp_path / name)))
        assert got.shape == want.shape and got.dtype == np.uint8
        lsb = max(lsb, int(np.abs(got.astype(int) - want.astype(int)).max()))
    _record(f"optimize_{run}", {"psnr_max_abs_diff_db": d_psnr, "data_best_rel_diff": d_data, "png_max_lsb": lsb})
    assert d_psnr < 2e-4, d_psnr                 # the CPU replay's bars
    assert d_data < 2e-5, d_data
    assert lsb <= 1, lsb
    # without --render_interval nothing is written
    args.render_interval, args.input = 0, str(tmp_path / "quiet" / "tree.npz")
    OPT.optimize(args, to_device_tree(_golden_tree(zs)), list(zs["train_c2w"]), to(zs["train_gt"]),
                 list(zs["val_c2w"]), to(zs["val_gt"]), focal, log=lambda *a: None)
    assert not (tmp_path / "quiet").exists()


@pytest.mark.gpu
def test_cli_momentum_render_interval_and_write_vid(tmp_path):
    """`python -m octree.optimization ... --sgd_momentum 0.9 --sgd_nesterov --render_interval 2` writes the [gt |
    render] PNGs of validation views 0 and 2 at every validation and a tree; `python -m octree.evaluation ...
    --write_vid v.mp4` writes one frame per test view (or says that no encoder is available)."""
    from PIL import Image
    common = _scene(tmp_path)
    out = _cli("octree.optimization", common + [
        "--input", str(tmp_path / "tree.npz"), "--output", str(tmp_path / "tree_opt.npz"), "--num_epochs", "2",
        "--val_interval", "1", "--lr", "1e3", "--sgd_momentum", "0.9", "--sgd_nesterov", "--render_interval", "2",
        "--continue_on_decrease"])
    assert os.path.exists(tmp_path / "tree_opt.npz"), out[-2000:]
    vis = tmp_path / "tree_render"
    assert sorted(os.listdir(vis)) == [f"{i:04}_{j:04}.png" for i in range(3) for j in (0, 2)]
    for f in os.listdir(vis):
        im = np.asarray(Image.open(str(vis / f)))
        assert im.shape == (32, 64, 3) and im.dtype == np.uint8
    gt = np.asarray(Image.open(str(tmp_path / "scene" / "val" / "r_2.png")))[..., :3]
    assert np.abs(np.asarray(Image.open(str(vis / "0002_0002.png")))[:, :32].astype(int) - gt).max() <= 1
    out = _cli("octree.evaluation", common + ["--input", str(tmp_path / "tree_opt.npz"),
                                              "--write_vid", str(tmp_path / "v.mp4")])
    if "* No mp4 encoder available" in out:
        assert not os.path.exists(tmp_path / "v.mp4") or os.path.getsize(tmp_path / "v.mp4") == 0
        return
    import cv2
    cap = cv2.VideoCapture(str(tmp_path / "v.mp4"))
    frames = 0
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        assert fr.shape == (32, 32, 3)
        frames += 1
    cap.release()
    assert frames == 2

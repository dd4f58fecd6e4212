"""SH projection of a vanilla NeRF (use_viewdirs) in octree extraction: scope, checkpoints, the executed reference
(tests/golden/ref_projection.npz) and, on the GPU, the point stage, the projection kernel against fp64, recovery of a
known function and the README command end to end."""
import math
import os
import types

import numpy as np
import pytest
import torch

from oracle import nerf_sh_oracle as O
from oracle import projection_oracle as PJ

U = 2.0 ** -24   # fp32 unit roundoff


def _args(**kw):
    a = dict(use_viewdirs=True, sh_deg=4, sg_dim=-1, dataset="blender", net_depth=8, net_width=256, skip_layer=4,
             net_depth_condition=1, net_width_condition=128, deg_view=4, min_deg_point=0, max_deg_point=10,
             legacy_posenc_order=False, num_coarse_samples=64, num_fine_samples=128, net_activation="ReLU",
             rgb_activation="Sigmoid", sigma_activation="ReLU", render_path=False, spherify=False)
    a.update(kw)
    return types.SimpleNamespace(**a)


# ---- CPU ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(), dict(sh_deg=1), dict(sh_deg=2), dict(sh_deg=3), dict(deg_view=0),
                                dict(deg_view=10), dict(min_deg_point=2, max_deg_point=8, legacy_posenc_order=True),
                                dict(num_coarse_samples=256, num_fine_samples=768), dict(num_fine_samples=0),
                                dict(sigma_activation="softplus"), dict(dataset="nsvf"), dict(net_activation="relu")])
def test_projection_scope_accepts(kw):
    from plenoctree_b200.nerf import flags as F
    F.check_projection_scope(_args(**kw))


@pytest.mark.parametrize("kw,match", [
    (dict(sh_deg=0), "sh_deg"), (dict(sh_deg=-1), "sh_deg"), (dict(sh_deg=5), "sh_deg"),
    (dict(net_depth_condition=2), "condition"), (dict(net_width_condition=256), "condition"),
    (dict(deg_view=-1), "deg_view"), (dict(deg_view=33), "deg_view"), (dict(net_activation="elu"), "relu"),
    (dict(rgb_activation="relu"), "relu"), (dict(sg_dim=4), "spherical"), (dict(net_depth=6), "trunk"),
    (dict(max_deg_point=12), "posenc"), (dict(num_coarse_samples=512, num_fine_samples=1024), "num_coarse"),
    (dict(sigma_activation="exp"), "sigma_activation")])
def test_projection_scope_refuses(kw, match):
    from plenoctree_b200.nerf import flags as F
    with pytest.raises(NotImplementedError, match=match):
        F.check_projection_scope(_args(**kw))


def test_check_scope_still_refuses_use_viewdirs():
    from plenoctree_b200.nerf import flags as F
    with pytest.raises(NotImplementedError, match="use_viewdirs"):
        F.check_scope(_args())
    # check_scope builds an elu trunk for NeRF-SH; the projection refuses it itself
    F.check_scope(_args(use_viewdirs=False, net_activation="elu"))
    with pytest.raises(NotImplementedError, match="projection kernel is built for a relu trunk"):
        F.check_projection_scope(_args(net_activation="elu"))


def test_proj_preset_and_file_on_disk_wins(tmp_path):
    import yaml
    from plenoctree_b200.nerf import flags as F
    more = dict(image_batching=True, factor=4, white_bkgd=False, batch_size=8, randomized=False, max_steps=1)
    args = _args(config="nerf_sh/config/misc/proj", use_viewdirs=False, sh_deg=3, **more)
    F.update_flags(args)
    assert args.use_viewdirs is True and args.sh_deg == 4 and args.dataset == "blender" and args.factor == 0
    (tmp_path / "proj.yaml").write_text(yaml.safe_dump({"sh_deg": 2, "use_viewdirs": True}))
    args = _args(config=str(tmp_path / "proj"), **more)
    F.update_flags(args)
    assert args.sh_deg == 2


def test_vanilla_checkpoints_round_trip(tmp_path):
    from plenoctree_b200.nerf import checkpoints as C
    pe = (1, 9, True)
    mlps = {"MLP_0": PJ.init_params(1, pe, 3), "MLP_1": PJ.init_params(2, pe, 3)}
    flax_dir = tmp_path / "flax"
    flax_dir.mkdir()
    (flax_dir / "checkpoint_5").write_bytes(
        C.msgpack_serialize({"optimizer": {"target": {"params": C.vanilla_to_flax_params(mlps)}}}))
    torch_dir = tmp_path / "torch"
    torch_dir.mkdir()
    torch.save({"model": {k: torch.from_numpy(np.ascontiguousarray(v))
                          for k, v in C.vanilla_to_torch_state_dict(mlps).items()}}, torch_dir / "000005.ckpt")
    for got in (C.restore_vanilla(str(flax_dir), True, pe, 3), C.restore_vanilla(str(torch_dir), False, pe, 3)):
        assert sorted(got) == ["MLP_0", "MLP_1"]
        for m in mlps:
            assert len(got[m]) == 12
            for (k0, b0), (k1, b1) in zip(mlps[m], got[m]):
                assert k1.dtype == np.float32 and np.array_equal(k0, k1) and np.array_equal(b0, b1)
    assert C.restore_vanilla(str(tmp_path), True, pe, 3) is None and C.restore_vanilla(str(tmp_path), False) is None
    sd = C.vanilla_to_torch_state_dict(mlps)
    assert sd["MLP_1.condition_layers.0.weight"].shape == (128, 256 + 3 + 18)
    assert sd["MLP_0.bottleneck_layer.weight"].shape == (256, 256) and sd["MLP_0.rgb_layer.weight"].shape == (3, 128)


@pytest.mark.parametrize("bad,match", [((10, 4), "Dense_10.*deg_view"), ((0, 0), "Dense_0.*min_deg_point"),
                                       ((11, 4), "Dense_11"), ((9, 4), "Dense_9")])
def test_vanilla_wrong_shapes_are_refused(bad, match):
    from plenoctree_b200.nerf import checkpoints as C
    mlps = {"MLP_0": PJ.init_params(1)}
    i, _ = bad
    k, b = mlps["MLP_0"][i]
    mlps["MLP_0"][i] = (np.zeros((k.shape[0] + 6, k.shape[1]) if i in (0, 10) else (k.shape[0], k.shape[1] + 1),
                                 np.float32), b if i in (0, 10) else np.zeros(b.shape[0] + 1, np.float32))
    with pytest.raises(ValueError, match=match):
        C.vanilla_from_flax_params(C.vanilla_to_flax_params(mlps))
    with pytest.raises(ValueError, match=match):
        C.vanilla_from_torch_state_dict(C.vanilla_to_torch_state_dict(mlps))
    with pytest.raises(ValueError, match="deg_view"):
        C.vanilla_from_flax_params(C.vanilla_to_flax_params({"MLP_0": PJ.init_params(1)}), deg_view=5)


def test_missing_fine_mlp_and_too_many_blocks_are_refused():
    from plenoctree_b200 import _lib
    from plenoctree_b200.octree.projection import VanillaNerf
    with pytest.raises(ValueError, match="MLP_1"):
        VanillaNerf({"MLP_0": PJ.init_params(1)}, num_fine_samples=128)
    buf = np.zeros(4, np.float32)
    assert _lib.lib.pob_sh_proj_directions(0, 0, 65536, 10, 4, 0, 4, buf.ctypes.data, None, buf.ctypes.data,
                                           buf.ctypes.data, None) != 0
    assert "65535" in _lib.lib.pob_last_error().decode()
    assert _lib.lib.pob_sh_proj_points_workspace_bytes(-1) == -1
    assert _lib.lib.pob_sh_proj_points_workspace_bytes(1) > _lib.lib.pob_sh_proj_points_workspace_bytes(0)


def test_mismatched_deg_view_is_refused_before_upload(monkeypatch):
    """VanillaNerf checks Dense_10's rows against deg_view (pob_sh_proj_directions reads 3 + 6 deg_view rows of
    W10_e) before it uploads or packs anything"""
    from plenoctree_b200.octree import projection as P
    mlps = {"MLP_0": PJ.init_params(1), "MLP_1": PJ.init_params(2)}              # deg_view 4: 283 rows

    def no_upload(*a, **k):
        raise AssertionError("uploaded before the Dense_10 check")
    monkeypatch.setattr(torch.Tensor, "to", no_upload)
    monkeypatch.setattr(P.ops, "pack_weights", no_upload)
    for nfs, name in ((0, "MLP_0"), (128, "MLP_1")):
        with pytest.raises(ValueError, match=f"{name}/Dense_10 has 283 input rows, deg_view=5 needs 289"):
            P.VanillaNerf(mlps, deg_view=5, num_fine_samples=nfs)


def test_oracle_reproduces_the_executed_reference(golden_dir):
    z = np.load(os.path.join(golden_dir, "ref_projection.npz"))
    layers = PJ.init_params(int(z["seeds"][1]))                  # MLP_1: eval_points_raw's fine MLP
    pts = torch.from_numpy(z["points"])
    dirs = PJ.spher2cart(torch.from_numpy(z["theta"]), torch.from_numpy(z["phi"]))
    assert np.array_equal(dirs.numpy(), z["dirs"])
    raw_rgb, raw_sigma = PJ.eval_points_raw(layers, pts, dirs)
    scale = np.abs(z["raw_rgb"]).max()
    assert np.abs(raw_rgb.numpy() - z["raw_rgb"]).max() <= 1e-5 * scale
    assert np.abs(raw_sigma.numpy() - z["raw_sigma"]).max() <= 1e-5 * np.abs(z["raw_sigma"]).max()
    for deg in range(1, 5):
        coeffs, sigma = PJ.project(layers, pts, dirs, deg)
        ref = z[f"coeffs_deg{deg}"]
        assert coeffs.reshape(pts.shape[0], -1).shape == ref.shape
        assert np.abs(coeffs.reshape(pts.shape[0], -1).numpy() - ref).max() <= 1e-5 * np.abs(ref).max(), deg
        assert np.array_equal(sigma.numpy(), raw_sigma.numpy())
    # rows of a split branch: a_p + W10_e posenc(d) is the condition layer's input
    a = PJ.a_p([(k.astype(np.float64), b.astype(np.float64)) for k, b in layers], pts.double())
    enc = PJ.PO.posenc(dirs.double(), 0, 4)
    z64 = torch.relu(a[:, None] + enc[None] @ torch.from_numpy(layers[10][0][256:]).double())
    rgb64 = z64 @ torch.from_numpy(layers[11][0]).double() + torch.from_numpy(layers[11][1]).double()
    assert np.abs(rgb64.numpy() - z["raw_rgb"]).max() <= 1e-5 * scale


def test_evalsh_is_the_basis_the_tree_renders_with(golden_dir):
    """sh_proj.EvalSH (the projection's basis) equals nerf_sh/nerf/sh.py's (the octree march's) for all 25
    functions in fp64; otherwise a projected tree would render a different function."""
    z = np.load(os.path.join(golden_dir, "ref_projection.npz"))
    ours = O.sh_basis(4, torch.from_numpy(z["basis_dirs"])).numpy()
    assert ours.shape == z["evalsh"].shape == (64, 25)
    assert np.abs(ours - z["evalsh"]).max() <= 1e-15


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _model(seed=11, pe=(0, 10, False), deg_view=4):
    from plenoctree_b200.octree.projection import VanillaNerf
    layers = PJ.init_params(seed, pe, deg_view)
    return layers, VanillaNerf({"MLP_0": layers}, pe, deg_view, num_fine_samples=0)


def _points(n, seed=3):
    rs = np.random.RandomState(seed)
    return torch.from_numpy(rs.uniform(-1.2, 1.2, size=(n, 3)).astype(np.float32)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("pe", [(0, 10, False), (2, 7, True)])
def test_point_stage_sigma_and_a(pe):
    """One trunk pass (the saving fp16 forward) gives raw sigma bit-identical to the sigma sweeps' forward on the
    same blob, and a_p = h7 W + b within the fp16 point-evaluation bound of tests/test_eval_points.py."""
    from plenoctree_b200 import ops
    from tests.support.eval_stages import TOL_FP16_ANY
    layers, nerf = _model(12, pe)
    pts = _points(3000)                                     # not a multiple of the 128-row tile
    a, sig = nerf.point_stage(pts)
    _, sig_raw = ops.eval_points_raw(nerf._blob(False), -1, pts, want_rgb=False, posenc=pe)
    cells = ops.eval_cells_mean(nerf._blob(False), -1, pts, 1, posenc=pe)
    assert torch.equal(sig, sig_raw.reshape(-1))
    assert torch.equal(sig, cells[:, 3]) and not bool((cells[:, :3] != 0).any())
    torch.cuda.synchronize()
    l64 = [(k.astype(np.float64), b.astype(np.float64)) for k, b in layers]
    a64 = PJ.a_p(l64, pts.cpu().double(), pe).numpy()
    err = np.abs(a.cpu().numpy() - a64).max()
    assert err <= TOL_FP16_ANY * np.abs(a64).max(), err
    _, s64 = PJ.trunk(l64, pts.cpu().double(), pe)
    assert np.abs(sig.cpu().numpy() - s64.numpy().reshape(-1)).max() <= TOL_FP16_ANY * np.abs(s64.numpy()).max()
    # a launch split over several trunk passes gives the same rows
    from plenoctree_b200.octree import projection as P
    old = P.POINTS_PER_LAUNCH
    try:
        P.POINTS_PER_LAUNCH = 1000
        a2, sig2 = nerf.point_stage(pts)
    finally:
        P.POINTS_PER_LAUNCH = old
    assert torch.equal(a2, a) and torch.equal(sig2, sig)


def _fp64_rows(nerf, layers, a, sigma, dirs, S, sh_deg, deg_view, legacy):
    """fp64 leaf rows from the kernel's own inputs (a_p, sigma, directions) and |terms| for the rounding bound"""
    n = a.shape[0] // S
    d64 = dirs.double()
    enc = PJ.PO.posenc(d64.cpu(), 0, deg_view, legacy).to(d64.device)
    w10e = torch.from_numpy(layers[10][0][256:]).double().cuda()
    t = enc @ w10e
    t_abs = enc.abs() @ w10e.abs()
    w11, b11 = torch.from_numpy(layers[11][0]).double().cuda(), torch.from_numpy(layers[11][1]).double().cuda()
    Y = O.sh_basis(sh_deg, d64)
    K = Y.shape[1]
    rows, bound = [], []
    for i in range(0, a.shape[0], 256):
        ai = a[i:i + 256].double()
        x = ai[:, None] + t[None]
        z = torch.relu(x)
        rgb = z @ w11 + b11                                    # [p, D, 3]
        rgb_abs = (ai.abs()[:, None] + t_abs[None] + x.abs()) @ w11.abs() + b11.abs()
        c = torch.einsum("pdc,dk->pck", rgb, Y)
        g = (128 + 3 + 6 * deg_view + 8) * U
        cb = torch.einsum("pdc,dk->pck", g * rgb_abs + (dirs.shape[0] * S + 40) * U * rgb.abs(), Y.abs())
        rows.append(c)
        bound.append(cb)
    c = torch.cat(rows).reshape(n, S, 3 * K).mean(1) * (4 * math.pi / dirs.shape[0])
    cb = torch.cat(bound).reshape(n, S, 3 * K).mean(1) * (4 * math.pi / dirs.shape[0])
    s = sigma.double().reshape(n, S).mean(1)
    return torch.cat([c, s[:, None]], 1), torch.cat([cb, (S + 2) * U * sigma.double().abs().reshape(n, S).mean(1)[:, None]], 1)


@pytest.mark.gpu
@pytest.mark.parametrize("D,S,sh_deg,n_cells,cpb", [
    (1, 1, 1, 77, 16), (1, 8, 4, 29, 8), (100, 1, 2, 150, 64), (100, 8, 3, 45, 16), (100, 8, 4, 70, 32),
    (100, 3, 4, 23, 7), (10000, 1, 4, 9, 4), (10000, 8, 1, 5, 2), (10000, 8, 4, 3, 2), (100, 100, 4, 3, 2)])
def test_projection_against_fp64(D, S, sh_deg, n_cells, cpb):
    from plenoctree_b200.octree import projection as P
    pe, deg_view = (0, 10, False), 4
    layers, nerf = _model(13, pe, deg_view)
    pts = _points(n_cells * S, seed=D + S)
    n_blk = (n_cells + cpb - 1) // cpb
    tables = P.directions(nerf, sh_deg, D, 5, n_blk, seed=77)
    a, sig = nerf.point_stage(pts)
    out = P.project_cells(nerf, a, sig, S, sh_deg, tables, cells_per_block=cpb)
    dirs, t, basis = tables
    assert torch.allclose(dirs.norm(dim=-1), torch.ones_like(dirs[..., 0]), atol=4e-7)
    K = (sh_deg + 1) ** 2
    assert torch.equal(basis, O.sh_basis(sh_deg, dirs).float()) or \
        (basis.double() - O.sh_basis(sh_deg, dirs.double())).abs().max() <= 8 * U * 4
    for b in range(n_blk):
        lo, hi = b * cpb, min(n_cells, (b + 1) * cpb)
        ref, bnd = _fp64_rows(nerf, layers, a[lo * S:hi * S], sig[lo * S:hi * S], dirs[b], S, sh_deg, deg_view, False)
        err = (out[lo:hi].double() - ref).abs()
        assert out.shape[1] == 3 * K + 1
        assert bool((err <= bnd + 1e-30).all()), (b, float((err / (bnd + 1e-30)).max()))
    # the same rows from other launch splits: a block's rows do not depend on the launch
    tail = P.directions(nerf, sh_deg, D, 5 + n_blk - 1, 1, seed=77)
    for k, v in zip(tables, tail):
        assert torch.equal(k[-1], v[0])
    lo = (n_blk - 1) * cpb
    part = P.project_cells(nerf, a[lo * S:], sig[lo * S:], S, sh_deg, tail, cells_per_block=cpb)
    assert torch.equal(part, out[lo:])


@pytest.mark.gpu
@pytest.mark.parametrize("legacy,deg_view", [(False, 4), (True, 2), (False, 0)])
def test_direction_tables_against_fp64(legacy, deg_view):
    from plenoctree_b200.octree import projection as P
    pe = (0, 10, legacy)
    layers, nerf = _model(14, pe, deg_view)
    dirs, t, basis = P.directions(nerf, 4, 300, 0, 3, seed=5)
    enc = PJ.PO.posenc(dirs.double().cpu(), 0, deg_view, legacy).cuda()
    w = torch.from_numpy(layers[10][0][256:]).double().cuda()
    ref = (enc @ w).transpose(1, 2)
    bnd = (enc.abs() @ w.abs()).transpose(1, 2) * (3 + 6 * deg_view + 8) * U + 2.0 ** (deg_view + 1) * U * \
        w.abs().sum(0)[None, :, None]
    assert bool(((t.double() - ref).abs() <= bnd).all())
    # uniform on the sphere: the mean direction of 900 draws is within 4 standard deviations of 0
    assert float(dirs.reshape(-1, 3).mean(0).abs().max()) < 4 / math.sqrt(3 * 900)
    d2, _, _ = P.directions(nerf, 4, 300, 1, 1, seed=5)
    assert torch.equal(d2[0], dirs[1]) and not torch.equal(dirs[0], dirs[1])


@pytest.mark.gpu
def test_known_function_is_recovered():
    """raw colour c + A d: condition units relu(d), relu(-d), the rgb layer A relu(d) - A relu(-d) + c."""
    from plenoctree_b200.octree import projection as P
    layers, _ = _model(15)
    rs = np.random.RandomState(4)
    c, A = rs.uniform(-1, 1, 3).astype(np.float32), rs.uniform(-1, 1, (3, 3)).astype(np.float32)
    k10 = np.zeros_like(layers[10][0])
    w11 = np.zeros_like(layers[11][0])
    for j in range(3):
        k10[256 + j, j], k10[256 + j, 3 + j] = 1.0, -1.0
        w11[j, :], w11[3 + j, :] = A[:, j], -A[:, j]
    layers[9] = (np.zeros_like(layers[9][0]), np.zeros_like(layers[9][1]))
    layers[10] = (k10, np.zeros_like(layers[10][1]))
    layers[11] = (w11, c)
    nerf = P.VanillaNerf({"MLP_0": layers}, (0, 10, False), 4, num_fine_samples=0)
    D, S, n = 10000, 2, 6
    tables = P.directions(nerf, 4, D, 0, 1, seed=9)
    a, sig = nerf.point_stage(_points(n * S))
    out = P.project_cells(nerf, a, sig, S, 4, tables, cells_per_block=n).cpu().double().numpy()
    dirs = tables[0][0].cpu().double()
    Y = O.sh_basis(4, dirs).numpy()
    f = (torch.from_numpy(c).double()[None] + dirs @ torch.from_numpy(A).double().T).numpy()     # [D, 3]
    coef = out[:, :75].reshape(n, 3, 25)
    mc = 4 * math.pi * np.einsum("dc,dk->ck", f, Y) / D                # the estimator on these directions
    sd = 4 * math.pi * np.sqrt(np.var(f[:, :, None] * Y[:, None, :], axis=0) / D)
    analytic = np.zeros((3, 25))
    analytic[:, 0] = 4 * math.pi * O.SH_C0 * c
    C1 = 4 * math.pi / 3 * 0.4886025119029199
    analytic[:, 1], analytic[:, 2], analytic[:, 3] = -C1 * A[:, 1], C1 * A[:, 2], -C1 * A[:, 0]
    for p in range(n):
        assert np.abs(coef[p, :, 0] - mc[:, 0]).max() <= 64 * U * np.abs(mc[:, 0]).max() + 1e-6
        assert np.abs(coef[p, :, 0] - analytic[:, 0]).max() <= 4 * sd[:, 0].max()
        assert (np.abs(coef[p, :, 1:] - analytic[:, 1:]) <= 4 * sd[:, 1:] + 1e-6).all()


@pytest.mark.gpu
def test_readme_command_end_to_end(tmp_path):
    """octree.extraction --is_jaxnerf_ckpt --config nerf_sh/config/misc/proj on a synthetic Blender scene, then
    octree.optimization and octree.evaluation on the SH25 tree; one rank and two ranks give the same tree."""
    from plenoctree_b200.nerf import checkpoints as C, datasets as DS
    from plenoctree_b200.nerf.utils import pose_spherical
    from plenoctree_b200.octree import N3Tree, extraction as EX, projection as P
    W = 32
    cam_x = 0.6911112070083618
    rs = np.random.RandomState(6)
    poses = {k: [pose_spherical(rs.uniform(-180, 180), rs.uniform(-80, -10), 4.0) for _ in range(n)]
             for k, n in (("train", 6), ("val", 1), ("test", 2))}
    images = {k: [rs.uniform(0, 1, (W, W, 3)).astype(np.float32) for _ in v] for k, v in poses.items()}
    data_dir, train_dir = str(tmp_path / "scene"), str(tmp_path / "ckpt")
    DS.write_blender_scene(data_dir, images, poses, cam_x)
    mlps = {"MLP_0": PJ.init_params(21), "MLP_1": PJ.init_params(22)}
    for layers in mlps.values():                      # a dense blob around the origin
        layers[8] = (layers[8][0] * 8.0, layers[8][1] + 2.0)
    os.makedirs(train_dir)
    with open(os.path.join(train_dir, "checkpoint_100"), "wb") as f:
        f.write(C.msgpack_serialize({"optimizer": {"target": {"params": C.vanilla_to_flax_params(mlps)}}}))
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root)
    tree_path = str(tmp_path / "tree.npz")
    cmd = [sys.executable, "-m", "octree.extraction", "--train_dir", train_dir, "--is_jaxnerf_ckpt", "--config",
           "nerf_sh/config/misc/proj", "--data_dir", data_dir, "--output", tree_path, "--projection_samples", "100",
           "--radius", "1.3", "--init_grid_depth", "5", "--masking_mode", "sigma", "--noeval"]
    # absl's app.run exits with the value main returns (the tree, as for the NeRF-SH path), so success is judged by
    # the output file and the absence of a traceback
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True)
    assert "Traceback" not in r.stderr and os.path.exists(tree_path), r.stdout[-3000:] + r.stderr[-3000:]
    tree = N3Tree.load(tree_path, map_location="cuda")
    assert tree.data_dim == 76 and tree.data_format.format != 0
    leaves = torch.where(tree.depths == tree.max_depth)[0]
    assert leaves.numel() > 100
    # the same leaves from a direct library call with the same seeds
    nerf = P.VanillaNerf(mlps, (0, 10, False), 4, num_fine_samples=128)
    args = EX.default_args(use_viewdirs=True, sh_deg=4, projection_samples=100, init_grid_depth=5,
                           masking_mode="sigma", radius="1.3", output=None, sigma_activation="ReLU")
    direct = EX.extract(args, nerf, None)
    n = direct.n_internal
    assert np.array_equal(direct.child[:n].cpu().numpy(), tree.child[:n].cpu().numpy())
    got, want = tree.data[:n].cpu().numpy(), direct.data[:n].cpu().numpy()
    assert np.array_equal(got, want.astype(np.float16).astype(np.float32))      # tree.npz holds fp16, as svox's
    assert np.abs(got[..., :-1]).max() > 0
    for mod, extra in (("octree.optimization", ["--num_epochs", "1", "--output", str(tmp_path / "opt.npz")]),
                       ("octree.evaluation", [])):
        r = subprocess.run([sys.executable, "-m", mod, "--input", tree_path, "--config", "nerf_sh/config/misc/proj", "--data_dir", data_dir] + extra,
                           cwd=str(tmp_path), env=env, capture_output=True, text=True)
        assert "Traceback" not in r.stderr, (mod, r.stdout[-3000:] + r.stderr[-3000:])
    # octree.optimization writes its output only when the validation PSNR improves, which random images need not do
    psnr = float(r.stdout.split("Average PSNR")[1].split()[0])
    assert np.isfinite(psnr)


def _proj_tree():
    from plenoctree_b200.octree import N3Tree, extraction as E, projection as P
    nerf = P.VanillaNerf({"MLP_0": PJ.init_params(31)}, (0, 10, False), 4, num_fine_samples=0)
    args = E.default_args(use_viewdirs=True, sh_deg=4, projection_samples=100, init_grid_depth=4, samples_per_cell=4,
                          masking_mode="sigma", alpha_thresh=1e-4, output=None)
    tree = N3Tree(N=2, data_dim=76, init_reserve=4096, geom_resize_fact=1.0, depth_limit=4, radius=[1.5] * 3,
                  center=[0.0] * 3, data_format="SH25")
    E.step1(args, tree, nerf, None)
    E.step2(args, tree, nerf, cells_per_launch=P.CELLS_PER_BLOCK)
    n = tree.n_internal
    return tree.child[:n].cpu().numpy(), tree.data[:n].cpu().numpy()


def _proj_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)   # both ranks share cuda:0, as tests/test_dist.py
    try:
        torch.cuda.set_device(0)
        q.put((rank,) + _proj_tree())
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_projected_tree_two_ranks_equals_one_rank():
    import torch.multiprocessing as mp
    child1, data1 = _proj_tree()
    leaves = (child1 == 0).sum()
    assert leaves > 1024 and np.abs(data1[..., :-1]).max() > 0
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35500 + os.getpid() % 2000
    procs = [ctx.Process(target=_proj_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for rank, child, data in res:
        assert np.array_equal(child, child1), rank
        assert np.array_equal(data, data1), rank

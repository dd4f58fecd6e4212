"""Vanilla NeRF (use_viewdirs, sh_deg -1) inference: the view branch in the tensor-core forward
(pob_render_rays_vanilla, pob_eval_points_vanilla), VanillaNerfModel, check_vanilla_scope, the og_nerf preset and the
nerf_sh.eval / gen_video command lines.

GPU checks: raw sigma bit-identical to the plain-RGB sigma blob extraction evaluates; raw rgb against an fp64 view
branch formed from the kernel's own fp16 h7, its packed fp16 folded head and its fp32 per-point table, within
C_BRANCH * 2^-24 * sum|terms|; renders with pinned fine depths against the fp64 restatement (tests/support/vanilla_ref.py)
within the NeRF-SH render budget; bit-identical outputs at every SM split; the refusals; the CLI end to end."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import posenc_oracle as PO
from oracle import projection_oracle as PJ
from tests.support import vanilla_ref as VR
from tests.support.vanilla_ref import C_BRANCH, RGB_TOL, U, _h7_fp16, _mlps, _rays, _view_features

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _args(**kw):
    a = dict(use_viewdirs=True, sh_deg=-1, sg_dim=-1, dataset="blender", net_depth=8, net_width=256, skip_layer=4,
             net_depth_condition=1, net_width_condition=128, deg_view=4, min_deg_point=0, max_deg_point=10,
             legacy_posenc_order=False, num_coarse_samples=64, num_fine_samples=128, net_activation="relu",
             rgb_activation="sigmoid", sigma_activation="relu", render_path=False, spherify=False)
    a.update(kw)
    return types.SimpleNamespace(**a)


# ---- CPU ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(), dict(deg_view=0), dict(deg_view=10), dict(deg_view=32),
                                dict(net_activation="elu"), dict(net_activation="Softplus"), dict(net_activation="tanh"),
                                dict(sigma_activation="softplus"), dict(min_deg_point=2, max_deg_point=8,
                                                                        legacy_posenc_order=True),
                                dict(num_coarse_samples=256, num_fine_samples=768), dict(num_fine_samples=0),
                                dict(dataset="nsvf"), dict(dataset="llff", render_path=True, spherify=True)])
def test_vanilla_scope_accepts(kw):
    from plenoctree_b200.nerf import flags as F
    F.check_vanilla_scope(_args(**kw))


@pytest.mark.parametrize("kw,exc,match", [
    (dict(sh_deg=4), NotImplementedError, "You can only use up to one of: SH, SG or use_viewdirs.*og_nerf"),
    (dict(sh_deg=0), NotImplementedError, "You can only use up to one of"),
    (dict(sg_dim=4), NotImplementedError, "You can only use up to one of"),
    (dict(use_viewdirs=False), ValueError, "use_viewdirs"),
    (dict(net_depth_condition=2), NotImplementedError, "condition"),
    (dict(net_width_condition=256), NotImplementedError, "condition"),
    (dict(deg_view=-1), NotImplementedError, "deg_view"), (dict(deg_view=33), NotImplementedError, "deg_view"),
    (dict(net_activation="gelu"), NotImplementedError, "pre-activation"),
    (dict(rgb_activation="relu"), NotImplementedError, "rgb_activation"),
    (dict(sigma_activation="exp"), NotImplementedError, "sigma_activation"),
    (dict(net_depth=6), NotImplementedError, "trunk"), (dict(max_deg_point=12), NotImplementedError, "posenc"),
    (dict(num_coarse_samples=512, num_fine_samples=1024), NotImplementedError, "num_coarse"),
    (dict(dataset="deepvoxels"), NotImplementedError, "dataset"),
    (dict(render_path=True), ValueError, "llff")])
def test_vanilla_scope_refuses(kw, exc, match):
    from plenoctree_b200.nerf import flags as F
    with pytest.raises(exc, match=match):
        F.check_vanilla_scope(_args(**kw))


def test_check_scope_still_refuses_use_viewdirs():
    from plenoctree_b200.nerf import flags as F
    with pytest.raises(NotImplementedError, match="use_viewdirs"):
        F.check_scope(_args())


def test_train_still_refuses_og_nerf(tmp_path):
    """nerf_sh.train's main with --config nerf_sh/config/misc/og_nerf stops at check_scope (its device set-up is
    replaced by the CPU, so this runs without a GPU)"""
    code = ("import sys, torch\n"
            "from plenoctree_b200.nerf_sh import train as T\n"
            "T._dist_init = lambda: (0, 1, torch.device('cpu'))\n"
            "T.FLAGS(sys.argv)\n"
            "T.main([])\n")
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", code, "--config", "nerf_sh/config/misc/og_nerf",
                        "--train_dir", str(tmp_path / "t"), "--data_dir", str(tmp_path / "d")],
                       cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode != 0, r.stdout + r.stderr
    assert "NotImplementedError: use_viewdirs (vanilla NeRF colour head) is outside the NeRF-SH path" in r.stderr, \
        r.stderr[-2000:]
    assert not (tmp_path / "t").exists()


def test_og_nerf_preset_equals_the_reference_file_and_a_file_on_disk_wins(tmp_path):
    import yaml
    from plenoctree_b200.nerf import flags as F
    from plenoctree_b200.presets import NERF_SH
    # nerf_sh/config/misc/og_nerf.yaml of the reference, as shipped
    ref = dict(dataset="blender", image_batching=False, factor=0, num_coarse_samples=64, num_fine_samples=128,
               use_viewdirs=True, white_bkgd=True, batch_size=1024, randomized=True, sparsity_weight=0.0,
               max_steps=2000000)
    assert NERF_SH["og_nerf"] == ref
    more = dict(config="nerf_sh/config/misc/og_nerf", image_batching=True, factor=4, white_bkgd=False, batch_size=8,
                randomized=False, max_steps=1, sparsity_weight=1e-3)
    args = _args(use_viewdirs=False, **more)
    F.update_flags(args)
    assert args.use_viewdirs is True and args.sh_deg == -1 and args.sparsity_weight == 0.0 and args.factor == 0
    F.check_vanilla_scope(args)
    (tmp_path / "og_nerf.yaml").write_text(yaml.safe_dump({"use_viewdirs": True, "deg_view": 2}))
    args = _args(**dict(more, config=str(tmp_path / "og_nerf")))
    F.update_flags(args)
    assert args.deg_view == 2 and args.factor == 4


def test_fold_is_formed_in_fp64_and_rounded_once():
    from plenoctree_b200.nerf import vanilla as V
    layers = _mlps(5)["MLP_1"]
    w, c = V.fold_view_branch(layers)
    k9, b9 = (np.asarray(a, np.float64) for a in layers[9])
    k10, b10 = (np.asarray(a, np.float64) for a in layers[10])
    assert np.array_equal(w, k9 @ k10[:256]) and np.array_equal(c, b9 @ k10[:256] + b10)
    flat = V.folded_flat(layers)
    head = flat[-256 * 128:].reshape(256, 128)
    assert np.array_equal(head, w.astype(np.float16).astype(np.float32))
    # within half an fp16 ulp of the fp64 product (not double-rounded through fp32)
    ulp = np.spacing(np.abs(w).astype(np.float16)).astype(np.float64)
    assert (np.abs(head - w) <= 0.5 * ulp).all()
    trunk = np.concatenate([np.asarray(a, np.float32).reshape(-1) for k, b in layers[:9] for a in (k, b)])
    assert np.array_equal(flat[:trunk.size], trunk)
    from plenoctree_b200 import _lib
    assert flat.size == _lib.lib.pob_vanilla_param_count(None)


@pytest.mark.parametrize("fmt", ["flax", "torch"])
def test_checkpoint_round_trip_into_the_packed_inputs(tmp_path, fmt):
    """a flax checkpoint_<step> and a torch *.ckpt of the same weights restore to the same folded inputs"""
    from plenoctree_b200.nerf import checkpoints as C, vanilla as V
    pe, dv = (1, 9, True), 6
    mlps = _mlps(7, pe, dv)
    if fmt == "flax":
        with open(tmp_path / "checkpoint_250", "wb") as f:
            f.write(C.msgpack_serialize({"optimizer": {"target": {"params": C.vanilla_to_flax_params(mlps)},
                                                       "state": {"step": 250}}}))
    else:
        torch.save({"model": {k: torch.from_numpy(np.ascontiguousarray(v))
                              for k, v in C.vanilla_to_torch_state_dict(mlps).items()}}, tmp_path / "m.ckpt")
    got = C.restore_vanilla(str(tmp_path), fmt == "flax", pe, dv)
    for name in ("MLP_0", "MLP_1"):
        assert np.array_equal(V.folded_flat(got[name]), V.folded_flat(mlps[name]))
        for a, b in zip(V.fold_view_branch(got[name]), V.fold_view_branch(mlps[name])):
            assert np.array_equal(a, b)


def test_oracle_render_matches_the_sh_oracle_per_ray_stages():
    """the oracle's vanilla render at deg_view 0 with a view branch that ignores the direction equals nerf_sh_oracle's
    plain-RGB (sh_deg -1) render of the composed head: the per-ray stages are the same code"""
    from oracle import nerf_sh_oracle as O
    rs = np.random.RandomState(2)
    layers = PJ.init_params(3, deg_view=0)
    layers[11] = (np.eye(128, 3, dtype=np.float32), np.zeros(3, np.float32))
    layers[9] = (np.eye(256, dtype=np.float32), np.zeros(256, np.float32))
    layers[10] = (np.concatenate([np.eye(256, 128, dtype=np.float32), np.zeros((3, 128), np.float32)]),
                  np.full(128, 5.0, np.float32))             # z = relu(h7[:128] + 5): h7 >= 0, so linear
    R = 16
    o = rs.normal(size=(R, 3))
    o = torch.from_numpy(o / np.linalg.norm(o, axis=1, keepdims=True) * 4)
    d = -o / 4 + torch.from_numpy(rs.uniform(-0.1, 0.1, (R, 3)))
    v = d / d.norm(dim=-1, keepdim=True)
    got = VR.render_rays(layers, layers, (o, d, v), 64, 0, 2.0, 6.0, deg_view=0)
    params = [(torch.from_numpy(k).double(), torch.from_numpy(b).double()) for k, b in layers[:9]]
    params.append((torch.from_numpy(np.eye(256, 3)).double(), torch.full((3,), 5.0, dtype=torch.float64)))
    want = O.nerf_forward(params, params, -1, (o, d, v), 64, 0, 2.0, 6.0)
    for g, w in zip(got[0], want[0]):
        assert torch.allclose(g, w, atol=1e-12)


def _golden(golden_dir):
    import json
    z = np.load(os.path.join(golden_dir, "ref_vanilla.npz"))
    scale, shift = (float(x) for x in z["sigma_scale_shift"])
    cases = {tag: (tuple(c), VR.golden_layers(c[0], c[1], c[2], scale, shift))
             for tag, c in json.loads(str(z["cases"])).items()}
    return z, cases


def _golden_inputs(z, rtag):
    """(t_rand, z_fine, sigma_noise) of the golden's randomized ("rand") or deterministic ("det") call"""
    std = np.float32(z["noise_std"])
    if rtag == "det":
        return None, None, None
    return z["t_rand"], None, ((z["noise_coarse"][..., 0] * std).astype(np.float32),
                              (z["noise_fine"][..., 0] * std).astype(np.float32))


def test_restatement_against_the_executed_reference(golden_dir):
    """tests/support/vanilla_ref.py in fp64 against the reference's NerfModel.__call__ executed over numpy (fp32), on
    the reference's own fine depths, and against its torch twin's eval_points_raw(points, viewdirs)"""
    z, cases = _golden(golden_dir)
    rays = tuple(torch.from_numpy(z[k]).double() for k in ("origins", "directions", "viewdirs"))
    partial = 0
    for tag, ((_, dv, legacy, act, sact), mlps) in cases.items():
        pe = (0, 10, bool(legacy))
        for rtag in ("det", "rand"):
            t_rand, _, noise = _golden_inputs(z, rtag)
            with torch.no_grad():
                ref = VR.render_rays(mlps["MLP_0"], mlps["MLP_1"], rays, 64, 128, 2.0, 6.0, True,
                                     None if t_rand is None else torch.from_numpy(t_rand).double(), None,
                                     torch.from_numpy(z[f"{tag}_{rtag}_z_fine"]).double(), pe=pe, deg_view=dv,
                                     act=act, sigma_act=sact,
                                     sigma_noise=None if noise is None else
                                     tuple(torch.from_numpy(n).double()[..., None] for n in noise))
            for lvl, r in zip(("coarse", "fine"), ref):
                for i, name in ((0, "rgb"), (2, "acc")):
                    err = float(np.abs(r[i].numpy() - z[f"{tag}_{rtag}_{lvl}_{name}"]).max())
                    assert err < 2e-5, (tag, rtag, lvl, name, err)
                assert float(r[2].mean()) > 0.02, (tag, rtag, lvl)                     # the rays cross density
                partial += int(((r[2] > 0.01) & (r[2] < 0.99)).sum())
    assert partial >= 10, partial                                                         # and not only opaque
    assert set(cases) == {"og_nerf", "dv10_legacy", "dv0", "elu_softplus"}
    pts, vd = (torch.from_numpy(z[k]).double() for k in ("twin_points", "twin_viewdirs"))
    for tag, ((_, dv, legacy, act, _), mlps) in cases.items():
        if act != "relu":
            continue
        for lvl, name in (("fine", "MLP_1"), ("coarse", "MLP_0")):
            rgb, sigma = VR.eval_points_paired(mlps[name], pts, vd, (0, 10, bool(legacy)), dv)
            assert np.abs(rgb.numpy() - z[f"twin_{tag}_{lvl}_raw_rgb"]).max() < 1e-5, (tag, lvl)
            assert np.abs(sigma.numpy() - z[f"twin_{tag}_{lvl}_raw_sigma"]).max() < 1e-4, (tag, lvl)


def test_og_nerf_preset_is_the_reference_config_the_golden_parsed(golden_dir):
    import json
    from plenoctree_b200.presets import NERF_SH
    z = np.load(os.path.join(golden_dir, "ref_vanilla.npz"))
    assert json.loads(str(z["og_nerf_config"])) == NERF_SH["og_nerf"]


def test_paired_oracle_is_the_cross_broadcast_diagonal():
    """eval_points_paired (one direction per point) is the diagonal of the golden-pinned cross-broadcast form"""
    layers = PJ.init_params(4)
    pts = torch.from_numpy(np.random.RandomState(1).uniform(-1, 1, (8, 3)))
    vd = pts / pts.norm(dim=-1, keepdim=True)
    cross, s1 = PJ.eval_points_raw(layers, pts, vd)
    paired, s2 = VR.eval_points_paired(layers, pts, vd)
    assert torch.allclose(paired, cross[torch.arange(8), torch.arange(8)], atol=1e-12) and torch.equal(s1, s2)


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _model(mlps, **kw):
    from plenoctree_b200.nerf.vanilla import VanillaNerfModel
    pe = kw.pop("pe", PO.DEFAULT)
    return VanillaNerfModel(mlps, min_deg_point=pe[0], max_deg_point=pe[1], legacy_posenc_order=pe[2], **kw)


def _act64(name, z):
    from tests.support.model_flags import _act64 as A
    return A(name, torch.from_numpy(z)).numpy()


@pytest.mark.gpu
def test_raw_sigma_bit_identical_to_the_sigma_blob():
    """the 136-column heads MMA gives column 0 the bits of the 80-column one extraction's sigma blob uses"""
    from plenoctree_b200 import ops
    from plenoctree_b200.octree.projection import VanillaNerf
    for pe, act in ((PO.DEFAULT, "relu"), ((2, 8, True), "relu")):
        mlps = _mlps(11, pe)
        nerf = VanillaNerf(mlps, pe, 4, num_fine_samples=128)
        model = _model(mlps, pe=pe, net_activation=act)
        rs = np.random.RandomState(4)
        pts = torch.from_numpy(rs.uniform(-1.5, 1.5, (20000, 3)).astype(np.float32)).cuda()
        vd = torch.nn.functional.normalize(torch.from_numpy(rs.normal(size=(20000, 3)).astype(np.float32)), dim=-1)
        _, s_blob = ops.eval_points_raw(nerf.sigma_blob, -1, pts, posenc=pe)
        _, s_van = model.eval_points_raw(pts, vd.cuda())
        assert torch.equal(s_blob.view(torch.int32), s_van.view(torch.int32)), pe


@pytest.mark.gpu
@pytest.mark.parametrize("deg_view,legacy,act", [(0, False, "relu"), (4, False, "relu"), (10, True, "relu"),
                                                 (32, False, "relu"), (4, True, "elu"), (4, False, "softplus"),
                                                 (10, False, "tanh")])
def test_view_branch_against_fp64_from_the_kernels_h7(deg_view, legacy, act):
    from plenoctree_b200 import _lib
    from plenoctree_b200.nerf import flags as F, vanilla as V
    pe = (0, 10, legacy)
    mlps = _mlps(31 + deg_view, pe, deg_view)
    model = _model(mlps, pe=pe, deg_view=deg_view, net_activation=act)
    rs = np.random.RandomState(deg_view)
    m = 3000
    pts = torch.from_numpy(rs.uniform(-1.5, 1.5, (m, 3)).astype(np.float32)).cuda()
    vd = torch.nn.functional.normalize(torch.from_numpy(rs.normal(size=(m, 3)).astype(np.float32)), dim=-1).cuda()
    layers = mlps["MLP_1"]
    table = torch.empty((m, 128), dtype=torch.float32, device="cuda")
    rgb = torch.empty((m, 3), dtype=torch.float32, device="cuda")
    sig = torch.empty((m, 1), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.pob_eval_points_vanilla(_lib.ptr(model.blobs[1]), _lib.posenc_ref(model._pe),
                                                _lib.ctypes.addressof(model.view), 1, _lib.ptr(pts), _lib.ptr(vd), m,
                                                _lib.ptr(table), _lib.ptr(rgb), _lib.ptr(sig), None, 0,
                                                _lib.stream_ptr()))
    torch.cuda.synchronize()
    t = table.cpu().numpy().astype(np.float64)
    # the fp32 table against fp64 at the kernel's fp32 sine arguments
    w10e = np.asarray(layers[10][0][256:], np.float64)
    _, c = V.fold_view_branch(layers)
    enc = _view_features(vd.cpu().numpy(), deg_view, legacy)
    t64 = enc @ w10e + c
    t_terms = np.abs(enc) @ np.abs(w10e) + np.abs(c)
    assert (np.abs(t - t64) <= 64 * U * t_terms + 1e-6 * np.abs(enc).max(axis=1, keepdims=True)).all()
    # the branch from the kernel's own fp16 h7, the packed fp16 fold and the fp32 table
    h = _h7_fp16(layers, pts, pe, F.net_activation_code(act))
    fold16 = V.folded_flat(layers)[-256 * 128:].reshape(256, 128).astype(np.float64)
    a = h @ fold16
    z = _act64(act, a + t)
    w11, b11 = (np.asarray(x, np.float64) for x in layers[11])
    want = z @ w11 + b11
    terms = ((np.abs(h) @ np.abs(fold16) + np.abs(t)) @ np.abs(w11)) + np.abs(z) @ np.abs(w11) + np.abs(b11)
    err = np.abs(rgb.cpu().numpy() - want)
    assert (err <= C_BRANCH * U * terms).all(), float((err / (U * terms)).max())
    assert float(np.abs(want).max()) > 0.05


@pytest.mark.gpu
@pytest.mark.parametrize("nc,nf", [(64, 128), (128, 384), (256, 768), (64, 0)])
@pytest.mark.parametrize("act,sigma_act", [("relu", "relu"), ("elu", "softplus")])
def test_render_with_pinned_fine_depths_against_fp64(nc, nf, act, sigma_act):
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf.models import Rays
    R = 512 if nc + nf <= 192 else 128
    mlps = _mlps(41, deg_view=4)
    model = _model(mlps, num_coarse_samples=nc, num_fine_samples=nf, max_rays=R, net_activation=act,
                   sigma_activation=sigma_act)
    o, d, v = _rays(R, 5)
    rays_t = tuple(torch.from_numpy(x).double() for x in (o, d, v))
    rs = np.random.RandomState(8)
    t_rand = rs.uniform(0, 1, (R, nc)).astype(np.float32)
    lay = lambda n: mlps[n]   # noqa: E731
    for randomized in (False, True):
        tr = torch.from_numpy(t_rand).double() if randomized else None
        z_fine = None
        if nf:
            z_c, _ = O.sample_along_rays(rays_t[0], rays_t[1], nc, 2.0, 6.0, tr)
            zf = torch.sort(torch.cat([z_c, z_c[:, :1] + (z_c[:, -1:] - z_c[:, :1]) *
                                       torch.from_numpy(rs.uniform(0, 1, (R, nf)))], -1), -1)[0]
            z_fine = zf.float().numpy()
        with torch.no_grad():
            ref = VR.render_rays(lay("MLP_0"), lay("MLP_1"), rays_t, nc, nf, 2.0, 6.0, True, tr, None,
                                 None if z_fine is None else torch.from_numpy(z_fine).double(), act=act,
                                 sigma_act=sigma_act)
        got = model(Rays(o, d, v), randomized=randomized, t_rand=t_rand if randomized else None, z_fine=z_fine)
        torch.cuda.synchronize()
        assert len(got) == len(ref)
        for lvl, (g, r) in enumerate(zip(got, ref)):
            e_rgb = float((g[0].cpu().double() - r[0]).abs().max())
            e_acc = float((g[2].cpu().double() - r[2]).abs().max())
            assert e_rgb < RGB_TOL and e_acc < RGB_TOL, (randomized, lvl, e_rgb, e_acc)
            assert float(r[2].mean()) > 0.05                   # the rays cross the density


@pytest.mark.gpu
def test_render_against_the_executed_reference(golden_dir):
    """pob_render_rays_vanilla on the golden's rays against the reference's executed NerfModel.__call__: both levels,
    deterministic and randomized (the reference's jitter, its fine depths pinned, its density noise passed as
    sigma_noise), within the NeRF-SH render budget"""
    from plenoctree_b200.nerf.models import Rays
    z, cases = _golden(golden_dir)
    rays = Rays(*(z[k] for k in ("origins", "directions", "viewdirs")))
    for tag, ((_, dv, legacy, act, sact), mlps) in cases.items():
        model = _model(mlps, pe=(0, 10, bool(legacy)), deg_view=dv, net_activation=act, sigma_activation=sact,
                       max_rays=rays.origins.shape[0])
        for rtag in ("det", "rand"):
            t_rand, _, noise = _golden_inputs(z, rtag)
            got = model(rays, randomized=rtag == "rand", t_rand=t_rand, z_fine=z[f"{tag}_{rtag}_z_fine"],
                        sigma_noise=noise)
            torch.cuda.synchronize()
            for lvl, g in zip(("coarse", "fine"), got):
                for i, name in ((0, "rgb"), (2, "acc")):
                    err = float(np.abs(g[i].cpu().numpy() - z[f"{tag}_{rtag}_{lvl}_{name}"]).max())
                    assert err < RGB_TOL, (tag, rtag, lvl, name, err)


@pytest.mark.gpu
def test_noise_std_draws_density_noise_when_randomized():
    """randomized with noise_std set: the epilogue adds the draws to raw sigma (a different, finite render);
    deterministic calls take none"""
    from plenoctree_b200.nerf.models import Rays
    mlps = _mlps(91)
    o, d, v = _rays(256, 4)
    plain = _model(mlps, max_rays=256)
    noisy = _model(mlps, max_rays=256, noise_std=1.0)
    t = np.random.RandomState(1).uniform(0, 1, (256, 64)).astype(np.float32)
    u = np.random.RandomState(2).uniform(0, 1, (256, 128)).astype(np.float32)
    a = plain(Rays(o, d, v), randomized=True, t_rand=t, u=u)[-1][0]
    b = noisy(Rays(o, d, v), randomized=True, t_rand=t, u=u)[-1][0]
    c = noisy(Rays(o, d, v))[-1][0]
    e = plain(Rays(o, d, v))[-1][0]
    torch.cuda.synchronize()
    assert torch.isfinite(b).all() and float((a - b).abs().max()) > 1e-3
    assert torch.equal(c, e)


@pytest.mark.gpu
def test_full_frame_psnr_parity():
    """an 80 x 80 frame (render_image) of a vanilla model within 0.05 dB of the oracle render's PSNR"""
    from plenoctree_b200.nerf import utils as NU
    from plenoctree_b200.nerf.rays import generate_rays, pose_spherical
    mlps = _mlps(51)
    W = 80
    model = _model(mlps, max_rays=2048)
    rays = generate_rays(W, W, 0.5 * W / np.tan(0.35), pose_spherical(30.0, -30.0, 4.0)[None])
    rays = [np.asarray(r[0], np.float32) for r in rays]
    rgb, _, _ = NU.render_image(model, NU.Rays(*rays), chunk=2048)
    flat = [torch.from_numpy(r.reshape(-1, 3)).double() for r in rays]
    with torch.no_grad():
        ref = torch.cat([VR.render_rays(mlps["MLP_0"], mlps["MLP_1"], tuple(f[i:i + 1600] for f in flat), 64, 128,
                                        2.0, 6.0)[-1][0] for i in range(0, W * W, 1600)])
    target = np.random.RandomState(3).uniform(0, 1, (W * W, 3))
    psnr = lambda x: float(NU.compute_psnr(float(((x - target) ** 2).mean())))   # noqa: E731
    p_got, p_ref = psnr(rgb.reshape(-1, 3).cpu().double().numpy()), psnr(ref.numpy())
    assert abs(p_got - p_ref) < 0.05, (p_got, p_ref)


@pytest.mark.gpu
def test_outputs_do_not_depend_on_the_sm_split(monkeypatch):
    from plenoctree_b200 import _lib
    from plenoctree_b200.nerf.models import Rays
    R = 3000
    model = _model(_mlps(61), max_rays=R)
    o, d, v = _rays(R, 9)
    pts = torch.from_numpy(np.random.RandomState(2).uniform(-1.5, 1.5, (50000, 3)).astype(np.float32)).cuda()
    vd = torch.nn.functional.normalize(pts, dim=-1)
    outs = []
    for sms in ("16", "66", None):
        if sms is None:
            monkeypatch.delenv("POB_SM_COUNT", raising=False)
        else:
            monkeypatch.setenv("POB_SM_COUNT", sms)
        r = model(Rays(o, d, v))
        p = model.eval_points_raw(pts, vd)
        q = model.eval_points(pts, vd, coarse=True)
        torch.cuda.synchronize()
        outs.append([x.clone() for lvl in r for x in lvl] + list(p) + list(q))
    assert _lib.lib.pob_sm_count() > 66
    for other in outs[:2]:
        for a, b in zip(outs[2], other):
            assert torch.equal(a, b)


@pytest.mark.gpu
def test_point_chunks_give_the_unchunked_result(monkeypatch):
    """eval_points_raw / eval_points split into POINTS_PER_CALL chunks (one scratch table) give the bits of one call"""
    from plenoctree_b200.nerf import vanilla as V
    model = _model(_mlps(95), max_rays=64)
    rs = np.random.RandomState(3)
    pts = torch.from_numpy(rs.uniform(-1.5, 1.5, (5000, 3)).astype(np.float32)).cuda()
    vd = torch.nn.functional.normalize(torch.from_numpy(rs.normal(size=(5000, 3)).astype(np.float32)), dim=-1).cuda()
    whole = list(model.eval_points_raw(pts, vd)) + list(model.eval_points(pts, vd))
    monkeypatch.setattr(V, "POINTS_PER_CALL", 1152)
    chunked = list(model.eval_points_raw(pts, vd)) + list(model.eval_points(pts, vd))
    torch.cuda.synchronize()
    for a, b in zip(whole, chunked):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_refusals_fire_with_their_message_and_launch_nothing(monkeypatch):
    from plenoctree_b200 import _lib
    from plenoctree_b200._lib import PREC_FP16, PREC_FP16X3, RenderConfig, ViewBranch, lib, ptr
    from plenoctree_b200.nerf.models import ctypes_ref
    model = _model(_mlps(71), max_rays=64)
    f = torch.zeros(64 * 3, dtype=torch.float32, device="cuda")
    out = torch.zeros(64 * 5, dtype=torch.float32, device="cuda")
    ws = model.workspace()
    cfg = model.cfg

    def render(c=cfg, view=model.view, prec=PREC_FP16, packed=model.blobs[0]):
        return lib.pob_render_rays_vanilla(ctypes_ref(c), None if view is None else ctypes_ref(view), ptr(packed),
                                           ptr(model.blobs[1]), ptr(f), ptr(f), ptr(f), 64, ptr(model.z_base), None,
                                           ptr(model.u_table), 0, None, ptr(out), ptr(out), ptr(ws), prec,
                                           _lib.stream_ptr())

    def points(view=model.view, mlp=1, table=f, sigma_act=0):
        return lib.pob_eval_points_vanilla(ptr(model.blobs[1]), None, None if view is None else ctypes_ref(view), mlp,
                                           ptr(f), ptr(f), 1, ptr(table), ptr(f), ptr(f), None, sigma_act,
                                           _lib.stream_ptr())

    bad_deg = RenderConfig(3, 64, 128, 1, 64, 0)
    bad_view = ViewBranch()
    bad_view.deg_view = 33
    null_view = ViewBranch()
    null_view.deg_view = 4
    cases = [(lambda: render(c=bad_deg), "cfg->sh_deg must be -1"),
             (lambda: render(view=None), "view branch descriptor is NULL"),
             (lambda: render(prec=PREC_FP16X3), "precision must be POB_PREC_FP16"),
             (lambda: render(view=bad_view), "deg_view must be in \\[0, 32\\]"),
             (lambda: render(view=null_view), "NULL view branch array"),
             (lambda: render(packed=None), "packed weights pointer is NULL"),
             (lambda: points(mlp=2), "mlp must be 0 or 1"),
             (lambda: points(view=None), "view branch descriptor is NULL"),
             (lambda: points(table=None), "NULL pointer"),
             (lambda: points(table=f[1:]), "table_dev must be 8-byte aligned"),
             (lambda: points(sigma_act=5), "sigma_activation"),
             (lambda: lib.pob_pack_vanilla(None, None, ptr(out), None), "NULL pointer")]
    torch.cuda.synchronize()
    for call, match in cases:
        n0 = lib.pob_launch_count()
        assert call() != 0
        assert pytest.importorskip("re").search(match, lib.pob_last_error().decode()), lib.pob_last_error()
        assert lib.pob_launch_count() == n0
    monkeypatch.setenv("POB_SM_COUNT", "7")
    n0 = lib.pob_launch_count()
    assert render() != 0 and "POB_SM_COUNT" in lib.pob_last_error().decode() and lib.pob_launch_count() == n0
    assert lib.pob_vanilla_workspace_bytes(ctypes_ref(bad_deg)) == -1


def _scene(tmp_path, W=32):
    from plenoctree_b200.nerf import checkpoints as C, datasets as DS
    from plenoctree_b200.nerf.utils import pose_spherical
    cam_x = 0.6911112070083618
    rs = np.random.RandomState(6)
    poses = {k: [pose_spherical(rs.uniform(-180, 180), rs.uniform(-80, -10), 4.0) for _ in range(n)]
             for k, n in (("train", 6), ("val", 1), ("test", 2))}
    images = {k: [rs.uniform(0, 1, (W, W, 3)).astype(np.float32) for _ in v] for k, v in poses.items()}
    data_dir, train_dir = str(tmp_path / "scene"), str(tmp_path / "ckpt")
    DS.write_blender_scene(data_dir, images, poses, cam_x)
    mlps = _mlps(81)
    os.makedirs(train_dir)
    with open(os.path.join(train_dir, "checkpoint_100"), "wb") as f:
        f.write(C.msgpack_serialize({"optimizer": {"target": {"params": C.vanilla_to_flax_params(mlps)},
                                                   "state": {"step": 100}}}))
    return data_dir, train_dir, mlps


@pytest.mark.gpu
def test_eval_gen_video_and_projection_command_lines(tmp_path):
    """nerf_sh.eval --config nerf_sh/config/misc/og_nerf on a flax vanilla checkpoint prints the PSNR of the oracle's
    render of the same weights (within 0.05 dB); gen_video renders frames; the same checkpoint then goes through
    octree.extraction --config nerf_sh/config/misc/proj and octree.evaluation (source NeRF vs projected tree)."""
    from plenoctree_b200.nerf import datasets as DS, utils as NU
    data_dir, train_dir, mlps = _scene(tmp_path)
    env = dict(os.environ, PYTHONPATH=ROOT)

    def run(mod, *extra):
        r = subprocess.run([sys.executable, "-m", mod, *extra], cwd=str(tmp_path), env=env, capture_output=True,
                           text=True)
        assert "Traceback" not in r.stderr, (mod, r.stdout[-3000:] + r.stderr[-3000:])
        return r.stdout

    out = run("nerf_sh.eval", "--config", "nerf_sh/config/misc/og_nerf", "--train_dir", train_dir, "--data_dir",
              data_dir)
    psnr = float(out.split("Average PSNR")[1].split()[0])
    assert os.path.exists(os.path.join(train_dir, "test_preds", "psnrs_100.txt"))
    args = _args(data_dir=data_dir, factor=0, white_bkgd=True, near=2.0, far=6.0, render_path=False,
                 llffhold=8, spherify=False, batch_size=1024, image_batching=False, dataset="blender")
    ds = DS.get_dataset("test", args, device="cpu")
    ps = []
    for _ in range(ds.size):
        b = ds.next_test()
        flat = [torch.from_numpy(np.ascontiguousarray(r).reshape(-1, 3)).double() for r in b["rays"]]
        with torch.no_grad():
            ref = VR.render_rays(mlps["MLP_0"], mlps["MLP_1"], tuple(flat), 64, 128, 2.0, 6.0)[-1][0]
        ps.append(float(NU.compute_psnr(float(((ref.numpy() - b["pixels"].reshape(-1, 3)) ** 2).mean()))))
    assert abs(psnr - np.mean(ps)) < 0.05, (psnr, ps)
    run("nerf_sh.gen_video", "--config", "nerf_sh/config/misc/og_nerf", "--train_dir", train_dir, "--num_views", "2",
        "--width", "24", "--height", "24")
    assert len(os.listdir(os.path.join(train_dir, "video", "e300", "frames"))) == 2
    tree_path = str(tmp_path / "tree.npz")
    run("octree.extraction", "--train_dir", train_dir, "--is_jaxnerf_ckpt", "--config", "nerf_sh/config/misc/proj",
        "--data_dir", data_dir, "--output", tree_path, "--projection_samples", "100", "--radius", "1.3",
        "--init_grid_depth", "5", "--masking_mode", "sigma", "--noeval")
    assert os.path.exists(tree_path)
    out = run("octree.evaluation", "--input", tree_path, "--config", "nerf_sh/config/misc/proj", "--data_dir",
              data_dir)
    assert np.isfinite(float(out.split("Average PSNR")[1].split()[0]))

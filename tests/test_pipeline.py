"""End-to-end drop-in flow on a synthetic Blender-format scene (no dataset can be downloaded here), through the CLI
mains with the reference's flag names and a YAML config:

    nerf_sh.train -> checkpoint_<step> (flax format) -> nerf_sh.eval -> octree.extraction --is_jaxnerf_ckpt
    -> tree.npz -> octree.optimization -> tree_opt.npz -> octree.evaluation

CPU part: flags / YAML / dataset loader / SSIM golden.  GPU part: the whole chain on 48x48 images."""
import functools
import json
import os

import numpy as np
import pytest
import torch

from tests.support.model_flags import _set_flags
from tests.support.records import record


_record_pipeline = functools.partial(record, "pipeline.json")


def test_flags_yaml_and_scope(tmp_path):
    from plenoctree_b200.nerf import flags as F
    FLAGS = _set_flags(train_dir=str(tmp_path), data_dir=str(tmp_path), use_viewdirs=True, sh_deg=-1, batch_size=1024,
                       config=None)
    cfg = tmp_path / "blender.yaml"
    cfg.write_text("dataset: blender\nimage_batching: false\nfactor: 0\nnum_coarse_samples: 64\nnum_fine_samples: 128\n"
                   "use_viewdirs: false\nwhite_bkgd: true\nbatch_size: 1024\nsh_deg: 3\nrandomized: true\n"
                   "max_steps: 2000000\n")     # = nerf_sh/config/blender.yaml of the reference
    FLAGS.config = str(tmp_path / "blender")
    F.update_flags(FLAGS)
    assert FLAGS.sh_deg == 3 and FLAGS.use_viewdirs is False and FLAGS.max_steps == 2000000 and FLAGS.factor == 0
    F.check_flags(FLAGS, world=8)
    F.check_scope(FLAGS)
    with pytest.raises(ValueError):
        F.check_flags(FLAGS, world=3)                      # batch 1024 not divisible by 3 devices (utils.py:252)
    (tmp_path / "bad.yaml").write_text("not_a_flag: 1\n")
    FLAGS.config = str(tmp_path / "bad")
    with pytest.raises(ValueError, match="Invalid args"):
        F.update_flags(FLAGS)
    FLAGS.config = None
    FLAGS.use_viewdirs = True
    with pytest.raises(NotImplementedError):
        F.check_scope(FLAGS)
    FLAGS.use_viewdirs = False


# each CLI's workspace: (max_rays, sparsity_npoints) from its flags, world = 2 ranks for training
_CLI_WORKSPACE = {
    "train": lambda a: (a.batch_size // 2, a.sparsity_npoints if a.sparsity_weight > 0 else 0),
    "eval": lambda a: (min(a.chunk, 8192), 0),
    "gen_video": lambda a: (min(a.chunk, 8192), 0),
    "gen_mesh": lambda a: (1024, 0),
    "extraction": lambda a: (min(a.chunk, 8192), 0),
}


@pytest.mark.parametrize("cli", sorted(_CLI_WORKSPACE))
def test_model_from_flags_matches_hand_copied_arguments(cli):
    """NerfModel.from_flags builds the model that each CLI built from its own copy of the model flags"""
    import types
    from plenoctree_b200.nerf import flags as F
    from plenoctree_b200.nerf.models import NerfModel
    defaults = {name: default for name, (_, default, _) in F._COMMON.items()}
    if cli == "extraction":
        defaults.update(F._OCTREE_DEFAULTS)
    variants = [dict(), dict(min_deg_point=2, max_deg_point=8, legacy_posenc_order=True), dict(net_activation="elu"),
                dict(net_activation="Tanh", sigma_activation="Softplus"), dict(sigma_activation="softplus"),
                dict(num_coarse_samples=256, num_fine_samples=768), dict(sparsity_weight=0.0, batch_size=4096),
                dict(sh_deg=4, near=0.5, far=3.0, white_bkgd=False, lindisp=True, num_fine_samples=0, chunk=2048,
                     min_deg_point=1, max_deg_point=9, net_activation="softplus", sigma_activation="softplus")]
    for kw in variants:
        args = types.SimpleNamespace(**{**defaults, "sh_deg": 3, **kw})
        max_rays, nsp = _CLI_WORKSPACE[cli](args)
        # the hand-built copy the CLIs passed, read back as get_model_state read it
        margs = type("A", (), dict(sh_deg=args.sh_deg, sigma_activation=args.sigma_activation,
                                   net_activation=args.net_activation, min_deg_point=args.min_deg_point,
                                   max_deg_point=args.max_deg_point, legacy_posenc_order=args.legacy_posenc_order,
                                   num_coarse_samples=args.num_coarse_samples,
                                   num_fine_samples=args.num_fine_samples, near=args.near, far=args.far,
                                   white_bkgd=args.white_bkgd, lindisp=args.lindisp, batch_size=max_rays,
                                   sparsity_npoints=nsp))
        old = NerfModel(sh_deg=margs.sh_deg, num_coarse_samples=margs.num_coarse_samples,
                        num_fine_samples=margs.num_fine_samples, near=margs.near, far=margs.far,
                        white_bkgd=margs.white_bkgd, lindisp=margs.lindisp, max_rays=margs.batch_size,
                        sparsity_npoints=margs.sparsity_npoints, device="cpu", sigma_activation=margs.sigma_activation,
                        min_deg_point=margs.min_deg_point, max_deg_point=margs.max_deg_point,
                        legacy_posenc_order=margs.legacy_posenc_order, net_activation=margs.net_activation)
        new = NerfModel.from_flags(args, max_rays=max_rays, sparsity_npoints=nsp, device="cpu")

        def fields(m):
            cfg = {k: getattr(m.cfg, k) for k, _ in m.cfg._fields_ if k != "posenc"}
            desc = None if m._posenc_struct is None else tuple(getattr(m._posenc_struct, k)
                                                               for k, _ in m._posenc_struct._fields_)
            return dict(sh_deg=m.sh_deg, nc=m.num_coarse_samples, nf=m.num_fine_samples, near=m.near, far=m.far,
                        white_bkgd=m.white_bkgd, lindisp=m.lindisp, max_rays=m.max_rays,
                        sparsity_npoints=m.sparsity_npoints, posenc=m.posenc, net_act_code=m.net_act_code,
                        sigma_act_code=m.sigma_act_code, P=m.P, cfg=cfg, desc=desc,
                        cfg_posenc_set=m.cfg.posenc is not None)
        assert fields(new) == fields(old), kw
        assert torch.equal(new.z_base, old.z_base), kw


def test_ssim_matches_reference_torch_twin(golden_dir):
    from plenoctree_b200.nerf.utils import compute_ssim
    z = np.load(os.path.join(golden_dir, "ssim.npz"))
    assert abs(float(compute_ssim(z["a"], z["b"], padding="same")) - float(z["ssim"])) < 1e-6
    # the JAX-side function ("valid" borders, nerf_sh/nerf/utils.py:396-466) executed over the numpy stand-ins
    zj = np.load(os.path.join(golden_dir, "ref_llff.npz"))
    assert abs(float(compute_ssim(z["a"], z["b"], padding="valid")) - float(zj["ssim_jax_valid"])) < 2e-6
    got_map = compute_ssim(z["a"], z["b"], padding="valid", return_map=True)
    got_map = got_map.cpu().numpy() if hasattr(got_map, "cpu") else np.asarray(got_map)
    assert got_map.shape == zj["ssim_jax_valid_map"].shape and np.abs(got_map - zj["ssim_jax_valid_map"]).max() < 2e-5
    same = float(compute_ssim(z["a"], z["a"]))
    assert abs(same - 1.0) < 1e-6
    assert float(compute_ssim(z["a"], z["b"])) < 1.0        # "valid" borders (JAX side)


def test_blender_loader_cpu(tmp_path):
    from plenoctree_b200.nerf import datasets as D
    from plenoctree_b200.nerf.utils import generate_rays, pose_spherical
    rs = np.random.RandomState(0)
    poses = [pose_spherical(30.0 * i, -30.0, 4.0) for i in range(3)]
    ims = [rs.uniform(0, 1, size=(10, 12, 3)).astype(np.float32) for _ in range(3)]
    D.write_blender_scene(str(tmp_path), {"test": ims}, {"test": poses}, 0.6911112070083618)
    args = type("A", (), dict(data_dir=str(tmp_path), factor=0, white_bkgd=True, batch_size=64, image_batching=False,
                              dataset="blender", render_path=False))
    ds = D.get_dataset("test", args, device="cpu")
    assert ds.size == 3 and (ds.h, ds.w) == (10, 12)
    assert abs(ds.focal - 0.5 * 12 / np.tan(0.5 * 0.6911112070083618)) < 1e-4
    assert np.abs(ds.images - np.stack(ims)).max() <= 1.0 / 255.0 + 1e-6           # 8-bit PNG round trip
    b = ds.next_test()
    want = generate_rays(12, 10, ds.focal, np.stack(poses)[:1])
    assert np.array_equal(b["rays"].directions, want.directions[0]) and b["pixels"].shape == (10, 12, 3)
    with open(os.path.join(str(tmp_path), "transforms_test.json")) as f:
        assert len(json.load(f)["frames"]) == 3


def _write_llff(d, images_u8, poses_bounds, factor):
    from PIL import Image
    sub = os.path.join(d, "images" + (f"_{factor}" if factor > 0 else ""))
    os.makedirs(sub, exist_ok=True)
    for i, im in enumerate(images_u8):
        Image.fromarray(im, mode="RGB").save(os.path.join(sub, f"{i:03d}.png"))
    np.save(os.path.join(d, "poses_bounds.npy"), poses_bounds)


@pytest.mark.parametrize("case,factor,spherify", [("fwd", 0, False), ("ring", 2, True)])
def test_llff_loader_matches_executed_reference(tmp_path, golden_dir, case, factor, spherify):
    """LLFF loader against the reference's own (nerf_sh/nerf/datasets.py:235-487 executed by
    tests/golden/make_golden.py ref_llff on the same synthetic scenes): recentred / spherified poses, focal, split,
    spiral / circle render path, NDC rays of the views and of the path."""
    from plenoctree_b200.nerf import datasets as D
    z = np.load(os.path.join(golden_dir, "ref_llff.npz"))
    _write_llff(str(tmp_path), z[f"{case}_images"], z[f"{case}_poses_bounds"], factor)
    for split in ("train", "test"):
        args = type("A", (), dict(data_dir=str(tmp_path), factor=factor, spherify=spherify, llffhold=4, batch_size=32,
                                  image_batching=True, dataset="llff", render_path=(split == "test"), white_bkgd=False))
        ds = D.get_dataset(split, args, device="cpu")
        k = f"{case}_{split}_"
        h, w, n = z[k + "hw_n"]
        assert (ds.h, ds.w, ds.n_examples) == (h, w, n)
        assert np.array_equal(ds.images, z[k + "images"])
        np.testing.assert_allclose(ds.camtoworlds, z[k + "camtoworlds"], rtol=0, atol=2e-6)
        np.testing.assert_allclose(ds.focal, z[k + "focal"], rtol=1e-7)
        for f, r in zip("odv", ds.rays_np):
            np.testing.assert_allclose(r, z[k + "rays_" + f], rtol=2e-5, atol=2e-6)
        if split == "test":
            assert ds.n_examples == 120
            np.testing.assert_allclose(ds.render_poses, z[k + "render_poses"], rtol=0, atol=2e-6)
            for f, r in zip("odv", ds.render_rays_np):
                np.testing.assert_allclose(r[::15], z[k + "render_rays_" + f], rtol=2e-5, atol=2e-6)
            b = ds.next_test()                                  # render_path: rays of the path, no pixels
            assert set(b) == {"rays"} and b["rays"].origins.shape == (h, w, 3)
        else:
            b = ds.next_train()
            assert b["pixels"].shape == (32, 3) and b["rays"].origins.shape == (32, 3)
            if not spherify:                                    # NDC: every origin sits on the near plane z = -1
                assert np.allclose(ds.rays_np.origins[..., 2], -1.0, atol=1e-5)


def test_host_helpers_match_executed_reference(golden_dir):
    from plenoctree_b200.nerf.rays import convert_to_ndc, pose_spherical
    z = np.load(os.path.join(golden_dir, "ref_llff.npz"))
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf.train import learning_rate_decay
    for a, want in zip(z["lr_in"], z["lr_out"]):                                    # executed reference schedule
        args = (a[0], a[1], a[2], a[3], int(a[4]), a[5])
        assert abs(learning_rate_decay(*args) - want) <= 1e-12 * want and abs(O.learning_rate_decay(*args) - want) <= 1e-12 * want
    for (th, ph, rad, ua), want in zip(z["pose_sph_in"], z["pose_sph_out"]):        # all six up axes
        np.testing.assert_allclose(pose_spherical(th, ph, rad, int(ua)), want, rtol=0, atol=1e-6)
    for near in (1.0, 0.5):
        o, d = convert_to_ndc(z["ndc_in_o"], z["ndc_in_d"], np.float32(21.5), 16, 12, near=near)
        np.testing.assert_allclose(o, z[f"ndc_o_{near}"], rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(d, z[f"ndc_d_{near}"], rtol=1e-6, atol=1e-7)


def test_marching_tetrahedra_sphere_is_closed_oriented_manifold():
    """nerf/mesh.py (stands in for PyMCubes in gen_mesh): on a sphere's signed distance the surface is watertight
    (every edge in exactly two triangles, once per direction), has Euler characteristic 2, outward normals (positive
    signed volume, within 1 % of the ball's) and vertices on the sphere to second order in the grid spacing."""
    from plenoctree_b200.nerf.mesh import marching_tetrahedra, save_obj
    n, r0 = 40, 0.6
    g = np.linspace(-1, 1, n)
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    v, f = marching_tetrahedra((r0 - np.sqrt(X * X + Y * Y + Z * Z)).astype(np.float32), 0.0)
    w = v * (2.0 / (n - 1)) - 1.0
    rad = np.linalg.norm(w, axis=1)
    assert rad.max() < r0 + 1e-6 and rad.min() > r0 - (2.0 / (n - 1)) ** 2
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    fwd, rev = d[:, 0] * len(v) + d[:, 1], d[:, 1] * len(v) + d[:, 0]
    assert len(np.unique(fwd)) == len(fwd) and np.array_equal(np.sort(fwd), np.sort(rev))
    assert len(v) - len(fwd) // 2 + len(f) == 2
    p0, p1, p2 = w[f[:, 0]], w[f[:, 1]], w[f[:, 2]]
    vol = float((p0 * np.cross(p1, p2)).sum() / 6.0)
    assert abs(vol / (4.0 / 3.0 * np.pi * r0 ** 3) - 1.0) < 0.01
    assert marching_tetrahedra(np.zeros((4, 4, 4), np.float32), 1.0)[1].shape == (0, 3)      # nothing inside


def test_gen_mesh_grid_and_scaling_cpu(tmp_path):
    """gen_mesh's grid walk (points = linspace(c1, c2, reso) per axis, "ij" order, chunked) and the reference's
    vertex scaling c1 + index * (c2 - c1) / reso (gen_mesh.py:105-129), with an analytic density in place of the MLP."""
    from plenoctree_b200.nerf_sh import gen_mesh as GM
    from plenoctree_b200.nerf.mesh import save_obj

    class Field:
        device = torch.device("cpu")
        calls = 0

        def eval_points_raw(self, pts, coarse=False, want_rgb=True):
            Field.calls += 1
            assert pts.shape[1] == 3 and not want_rgb
            c = torch.tensor([0.2, -0.1, 0.3])
            return None, (10.0 - 10.0 * ((pts - c) ** 2).sum(1, keepdim=True).sqrt())         # sigma = 6 at r = 0.4

    reso, c1, c2 = [24, 30, 20], [-1.0, -1.5, -0.5], [1.0, 1.0, 1.5]
    sig = GM.sigma_grid(Field(), c1, c2, reso, chunk=1000)
    assert Field.calls == -(-24 * 30 * 20 // 1000) and sig.shape == (24, 30, 20)
    x, y, z = np.linspace(-1, 1, 24)[5], np.linspace(-1.5, 1, 30)[17], np.linspace(-0.5, 1.5, 20)[3]
    assert abs(sig[5, 17, 3] - (10 - 10 * np.sqrt((x - 0.2) ** 2 + (y + 0.1) ** 2 + (z - 0.3) ** 2))) < 1e-4
    verts, faces = GM.marching_cubes(Field(), c1, c2, reso, 6.0, 5000)
    assert len(faces) > 100
    # the reference scales by (c2 - c1) / reso (not reso - 1): undo it to land on the sampled field's sphere
    idx = (verts - np.array(c1)) / ((np.array(c2) - np.array(c1)) / np.array(reso))
    world = np.array(c1) + idx * (np.array(c2) - np.array(c1)) / (np.array(reso) - 1)
    rad = np.linalg.norm(world - np.array([0.2, -0.1, 0.3]), axis=1)
    assert abs(rad - 0.4).max() < 0.01
    save_obj(verts, faces, str(tmp_path / "m.obj"), vert_rgb=np.zeros_like(verts))
    lines = open(tmp_path / "m.obj").read().splitlines()
    assert sum(l.startswith("v ") for l in lines) == len(verts) and sum(l.startswith("f ") for l in lines) == len(faces)
    assert len(lines[0].split()) == 7 and min(int(t) for l in lines if l.startswith("f ") for t in l.split()[1:]) == 1


def test_task_manager_expands_dispatches_and_records(tmp_path):
    """octree.task_manager (octree/task_manager.py:28-195; scene-level replicas): task expansion with the "{%}" scene
    mark, one command triple per task with the task's flags (the reference's syn_sh16.json flag set), one worker per
    GPU id with CUDA_VISIBLE_DEVICES pinned, results.txt = capacity / raw metrics / optimised metrics."""
    import subprocess
    from plenoctree_b200.octree import task_manager as TM
    spec = {"data_root": str(tmp_path / "data"), "train_root": str(tmp_path / "ckpt"),
            "scenes": ["chair", "drums", "lego"],
            "scene_tasks": [{"octree_name": "", "train_dir": "{%}", "data_dir": "{%}", "config": "nerf_sh/config/blender",
                             "extr_flags": ["--autoscale", "--scale_alpha_thresh", "0.1", "--radius", "1.4",
                                            "--samples_per_cell", "256", "--no_early_stop", "--renderer_step_size", "1e-5"],
                             "opt_flags": ["--num_epochs", "80", "--sgd", "--lr", "1e7", "--no_early_stop",
                                           "--renderer_step_size", "1e-5"],
                             "eval_flags": ["--renderer_step_size", "1e-5"]}],
            "tasks": [{"octree_name": "oct_m", "train_dir": "materials", "data_dir": "materials",
                       "config": "nerf_sh/config/blender", "extr_flags": ["--bbox_scale", "1.1"], "opt_flags": [],
                       "eval_flags": []}]}
    tasks = TM.expand_tasks(spec)
    assert [os.path.basename(t["train_dir"]) for t in tasks] == ["materials", "chair", "drums", "lego"]
    store, cmds, raw, final = TM.commands_for(tasks[1], keep_raw=True, python="python")
    assert store == os.path.join(spec["train_root"], "chair", "octrees", "")          # octree_name "" like the reference's
    assert cmds["extract"][:4] == ["python", "-u", "-m", "octree.extraction"] and "--is_jaxnerf_ckpt" in cmds["extract"]
    assert cmds["extract"][cmds["extract"].index("--output") + 1] == raw and raw.endswith("tree.npz")
    assert cmds["optimize"][cmds["optimize"].index("--output") + 1] == final and final.endswith("tree_opt.npz")
    assert cmds["evaluate"][cmds["evaluate"].index("--input") + 1] == final and cmds["extract"][-2:] == ["--renderer_step_size", "1e-5"]
    assert TM.parse_capacity("x\nplenoctree_b200.N3Tree(N=2, data_dim=49, depth_limit=10, capacity:1234/2048, ...)\n") == 1234
    assert TM.parse_metrics("foo\nAverage PSNR 31.25 SSIM 0.961\n") [:2] == (31.25, 0.961)
    assert TM.parse_metrics("Average PSNR 30.0 SSIM 0.9 LPIPS 0.05\n") == (30.0, 0.9, 0.05) and TM.parse_metrics("nothing") is None
    seen = []

    def fake_run(argv, env=None, check=False, stdout=None, text=None):
        seen.append((argv[3], env["CUDA_VISIBLE_DEVICES"], argv[argv.index("--data_dir") + 1]))
        out = ""
        if argv[3] == "octree.extraction":
            out = "tree(capacity:77/128)\nAverage PSNR 25.5 SSIM 0.9\n"
        elif argv[3] == "octree.optimization":
            if "drums" not in argv[argv.index("--data_dir") + 1]:               # drums: optimisation leaves no tree
                open(argv[argv.index("--output") + 1], "w").write("npz")
        else:
            out = "Average PSNR 28.5 SSIM 0.95\n"
        return subprocess.CompletedProcess(argv, 0, stdout=out)

    for t in tasks[1:]:
        os.makedirs(t["train_dir"]); os.makedirs(t["data_dir"])
    res = TM.run_all(tasks[1:], gpus=[3, 5], keep_raw=True, run=fake_run)
    assert {g for _, g, _ in seen} <= {"3", "5"} and len(seen) == 3 + 2 + 3      # drums skips the evaluation
    assert res[0]["capacity"] == 77 and res[0]["opt"][:2] == (28.5, 0.95) and res[1]["opt"] is None
    lines = open(os.path.join(tasks[1]["train_dir"], "octrees", "results.txt")).read().split("\n")
    assert lines[0] == "77" and lines[1].startswith("25.5000000000 0.9000000000 nan") and lines[2].startswith("28.5000000000")
    drums = open(os.path.join(tasks[2]["train_dir"], "octrees", "results.txt")).read().split("\n")
    assert drums[2] == drums[1]                                                   # raw metrics repeated
    (tmp_path / "t.json").write_text(json.dumps(spec))
    assert TM.main([str(tmp_path / "t.json"), "--gpus", "0 1", "--dry_run"]) == 0


def test_presets_equal_reference_config_files(golden_dir, tmp_path):
    """plenoctree_b200/presets.py stands in for nerf_sh/config/{blender,tt}.yaml and octree/config/{syn_sh16,tt_sh25}.json
    when those files are absent (README command lines); values pinned by tests/golden/ref_configs.json, which
    make_golden.py parsed from the reference's files.  `--config <dir>/blender` without a file selects the preset."""
    from plenoctree_b200 import presets as P
    from plenoctree_b200.nerf import flags as F
    from plenoctree_b200.octree.task_manager import expand_tasks
    ref = json.load(open(os.path.join(golden_dir, "ref_configs.json")))
    for n in ("blender", "tt"):
        assert P.NERF_SH[n] == ref["nerf_sh"][n]

    def options(fl):
        d, i = {}, 0
        while i < len(fl):
            if i + 1 < len(fl) and not fl[i + 1].startswith("--"):
                d[fl[i]] = fl[i + 1]; i += 2
            else:
                d[fl[i]] = True; i += 1
        return d
    for n in ("syn_sh16", "tt_sh25"):
        mine = P.octree_tasks_preset(f"octree/config/{n}.json")
        a = sorted(expand_tasks(ref["octree"][n]), key=lambda t: t["train_dir"])
        b = sorted(expand_tasks(mine), key=lambda t: t["train_dir"])
        assert len(a) == len(b) and len(a) == {"syn_sh16": 8, "tt_sh25": 5}[n]
        for x, y in zip(a, b):
            assert all(x[k] == y[k] for k in ("train_dir", "data_dir", "octree_name", "config", "opt_flags", "eval_flags"))
            assert options(x["extr_flags"]) == options(y["extr_flags"])
    assert P.octree_tasks_preset("octree/config/other.json") is None
    FLAGS = _set_flags(train_dir="/tmp/x", data_dir="/tmp/y", config=str(tmp_path / "nerf_sh" / "config" / "tt"), sh_deg=1)
    F.update_flags(FLAGS)
    assert (FLAGS.dataset, FLAGS.sh_deg, FLAGS.far, FLAGS.sparsity_length) == ("nsvf", 4, 4.0, 0.2)
    FLAGS.config = str(tmp_path / "unknown")
    with pytest.raises(FileNotFoundError):
        F.update_flags(FLAGS)
    _set_flags(config=None, dataset="blender", sh_deg=3, near=2.0, far=6.0, sparsity_radius=1.5, sparsity_length=0.05)


def test_median_cut_and_tree_compression(tmp_path):
    """octree.compression (octree/compression.py:39-145): balanced median cut (2^bits boxes of equal population,
    palette = box mean, error falling with bits), the compressed npz's keys / shapes / dtypes, sigma thresholding,
    --retain, and the CLI's skip rules.  svox's own quantiser is absent: parity unpinned (module docstring)."""
    from plenoctree_b200.octree import compression as C
    rs = np.random.RandomState(0)
    pts = (rs.normal(size=(5000, 3)) * np.array([3.0, 1.0, 0.3])).astype(np.float32)
    errs = []
    for bits in (0, 1, 4, 8):
        pal, idx = C.median_cut(pts, bits)
        assert pal.shape == (1 << bits, 3) and idx.shape == (5000,) and idx.min() >= 0 and idx.max() < (1 << bits)
        cnt = np.bincount(idx, minlength=1 << bits)
        assert cnt.max() - cnt.min() <= bits                            # halves differ by at most one per round
        for b in (0, (1 << bits) - 1):
            assert np.allclose(pal[b], pts[idx == b].mean(0), atol=1e-5)
        errs.append(float(((pts - pal[idx]) ** 2).mean()))
    assert errs[0] > errs[1] > errs[2] > errs[3] and errs[3] < 0.02 * errs[0]
    pal, idx = C.median_cut(pts[:1].repeat(7, 0), 3)                        # identical points: never split
    assert set(idx.tolist()) == {0} and np.allclose(pal[0], pts[0]) and not pal[1:].any()
    palw, idxw = C.median_cut(pts, 3, weights=rs.uniform(size=5000))
    assert len(np.unique(idxw)) == 8
    # ---- a small SH4 (K = 4) tree file ----
    n_nodes, N, K = 20, 2, 4
    data = rs.normal(size=(n_nodes, N, N, N, 3 * K + 1)).astype(np.float32)
    data[..., -1] = rs.uniform(0, 10, size=data.shape[:-1])
    z = dict(data=data.astype(np.float16), child=np.zeros((n_nodes, N, N, N), np.int32), parent_depth=np.zeros((n_nodes, 2), np.int32),
             geom_resize_fact=np.float64(1.5), n_free=np.int32(0), n_internal=np.int32(n_nodes), depth_limit=np.int32(10),
             invradius3=np.ones(3, np.float32), offset=np.zeros(3, np.float32), data_dim=np.int32(3 * K + 1), data_format="SH4")
    c = C.compress_tree(dict(z), bits=5, sigma_thresh=2.0, retain=1)
    assert not {"data", "parent_depth", "geom_resize_fact", "n_free", "n_internal", "depth_limit"} & set(c)
    assert c["quant_colors"].shape == (K - 1, 32, 3) and c["quant_colors"].dtype == np.float16
    assert c["quant_map"].shape == (K - 1, n_nodes, N, N, N) and c["quant_map"].dtype == np.uint16
    assert c["sigma"].shape == (n_nodes, N, N, N) and c["data_retained"].shape == (1, n_nodes, N, N, N, 3)
    sig = z["data"][..., -1].astype(np.float32)
    assert np.array_equal(c["sigma"] == 0, sig <= 2.0) and np.array_equal(c["sigma"][sig > 2.0], sig[sig > 2.0])
    back = C.decompress_data(c)
    kept = sig > 2.0
    orig = z["data"].astype(np.float32)
    assert not back[~kept].any()
    rgb_o = orig[kept][:, :-1].reshape(-1, 3, K)
    rgb_b = back[kept][:, :-1].reshape(-1, 3, K)
    assert np.abs(rgb_o[..., 0] - rgb_b[..., 0]).max() < 2e-3                       # retained basis function: fp16 copy
    assert 0 < ((rgb_o[..., 1:] - rgb_b[..., 1:]) ** 2).mean() < 0.35 * (rgb_o[..., 1:] ** 2).mean()
    src = tmp_path / "tree.npz"
    np.savez(src, **z)
    assert C.main([str(src), "--out_dir", str(tmp_path / "min"), "--bits", "6"]) == 0
    out = np.load(tmp_path / "min" / "tree.npz")
    assert "quant_map" in out.files and "data" not in out.files and out["quant_colors"].shape == (K, 64, 3)
    stamp = os.path.getmtime(tmp_path / "min" / "tree.npz")
    C.main([str(src), "--out_dir", str(tmp_path / "min")])                            # exists, no --overwrite: skipped
    assert os.path.getmtime(tmp_path / "min" / "tree.npz") == stamp
    C.main([str(src), "--out_dir", str(tmp_path / "raw"), "--noquant"])
    assert "data" in np.load(tmp_path / "raw" / "tree.npz").files


def test_lpips_network_and_optional_weights(tmp_path, monkeypatch):
    """nerf/lpips.py: the VGG-16 feature stack reproduces torchvision's `vgg16().features` at the five LPIPS taps
    when loaded from its state dict (random weights: the ImageNet file cannot ship), the linear heads load from
    LPIPS-v0.1-style keys, the distance is 0 for identical images / symmetric / positive, `load_lpips` finds weights in
    $POB_LPIPS_DIR and returns None without them."""
    import torchvision
    from plenoctree_b200.nerf import lpips as L
    torch.manual_seed(0)
    tv = torchvision.models.vgg16(weights=None).eval()
    net = L.LPIPSVGG().eval()
    net.load_vgg16(tv.state_dict())
    x = torch.rand(2, 3, 40, 36)
    taps = net.features(x)
    for tap, end in zip(taps, (4, 9, 16, 23, 30)):                      # relu1_2, relu2_2, relu3_3, relu4_3, relu5_3
        with torch.no_grad():
            want = tv.features[:end](x)
        assert tap.shape == want.shape and torch.allclose(tap, want, atol=1e-5)
    heads = {f"lin{l}.model.1.weight": torch.rand(1, c, 1, 1) for l, (_, c) in enumerate(L._BLOCKS)}
    net.load_linear_heads(heads)
    a, b = torch.rand(3, 40, 36), torch.rand(3, 40, 36)
    d_ab, d_ba, d_aa = float(net(a, b)[0]), float(net(b, a)[0]), float(net(a, a)[0])
    assert d_aa == 0.0 and d_ab > 0 and abs(d_ab - d_ba) < 1e-6 * d_ab
    assert abs(float(net(2 * a - 1, 2 * b - 1, normalize=False)[0]) - d_ab) < 1e-6 * d_ab
    # by hand for the first tap: unit-normalised features, squared difference, head weights, spatial mean
    sa, sb = [(2 * v[None] - 1 - net.shift) / net.scale for v in (a, b)]
    fa, fb = net.features(sa)[0], net.features(sb)[0]
    fa, fb = fa / (fa.pow(2).sum(1, keepdim=True).sqrt() + 1e-10), fb / (fb.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
    first = float((((fa - fb) ** 2) * heads["lin0.model.1.weight"]).sum(1).mean())
    zero_rest = {k: (v if k.startswith("lin0") else torch.zeros_like(v)) for k, v in heads.items()}
    assert abs(float(L.LPIPSVGG().load_vgg16(tv.state_dict()).load_linear_heads(zero_rest)(a, b)[0]) - first) < 1e-6
    # weight discovery
    monkeypatch.setenv("POB_LPIPS_DIR", str(tmp_path))
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "nohub"))
    assert L.load_lpips() is None
    torch.save(tv.state_dict(), tmp_path / "vgg16-397923af.pth")
    torch.save(heads, tmp_path / "vgg.pth")
    fn = L.load_lpips()
    assert fn is not None and abs(fn(a, b) - d_ab) < 1e-6 * d_ab


def test_eval_octree_metrics_with_a_stub_renderer(monkeypatch):
    """octree.evaluation.eval_octree's bookkeeping (PSNR / SSIM averages, optional LPIPS into `metrics`, frames) on the
    CPU, the renderer replaced by a stub that returns the ground truth plus a known offset."""
    from plenoctree_b200.octree import evaluation as EV

    class Tree:
        device = torch.device("cpu")

    class Renderer:
        def __init__(self, t, step_size):
            self.calls = 0

        def render_persp(self, c2w, width, height, fx, fast):
            return torch.full((height, width, 3), 0.5 + 0.1 * float(c2w[0, 0]))
    monkeypatch.setattr(EV, "VolumeRenderer", Renderer)
    ds = type("D", (), dict(w=20, h=16, focal=30.0, size=2, camtoworlds=np.stack([np.eye(4), 2 * np.eye(4)]).astype(np.float32),
                            images=np.full((2, 16, 20, 3), 0.5, np.float32)))
    args = type("A", (), dict(renderer_step_size=1e-3, no_early_stop=False))
    psnr, ssim = EV.eval_octree(Tree(), ds, args)
    want = np.mean([-10 * np.log10(0.1 ** 2), -10 * np.log10(0.2 ** 2)])
    assert abs(psnr - want) < 1e-4 and 0 < ssim < 1
    m = {}
    psnr2, ssim2, frames = EV.eval_octree(Tree(), ds, args, want_frames=True, lpips_fn=lambda gt, im: float((gt - im).abs().mean()),
                                          metrics=m)
    assert (psnr2, ssim2) == (psnr, ssim) and len(frames) == 2 and frames[0].dtype == np.uint8
    assert abs(m["lpips"] - 0.15) < 1e-6
    m = {}
    EV.eval_octree(Tree(), ds, args, metrics=m)
    assert np.isnan(m["lpips"])


@pytest.mark.gpu
def test_cli_chain_train_eval_extract_optimize(tmp_path):
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf import datasets as D
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf.utils import generate_rays, pose_spherical, render_image
    from plenoctree_b200.nerf_sh import eval as EV, train as TR
    from plenoctree_b200.octree import evaluation as OE, extraction as EX, optimization as OP
    from plenoctree_b200.octree import N3Tree
    # ---- synthetic scene: views of a teacher NeRF-SH field (random weights, density head scaled up) ----
    sh_deg, W = 3, 48
    ft = np.concatenate([O.init_flat_params(sh_deg, 7001, bias_scale=0.05), O.init_flat_params(sh_deg, 7002, bias_scale=0.05)])
    P = O.param_count(sh_deg)
    for m in range(2):
        off = m * P + P - 48 - 1 - 256 * 48 - 256
        ft[off:off + 256] *= 30.0
    teacher = NerfModel(sh_deg=sh_deg, max_rays=4096)
    teacher.set_params(ft)
    cam_x = 0.6911112070083618
    focal = 0.5 * W / np.tan(0.5 * cam_x)
    rs = np.random.RandomState(3)
    splits = {"train": 8, "val": 2, "test": 2}
    poses = {k: [pose_spherical(rs.uniform(-180, 180), rs.uniform(-80, -10), 4.0) for _ in range(n)] for k, n in splits.items()}
    images = {}
    for k in splits:
        rays = generate_rays(W, W, focal, np.stack(poses[k]))
        images[k] = [render_image(teacher, Rays(rays.origins[i], rays.directions[i], rays.viewdirs[i]))[0].cpu().numpy()
                     for i in range(splits[k])]
    data_dir, train_dir = str(tmp_path / "scene"), str(tmp_path / "ckpt")
    D.write_blender_scene(data_dir, images, poses, cam_x)
    (tmp_path / "cfg.yaml").write_text("dataset: blender\nfactor: 0\nnum_coarse_samples: 64\nnum_fine_samples: 128\n"
                                       "use_viewdirs: false\nwhite_bkgd: true\nbatch_size: 1024\nsh_deg: 3\n"
                                       "randomized: true\nmax_steps: 300\n")
    EX._define_cli_flags()
    OP._define_cli_flags()
    FLAGS = _set_flags(train_dir=train_dir, data_dir=data_dir, config=str(tmp_path / "cfg"), save_every=300,
                       print_every=100, render_every=0, sparsity_npoints=1000, lr_init=2e-3, lr_final=2e-4, chunk=4096,
                       noise_std=None, image_batching=True)
    # ---- nerf_sh.train / nerf_sh.eval ----
    model, state = TR.main(None)
    assert os.path.exists(os.path.join(train_dir, "checkpoint_300")) and state.step == 300
    psnr, ssim = EV.main(None)
    from plenoctree_b200.nerf_sh import gen_video as GV                 # orbit video from the same checkpoint
    FLAGS.num_views, FLAGS.height, FLAGS.width, FLAGS.elevation, FLAGS.radius = 3, 32, 32, -30.0, "4.0"
    vdir = GV.main(None)
    assert sorted(os.listdir(os.path.join(vdir, "frames"))) == ["0000.png", "0001.png", "0002.png"]
    assert os.path.exists(os.path.join(train_dir, "test_preds", "000.png"))
    assert float(open(os.path.join(train_dir, "test_preds", "psnr.txt")).read()) == pytest.approx(psnr)
    fresh = NerfModel(sh_deg=sh_deg, max_rays=4096)
    fresh.init_params(20200823)
    rays = generate_rays(W, W, focal, np.stack(poses["test"]))
    gt = torch.from_numpy(images["test"][0]).cuda()
    p_init = -10 * np.log10(float(((render_image(fresh, Rays(rays.origins[0], rays.directions[0], rays.viewdirs[0]))[0] - gt) ** 2).mean()))
    assert psnr > p_init + 2.0, (p_init, psnr)          # 300 steps on 8 tiny views: it learns
    # ---- north-star parity bar on a full 800x800 frame of the TRAINED field: the timed precision (fp16 operands)
    # against the fp32-class mode (fp16x3, itself within 1e-5 of the oracle: test_render.py), PSNR vs the teacher's
    # own 800x800 render must agree within 0.05 dB, and the two renders within 1e-3 RMS of each other
    from plenoctree_b200 import ops
    big = 800
    fbig = 0.5 * big / np.tan(0.5 * cam_x)
    rb = generate_rays(big, big, fbig, np.stack(poses["test"][:1]))
    rb = Rays(rb.origins[0], rb.directions[0], rb.viewdirs[0])
    gt_big = render_image(teacher, rb, precision=ops.PREC_FP16X3)[0]
    im16 = render_image(model, rb, precision=ops.PREC_FP16)[0]
    im32 = render_image(model, rb, precision=ops.PREC_FP16X3)[0]
    psnr16 = -10 * np.log10(float(((im16 - gt_big) ** 2).mean()))
    psnr32 = -10 * np.log10(float(((im32 - gt_big) ** 2).mean()))
    rms = float(((im16 - im32) ** 2).mean().sqrt())
    _record_pipeline("fullframe_800x800_trained", dict(psnr_fp16=psnr16, psnr_fp16x3=psnr32, rms_fp16_vs_fp16x3=rms))
    assert abs(psnr16 - psnr32) < 0.05, (psnr16, psnr32)
    assert rms < 1e-3, rms
    # resuming continues from the checkpoint's step and Adam state
    FLAGS.config = None          # the YAML would re-apply max_steps: 300 (update_flags overrides, like the reference)
    FLAGS.max_steps = 310
    FLAGS.save_every = 10
    _, state2 = TR.main(None)
    assert state2.step == 310 and os.path.exists(os.path.join(train_dir, "checkpoint_310"))
    # ---- octree.extraction (flax-format checkpoint) ----
    FLAGS.is_jaxnerf_ckpt = True
    FLAGS.init_grid_depth = 5
    FLAGS.samples_per_cell = 8
    FLAGS.masking_mode = "sigma"      # 8 views of 48x48 rays are too sparse for the weight mask (tests/test_octree.py covers it)
    FLAGS.alpha_thresh = 0.01
    FLAGS.renderer_step_size = 1e-3
    FLAGS.radius = "1.5"
    FLAGS.output = str(tmp_path / "tree.npz")
    FLAGS.eval = False
    tree = EX.main(None)
    assert os.path.exists(FLAGS.output) and tree.max_depth == 5
    test_ds = D.get_dataset("test", FLAGS, device="cuda")
    p_tree, s_tree = OE.eval_octree(tree, test_ds, FLAGS)
    # the 64^3 tree of a field trained for 300 steps is a coarse stand-in; it must still beat the untrained model
    assert p_tree > p_init + 1.0 and np.isfinite(s_tree), (p_init, psnr, p_tree)
    # ---- octree.optimization ----
    FLAGS.input = FLAGS.output
    FLAGS.output = str(tmp_path / "tree_opt.npz")
    FLAGS.num_epochs = 6
    FLAGS.val_interval = 2
    FLAGS.lr = 1e7 * (W * W) / (800.0 * 800.0) / 4
    FLAGS.continue_on_decrease = True
    best, p_val = OP.main(None)
    if best is not None:
        assert os.path.exists(FLAGS.output)
        t2 = N3Tree.load(FLAGS.output)
        p_opt, _ = OE.eval_octree(t2, test_ds, FLAGS)
        assert p_opt > p_tree - 0.5, (p_tree, p_opt)
    _record_pipeline("cli_chain", {"psnr_nerf_init": p_init, "psnr_nerf_300_steps": psnr, "ssim_nerf": ssim,
                                   "psnr_tree": p_tree, "psnr_tree_val_after_opt": p_val,
                                   "tree_nodes": int(tree.n_internal)})
def test_nsvf_loader_and_tt_config_cpu(tmp_path):
    """nerf_sh/config/tt.yaml selects `dataset: nsvf` (BASELINE configs[2]); the loader honours the split prefixes,
    the camera flip and bbox.txt (extraction --bbox_from_data)."""
    from plenoctree_b200.nerf import datasets as D, flags as F
    from plenoctree_b200.nerf.utils import pose_spherical
    rs = np.random.RandomState(1)
    poses = {"train": [pose_spherical(40.0 * i, -20.0, 2.5) for i in range(3)], "val": [pose_spherical(10.0, -60.0, 2.5)]}
    ims = {k: [rs.uniform(0, 1, size=(9, 16, 3)).astype(np.float32) for _ in v] for k, v in poses.items()}
    D.write_nsvf_scene(str(tmp_path / "scene"), ims, poses, focal=20.0, bbox=[-1, -2, -3, 1, 2, 3])
    (tmp_path / "tt.yaml").write_text("dataset: nsvf\nimage_batching: false\nfactor: 0\nnum_coarse_samples: 64\n"
                                      "num_fine_samples: 128\nuse_viewdirs: false\nwhite_bkgd: true\nbatch_size: 1024\n"
                                      "randomized: true\nsh_deg: 4\nmax_steps: 2000000\nnear: 0.0\nfar: 4.0\n"
                                      "sparsity_radius: 5.0\nsparsity_length: 0.2\n")   # = nerf_sh/config/tt.yaml
    FLAGS = _set_flags(train_dir=str(tmp_path), data_dir=str(tmp_path / "scene"), config=str(tmp_path / "tt"))
    F.update_flags(FLAGS)
    F.check_scope(FLAGS)
    assert (FLAGS.dataset, FLAGS.sh_deg, FLAGS.far, FLAGS.sparsity_radius) == ("nsvf", 4, 4.0, 5.0)
    tr = D.get_dataset("train", FLAGS, device="cpu")
    te = D.get_dataset("test", FLAGS, device="cpu")          # no 2_ files: falls back to the 1_ (val) images
    assert tr.size == 3 and te.size == 1 and (tr.h, tr.w) == (9, 16) and tr.focal == 20.0
    assert np.allclose(tr.camtoworlds, np.stack(poses["train"]), atol=1e-6)
    assert np.allclose(te.camtoworlds[0], poses["val"][0], atol=1e-6)
    assert np.allclose(tr.bbox, [-1, -2, -3, 1, 2, 3])
    b = tr.next_train()
    assert b["pixels"].shape == (1024, 3) and b["rays"].origins.shape == (1024, 3)
    FLAGS.config = None
    FLAGS.dataset = "blender"
    FLAGS.sh_deg = 3
    FLAGS.near, FLAGS.far, FLAGS.sparsity_radius, FLAGS.sparsity_length = 2.0, 6.0, 1.5, 0.05


def test_flag_tables_match_the_reference(golden_dir):
    """tests/golden/flags.json = every flags.DEFINE_* of the reference (AST of nerf_sh/nerf/utils.py,
    octree/nerf/utils.py, octree/extraction.py, octree/optimization.py): same names, kinds and defaults here."""
    import re
    from plenoctree_b200.nerf import flags as F
    ref = json.load(open(os.path.join(golden_dir, "flags.json")))
    kind_of = lambda k: "string" if k == "enum" else k
    mine = F._COMMON
    r = ref["nerf_sh/nerf/utils.py"]
    assert len(r) >= 50
    for name, (kind, default) in r.items():
        assert name in mine, name
        assert mine[name][0] == kind_of(kind) and mine[name][1] == default, (name, mine[name][:2], kind, default)
    for name, (kind, default) in ref["octree/nerf/utils.py"].items():
        assert name in mine, name
        want = F._OCTREE_DEFAULTS.get(name, mine[name][1])
        assert mine[name][0] == kind_of(kind) and want == default, (name, want, default)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for mod, key in (("extraction", "octree/extraction.py"), ("optimization", "octree/optimization.py")):
        src = open(os.path.join(root, "plenoctree_b200", "octree", mod + ".py")).read()
        table = eval("{" + re.search(r"F\.define\(\{(.*?)\}\)", src, re.S).group(1) + "}")
        assert set(table) == set(ref[key]), (mod, set(table) ^ set(ref[key]))
        for name, (kind, default) in ref[key].items():
            assert table[name][0] == kind_of(kind) and table[name][1] == default, (mod, name)


def test_reference_module_paths_and_yaml(tmp_path):
    """README.md:58-67,120-135 call `python -m nerf_sh.train --config nerf_sh/config/blender ...` and
    `python -m octree.extraction ...`: the top-level shims resolve to this package's CLIs and a config file with the
    reference's keys (nerf_sh/config/blender.yaml) overrides the flags (YAML > command line, utils.py:233-244)."""
    import subprocess
    import sys
    cfg = tmp_path / "blender.yaml"
    cfg.write_text("dataset: blender\nimage_batching: false\nfactor: 0\nnum_coarse_samples: 64\n"
                   "num_fine_samples: 128\nuse_viewdirs: false\nwhite_bkgd: true\nbatch_size: 1024\nsh_deg: 3\n"
                   "randomized: true\nmax_steps: 2000000\n")
    code = (
        "import sys\n"
        "from absl import flags\n"
        "import nerf_sh.train as T, nerf_sh.eval, nerf_sh.gen_video as GV, nerf_sh.gen_mesh\n"
        "import octree.extraction, octree.optimization, octree.evaluation\n"
        "assert GV.orbit_poses(8, -30.0, 4.0, 3).shape == (8, 4, 4)\n"
        "from plenoctree_b200.nerf import flags as F\n"
        "assert T.main.__module__ == 'plenoctree_b200.nerf_sh.train'\n"
        f"flags.FLAGS(['prog', '--train_dir', '/tmp/x', '--data_dir', '/tmp/y', '--config', r'{cfg.with_suffix('')}', "
        "'--sh_deg', '1', '--batch_size', '4096'])\n"
        "F.update_flags(flags.FLAGS)\n"
        "F.check_flags(flags.FLAGS)\n"
        "print(flags.FLAGS.sh_deg, flags.FLAGS.batch_size, flags.FLAGS.num_fine_samples, flags.FLAGS.max_steps)\n")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=root, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split()[-4:] == ["3", "1024", "128", "2000000"], r.stdout    # the YAML wins over the command line

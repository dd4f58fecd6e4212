"""Generate tests/golden/ref_optimization_momentum.npz by EXECUTING the reference's octree/optimization.py `main`
unmodified (the reference tree make_golden.py reads, whose helpers this imports) with torch.optim.SGD
momentum and Nesterov momentum and --render_interval, on the scene of ref_optimization.npz.

    python tests/golden/make_golden_momentum.py

The run harness restates make_golden.py's gen_ref_optimization (same scene, same svox stand-in) and adds an imageio
stand-in that records what --render_interval writes.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, O, _use_reference_octree, synthetic_octree  # noqa: E402


def run_ref_optimization(runs):
    """Execute the reference's octree/optimization.py `main` (:133-248) unmodified on the CPU: Blender loader of the
    octree side, per-image render -> clamp -> MSE -> backward -> torch.optim.SGD step, validation PSNR every epoch,
    best-model bookkeeping and save.  `svox` is a stand-in: N3Tree = an nn.Module holding the oracle tree's arrays
    (`data` is the Parameter SGD updates), VolumeRenderer.render_persp = an autograd Function around the oracle's
    forward / backward march.  The renderer internals are therefore the oracle's; what is pinned is the reference's
    training-step semantics around it (clamp gradient, mean normalisation, update order, PSNR, best-of-validation).
    `imageio` is a stand-in that records every imwrite call (path relative to the scene directory, array, and the
    render the reference took it from).

    runs: list of (lr, extra command-line flags), executed in order on the scene of ref_optimization.npz (built by
    make_golden.py's gen_ref_optimization with the same seeds; checked against the committed file).
    -> [per-run dict]"""
    import contextlib
    import copy
    import io
    import json
    import tempfile
    import types
    from PIL import Image
    from oracle import octree_oracle as OO
    H = W = 6
    focal_angle = 0.9
    focal = 0.5 * W / np.tan(0.5 * focal_angle)
    step_size = 1e-3
    teacher = synthetic_octree(77)
    student = synthetic_octree(77)
    rs = np.random.RandomState(5)
    n = student.n_internal
    student.data[:n] = (student.data[:n] + rs.normal(scale=0.3, size=student.data[:n].shape)).astype(np.float32)
    student.data[:n, ..., -1] = np.maximum(student.data[:n, ..., -1], 0.0)
    poses = {"train": [O.pose_spherical(40.0 * i - 60.0, -30.0, 3.0) for i in range(3)],
             "val": [O.pose_spherical(25.0, -20.0, 3.0), O.pose_spherical(-110.0, -45.0, 3.0)]}

    class TreeModule(torch.nn.Module):
        def __init__(self, o):
            super().__init__()
            self.o = o
            self.data = torch.nn.Parameter(torch.from_numpy(o.data[:o.n_internal].copy()))

        @classmethod
        def load(cls, path, map_location="cpu"):
            z = np.load(path)
            o = OO.N3Tree(N=2, data_dim=int(z["data_dim"]), depth_limit=int(z["depth_limit"]), init_reserve=int(z["n_internal"]),
                          geom_resize_fact=float(z["geom_resize_fact"]), data_format=str(z["data_format"]))
            o.invradius, o.offset = z["invradius3"].astype(np.float32), z["offset"].astype(np.float32)
            o.child, o.parent_depth = z["child"].copy(), z["parent_depth"].copy()
            o.data = z["data"].astype(np.float32)
            o.n_internal = int(z["n_internal"])
            return cls(o)

        def clone(self, device="cpu"):
            c = TreeModule(copy.deepcopy(self.o))
            c.data = torch.nn.Parameter(self.data.detach().clone())
            return c

        def save(self, path, compress=False):
            self.o.data = self.data.detach().numpy().copy()
            st = self.o.state()
            st["data"] = self.o.data[:self.o.n_internal].astype(np.float32)          # keep fp32 for the comparison
            np.savez(path, **st)

    class March(torch.autograd.Function):
        @staticmethod
        def forward(ctx, data, tree, rays):
            tree.o.data = data.detach().numpy().copy()
            ctx.tree, ctx.rays = tree, rays
            return torch.from_numpy(OO.volume_render(tree.o, *rays, step_size=step_size))

        @staticmethod
        def backward(ctx, g):
            grad = OO.volume_render_backward(ctx.tree.o, *ctx.rays, g.numpy().astype(np.float32), step_size=step_size)
            return torch.from_numpy(grad), None, None

    class VolumeRenderer:
        def __init__(self, tree, step_size=1e-3, ndc=None):
            assert ndc is None
            self.tree = tree

        def render_persp(self, c2w, height, width, fx, fast=False, cuda=True):
            assert not fast
            rays = OO.persp_rays(c2w.numpy(), width, height, fx)
            im = March.apply(self.tree.data, self.tree, rays).reshape(height, width, 3)
            last_render[0] = im.detach().numpy().copy()
            return im

    last_render, writes = [None], []
    svox = types.ModuleType("svox")
    svox.N3Tree, svox.VolumeRenderer, svox.NDCConfig = TreeModule, VolumeRenderer, object
    sys.modules["svox"] = svox
    sys.modules["imageio"] = types.SimpleNamespace(
        imwrite=lambda path, im, *a, **k: writes.append((path, np.array(im), last_render[0])))
    _use_reference_octree()
    from octree import optimization as RO
    with tempfile.TemporaryDirectory() as d:
        gts = {}
        for split, ps in poses.items():
            os.makedirs(os.path.join(d, split))
            frames = []
            for i, c2w in enumerate(ps):
                im = OO.volume_render(teacher, *OO.persp_rays(c2w, W, H, focal), step_size=step_size).reshape(H, W, 3)
                rgba = np.concatenate([np.clip(im, 0, 1), np.ones((H, W, 1), np.float32)], axis=-1)
                Image.fromarray((rgba * 255.0 + 0.5).astype(np.uint8), mode="RGBA").save(os.path.join(d, split, f"r_{i}.png"))
                frames.append({"file_path": f"./{split}/r_{i}", "transform_matrix": np.asarray(c2w, dtype=np.float64).tolist()})
            json.dump({"camera_angle_x": focal_angle, "frames": frames}, open(os.path.join(d, f"transforms_{split}.json"), "w"))
        st = student.state()
        st["data"] = student.data[:student.n_internal].astype(np.float32)
        np.savez(os.path.join(d, "tree.npz"), **st)
        open(os.path.join(d, "cfg.yaml"), "w").write("dataset: blender\nfactor: 0\nwhite_bkgd: true\n")
        results = []
        for lr, extra in runs:
            del writes[:]
            RO.FLAGS(["make_golden", "--config", os.path.join(d, "cfg"), "--input", os.path.join(d, "tree.npz"), "--output", os.path.join(d, "tree_opt.npz"),
                      "--data_dir", d, "--dataset", "blender", "--factor", "0", "--white_bkgd", "--num_epochs", "3",
                      "--val_interval", "1", "--sgd", "--lr", str(lr), "--continue_on_decrease", "--renderer_step_size", str(step_size)]
                     + list(extra))
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                RO.main(None)
            log = buf.getvalue()
            out = np.load(os.path.join(d, "tree_opt.npz"))
            results.append(dict(
                lr=lr, data_best=out["data"].astype(np.float32),
                train_psnr=[float(l.split()[-1]) for l in log.splitlines() if l.startswith("** train_psnr")],
                val_psnr=[float(l.split()[3]) for l in log.splitlines() if l.startswith("** val psnr")],
                initial_val_psnr=[float(l.split()[-1]) for l in log.splitlines() if l.startswith("** initial val psnr")][0],
                writes=[(os.path.relpath(p, d), im, r) for p, im, r in writes]))
        ds = {s_: RO.datasets.get_dataset(s_, RO.FLAGS) for s_ in ("train", "val")}
    z = np.load(os.path.join(HERE, "ref_optimization.npz"))       # the same scene as the plain-SGD golden
    assert np.array_equal(z["data0"], student.data[:n].astype(np.float32)) and np.array_equal(z["child"], student.child[:n])
    assert np.array_equal(z["val_gt"], ds["val"].images.astype(np.float32))
    return results

MOMENTUM_RUNS = {"momentum": ["--sgd_momentum", "0.9", "--nosgd_nesterov"],
                 "nesterov": ["--sgd_momentum", "0.9", "--sgd_nesterov"]}
MOMENTUM_LR = 15.0


def gen_ref_optimization_momentum():
    """ref_optimization_momentum.npz: the scene of ref_optimization.npz run twice more, with torch.optim.SGD momentum
    0.9 and with momentum 0.9 + Nesterov, both with --render_interval 1.  Per run <k>: <k>_flags, curves, data_best,
    and the imwrite calls: <k>_vis_names (relative paths), <k>_vis_images (uint8 [gt | render]), <k>_vis_renders (the
    float render each image was made from)."""
    results = run_ref_optimization([(MOMENTUM_LR, MOMENTUM_RUNS[k] + ["--render_interval", "1"])
                                           for k in MOMENTUM_RUNS])
    out = dict(lr=MOMENTUM_LR, momentum=0.9)
    for k, res in zip(MOMENTUM_RUNS, results):
        out.update({f"{k}_flags": np.array(MOMENTUM_RUNS[k]), f"{k}_train_psnr": np.array(res["train_psnr"]),
                    f"{k}_val_psnr": np.array(res["val_psnr"]), f"{k}_initial_val_psnr": res["initial_val_psnr"],
                    f"{k}_data_best": res["data_best"],
                    f"{k}_vis_names": np.array([w[0] for w in res["writes"]]),
                    f"{k}_vis_images": np.stack([w[1] for w in res["writes"]]),
                    f"{k}_vis_renders": np.stack([w[2] for w in res["writes"]]).astype(np.float32)})
        print("ref_optimization_momentum.npz", k, "initial val", res["initial_val_psnr"], "train", res["train_psnr"],
              "val", res["val_psnr"], "images", len(res["writes"]))
    np.savez_compressed(os.path.join(HERE, "ref_optimization_momentum.npz"), **out)


if __name__ == "__main__":
    torch.manual_seed(20200823)
    torch.set_num_threads(8)
    gen_ref_optimization_momentum()

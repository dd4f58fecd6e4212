"""`python -m plenoctree_b200.nerf_sh.gen_mesh` — the reference's `nerf_sh.gen_mesh` CLI (nerf_sh/gen_mesh.py:46-198):
restore the newest checkpoint of train_dir, evaluate the raw density of the fine (or, with --coarse, the coarse)
MLP on a regular grid between corners c1 and c2 (`eval_points_raw`, sigma only, `point_chunk` points per launch),
extract the `iso` surface and write `<train_dir>/mesh.obj`.  Vertex positions follow the reference's scaling
`c1 + index * (c2 - c1) / reso` (gen_mesh.py:126-129).  The surface extractor is nerf/mesh.py (marching tetrahedra;
PyMCubes is not available here)."""
import os

import numpy as np
import torch
from absl import app

from .. import _dist
from ..nerf import checkpoints, flags as F, models
from ..nerf.mesh import marching_tetrahedra, save_obj

FLAGS = F.FLAGS
F.define_flags()
F.define({       # nerf_sh/gen_mesh.py:48-77
    "reso": ("string", "300 300 300", "Marching cube resolution in each dimension: x y z"),
    "c1": ("string", "-2 -2 -2", "Marching cubes bounds lower corner 1 in x y z OR single number"),
    "c2": ("string", "2 2 2", "Marching cubes bounds upper corner in x y z OR single number"),
    "iso": ("float", 6.0, "Marching cubes isosurface"),
    "coarse": ("bool", False, "Force use corase network (else depends on renderer n_fine in conf)"),
    "point_chunk": ("integer", 720720, "Chunk (batch) size of points for evaluation. NOTE: --chunk will be ignored"),
})


def _triple(text, cast):
    vals = [cast(x) for x in str(text).split()]
    if len(vals) == 1:
        vals *= 3
    if len(vals) != 3:
        raise ValueError(f"expected one or three numbers, got {text!r}")
    return vals


def sigma_grid(model, c1, c2, reso, chunk, coarse=False):
    """raw sigma at linspace(c1, c2, reso) per axis ("ij" order), [rx,ry,rz] float32 on the host.  The points of a
    chunk are generated on the device from their flat index; only sigma is written (no 3K colour columns)."""
    dev = model.device
    axes = [torch.linspace(float(lo), float(hi), int(n), dtype=torch.float32, device=dev) for lo, hi, n in zip(c1, c2, reso)]
    total = int(reso[0]) * int(reso[1]) * int(reso[2])
    out = torch.empty(total, dtype=torch.float32, device=dev)
    for i in range(0, total, chunk):
        idx = torch.arange(i, min(total, i + chunk), device=dev)
        pts = torch.stack([axes[0][idx // (reso[1] * reso[2])], axes[1][(idx // reso[2]) % reso[1]],
                           axes[2][idx % reso[2]]], dim=1).contiguous()
        _, sigma = model.eval_points_raw(pts, coarse=coarse, want_rgb=False)
        out[i:i + pts.shape[0]] = sigma[:, 0]
    return out.reshape(*reso).cpu().numpy()


def marching_cubes(model, c1, c2, reso, isosurface, chunk, coarse=False):
    """gen_mesh.marching_cubes (gen_mesh.py:84-131): world-space vertices [V,3] and triangles [F,3] of the
    sigma = isosurface level set."""
    sig = sigma_grid(model, c1, c2, reso, chunk, coarse)
    vertices, triangles = marching_tetrahedra(sig, isosurface)
    c1, c2 = np.array(c1, dtype=np.float64), np.array(c2, dtype=np.float64)
    return vertices * ((c2 - c1) / np.array(reso, dtype=np.float64)) + c1, triangles


def main(unused_argv):
    F.update_flags(FLAGS)
    F.check_flags(FLAGS, require_data=False)
    F.check_scope(FLAGS)
    reso, c1, c2 = _triple(FLAGS.reso, int), _triple(FLAGS.c1, float), _triple(FLAGS.c2, float)
    rank, world, dev = _dist.dist_init()
    model, state = models.get_model_state(FLAGS, device=dev, restore=False, max_rays=1024)
    if checkpoints.restore_checkpoint(FLAGS.train_dir, model, state) is None:
        raise ValueError(f"no checkpoint_* in {FLAGS.train_dir}")
    mesh_path = os.path.join(FLAGS.train_dir, "mesh.obj")
    if rank == 0:          # 27 M points are ~20 ms of one GPU: nothing to shard
        print("* Eval reso", FLAGS.reso, "coarse?", FLAGS.coarse)
        verts, faces = marching_cubes(model, c1, c2, reso, FLAGS.iso, FLAGS.point_chunk,
                                      coarse=FLAGS.coarse)
        print(" Saving to", mesh_path, f"({len(verts)} vertices, {len(faces)} triangles)")
        save_obj(verts, faces, mesh_path)
    _dist.dist_finish()
    return mesh_path


if __name__ == "__main__":
    app.run(main)

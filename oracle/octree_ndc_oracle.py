"""CPU oracle of the NDC ray transform of the PlenOctree path (forward-facing LLFF scenes).  TEST INFRASTRUCTURE ONLY.

Only tests/ and the CPU legs of the bench scripts may import this module.

The reference renders a PlenOctree of a forward-facing scene through `svox.VolumeRenderer(t, ndc=NDCConfig(w, h,
focal))` (octree/optimization.py:170-174, octree/nerf/utils.py:451-457) and builds the extraction mask through the
same options (octree/extraction.py:187-193).  svox is absent from the reference tree; what follows restates its
transform as:

  1. the reference's own `convert_to_ndc` (nerf_sh/nerf/datasets.py:40-60) with near = 1, in float32 and in its
     operation order (the origin is moved onto the plane z = -1, then projected);
  2. the NDC direction normalised for the march;
  3. the view direction left as the normalised WORLD direction, the one the LLFF NeRF-SH model was trained with
     (Rays(ndc_origins, ndc_dirs, world_viewdirs), nerf_sh/nerf/datasets.py:410-425).

Steps 2 and 3 are the two svox-specific assumptions (DESIGN.md §8); the end-to-end test of tests/test_octree_ndc.py
checks them: a tree rendered under them matches the NeRF-SH model's own NDC render, and with NDC view directions or
without the transform it does not.  The march, its backward, the training pass and the grid-weight render are octree_oracle's, fed with these rays.
"""
import numpy as np

from oracle import octree_oracle as OO

f32 = np.float32


def convert_to_ndc(origins, dirs, focal, width, height):
    """nerf_sh/nerf/datasets.py:40-60 at near = 1, float32: -> (NDC origins, un-normalised NDC directions)."""
    o = np.asarray(origins, dtype=f32)
    d = np.asarray(dirs, dtype=f32)
    t = (-(f32(1.0) + o[:, 2]) / d[:, 2]).astype(f32)
    c = (o + (t[:, None] * d).astype(f32)).astype(f32)
    sx = -((f32(2.0) * f32(focal)) / f32(width))
    sy = -((f32(2.0) * f32(focal)) / f32(height))
    cx = (c[:, 0] / c[:, 2]).astype(f32)
    cy = (c[:, 1] / c[:, 2]).astype(f32)
    no = np.stack([sx * cx, sy * cy, f32(1.0) + f32(2.0) / c[:, 2]], axis=1).astype(f32)
    nd = np.stack([sx * ((d[:, 0] / d[:, 2]).astype(f32) - cx), sy * ((d[:, 1] / d[:, 2]).astype(f32) - cy),
                   f32(-2.0) / c[:, 2]], axis=1).astype(f32)
    return no, nd


def ndc_rays(origins, dirs, vdirs, focal, width, height):
    """the rays the octree march takes in NDC mode: (NDC origins, unit NDC directions, vdirs unchanged)."""
    no, nd = convert_to_ndc(origins, dirs, focal, width, height)
    nrm = np.sqrt(nd[:, 0] * nd[:, 0] + nd[:, 1] * nd[:, 1] + nd[:, 2] * nd[:, 2]).astype(f32)
    return no, (nd / nrm[:, None]).astype(f32), np.asarray(vdirs, dtype=f32).copy()


def ndc_persp_rays(c2w, width, height, focal):
    """OO.persp_rays of a camera, then the NDC transform with the camera's own (width, height, focal): the rays of
    render_persp / the training pass / the grid-weight render in NDC mode."""
    o, d, v = OO.persp_rays(c2w, width, height, focal)
    return ndc_rays(o, d, v, focal, width, height)

"""Thin torch-tensor front end over the C ABI (device memory and streams only; no math here)."""
import ctypes

import numpy as np
import torch

from ._lib import (NET_RELU, PREC_FP16, PREC_FP16X3, SIGMA_RELU, SIGMA_SOFTPLUS, check, lib,  # noqa: F401
                   posenc_ref, posenc_struct, ptr, stream_ptr)
from .layouts import K_of

# `posenc` below: the model's point encoder (min_deg_point, max_deg_point, legacy_posenc_order) as a tuple; None is
# the reference default (0, 10, False).  The blob must have been packed with the same encoder.  `net_activation`: the
# trunk activation (_lib.NET_*, flags.net_activation_code); the packed blob does not depend on it.


def _f32c(t, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
        raise ValueError(f"{name} must be a contiguous float32 CUDA tensor")
    return t


def param_count(sh_deg, posenc=None):
    n = lib.pob_param_count_pe(sh_deg, posenc_ref(posenc_struct(posenc)))
    if n < 0:
        raise ValueError("sh_deg must be in [-1, 4] and posenc degrees in 0 <= min_deg <= max_deg <= 10")
    return int(n)


def pack_weights(flat, sh_deg, out=None, posenc=None):
    """flat fp32 parameters of one MLP (reference order) -> packed operand blob (uint8 tensor)."""
    _f32c(flat, "flat")
    if flat.numel() != param_count(sh_deg, posenc):
        raise ValueError(f"expected {param_count(sh_deg, posenc)} parameters, got {flat.numel()}")
    nbytes = int(lib.pob_packed_bytes(sh_deg))
    if out is None:
        out = torch.zeros(nbytes, dtype=torch.uint8, device=flat.device)
    pe = posenc_struct(posenc)
    check(lib.pob_pack_weights_pe(ptr(flat), sh_deg, posenc_ref(pe), ptr(out), stream_ptr()))
    return out


def eval_points_raw(blob, sh_deg, points, want_rgb=True, precision=PREC_FP16, posenc=None, net_activation=NET_RELU):
    """NerfModel.eval_points_raw (nerf_sh/nerf/models.py:143-181): -> (raw_rgb [M,3K] | None, raw_sigma [M,1])."""
    _f32c(points, "points")
    m = points.shape[0]
    K = K_of(sh_deg)
    rgb = torch.empty((m, 3 * K), dtype=torch.float32, device=points.device) if want_rgb else None
    sig = torch.empty((m, 1), dtype=torch.float32, device=points.device)
    pe = posenc_struct(posenc, net_activation)
    check(lib.pob_eval_points_raw_pe(ptr(blob), sh_deg, posenc_ref(pe), ptr(points), m, ptr(rgb), ptr(sig),
                                     precision, stream_ptr()))
    return rgb, sig


def eval_points(blob, sh_deg, points, viewdirs, precision=PREC_FP16, sigma_activation=SIGMA_RELU, posenc=None,
                net_activation=NET_RELU):
    """NerfModel.eval_points (models.py:183-214): -> (rgb [M,3], sigma [M,1]) after sigmoid / the density activation
    (SIGMA_RELU or SIGMA_SOFTPLUS)."""
    _f32c(points, "points")
    if viewdirs is not None:
        _f32c(viewdirs, "viewdirs")
    m = points.shape[0]
    out = torch.empty((m, 4), dtype=torch.float32, device=points.device)
    pe = posenc_struct(posenc, net_activation)
    check(lib.pob_eval_points_pe(ptr(blob), sh_deg, posenc_ref(pe), ptr(points), ptr(viewdirs), m, ptr(out),
                                 int(sigma_activation), precision, stream_ptr()))
    return out[:, :3], out[:, 3:4]


def eval_cells_mean(blob, sh_deg, points, samples_per_cell, precision=PREC_FP16, posenc=None,
                    net_activation=NET_RELU):
    """extraction step 2 (octree/extraction.py:367-394): points [n_cells, S, 3] -> [n_cells, 3K+1] means."""
    _f32c(points, "points")
    pts = points.reshape(-1, 3)
    if pts.shape[0] % samples_per_cell:
        raise ValueError("points must hold samples_per_cell points per cell")
    n_cells = pts.shape[0] // samples_per_cell
    out = torch.empty((n_cells, 3 * K_of(sh_deg) + 1), dtype=torch.float32, device=points.device)
    pe = posenc_struct(posenc, net_activation)
    check(lib.pob_eval_cells_mean_pe(ptr(blob), sh_deg, posenc_ref(pe), ptr(pts), n_cells, samples_per_cell, ptr(out),
                                     precision, stream_ptr()))
    return out


def eval_grid(blob, sh_deg, reso, offset, scale, x0=0, nx=None, ny=None, nz=None, want_rgb=False,
              precision=PREC_FP16, device="cuda", posenc=None, net_activation=NET_RELU):
    """Dense-grid sweep of octree.extraction (octree/extraction.py:244-320) for one x-slab."""
    nx = reso - x0 if nx is None else nx
    ny = reso if ny is None else ny
    nz = reso if nz is None else nz
    m = nx * ny * nz
    K = K_of(sh_deg)
    rgb = torch.empty((m, 3 * K), dtype=torch.float32, device=device) if want_rgb else None
    sig = torch.empty((m,), dtype=torch.float32, device=device)
    off = (ctypes.c_float * 3)(*[float(v) for v in offset])
    sc = (ctypes.c_float * 3)(*[float(v) for v in scale])
    pe = posenc_struct(posenc, net_activation)
    check(lib.pob_eval_grid_pe(ptr(blob), sh_deg, posenc_ref(pe), reso, x0, nx, ny, nz, off, sc, ptr(rgb), ptr(sig),
                               precision, stream_ptr()))
    return rgb, sig


def grid_slab(reso, rank, world):
    """x-slab [x0, x0+nx) of the extraction grid owned by `rank` (voxel slabs, no collective)."""
    base, rem = divmod(reso, world)
    x0 = rank * base + min(rank, rem)
    return x0, base + (1 if rank < rem else 0)

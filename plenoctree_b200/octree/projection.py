"""Vanilla NeRF (use_viewdirs) -> PlenOctree: the SH projection of octree.extraction step2 (octree/extraction.py:
217-241,362-394, octree/nerf/sh_proj.py:273-306) on the device.

The reference evaluates the view branch for every (sample point, direction) pair.  Here the branch is split at the
condition layer (include/plenoctree_b200.h, pob_sh_proj_*):

  point stage      pob_sh_proj_points runs the trunk once, on the tensor-core forward of a plain-RGB (sh_deg -1)
                   blob of the trunk and Dense_8 with zero rgb columns (the blob auto_scale / step1 sweep): raw sigma,
                   and h7 kept as fp16, from which a_p = W10_b (W9 h7 + b9) + b10 is one 256 x 128 fp32 GEMM.
                   Dense_9 has no activation, so its composition with W10_b is formed once on the host in fp64 and
                   rounded once to fp32.
  direction stage  pob_sh_proj_directions draws one direction set per block of `cells_per_block` leaves and tabulates
                   t_d = W10_e posenc(d) and Y_k(d); pob_sh_proj_cells forms relu(a_p + t_d), the rgb layer and
                   the projection in fp32 and writes the leaf rows [3K coefficients, raw sigma].

A block's directions depend only on (seed, block index), so the tree does not depend on how the leaf blocks are split
over launches or ranks.
"""
import numpy as np
import torch

from .._lib import NET_RELU, PREC_FP16, check, lib, posenc_ref, posenc_struct, ptr, stream_ptr
from .. import ops

PROJ_SEED = 20200823
CELLS_PER_BLOCK = 1024          # leaves sharing one direction set
TABLE_BUDGET = 256 << 20        # bytes of direction tables per launch
POINTS_PER_LAUNCH = 1 << 18     # sample points per point-stage launch (4.4 KB of workspace and 512 B of a_p each)


class VanillaNerf:
    """The parts of a vanilla NeRF MLP (MLP_1 when there is a fine level, as eval_points_raw picks it) that
    extraction needs, on the device.  It stands where NerfModel stands for auto_scale / step1 (`_blob`, `sh_deg`,
    `posenc`, `net_act_code`, `precision`, `device`: the sigma blob, plain RGB) and adds the projection inputs."""

    def __init__(self, mlps, posenc=(0, 10, False), deg_view=4, num_fine_samples=128, device="cuda",
                 precision=PREC_FP16):
        self.posenc = tuple(posenc)
        self.deg_view = int(deg_view)
        self.device = torch.device(device)
        self.precision = precision
        self.net_act_code = NET_RELU
        self.sh_deg = -1            # format of the sigma blob (plain RGB head, zero rgb columns)
        if num_fine_samples > 0 and "MLP_1" not in mlps:
            raise ValueError("num_fine_samples > 0 but the checkpoint has no MLP_1 (eval_points_raw evaluates the fine "
                             "MLP of a model with a fine level)")
        layers = mlps["MLP_1"] if num_fine_samples > 0 else mlps["MLP_0"]
        trunk = [np.asarray(a, dtype=np.float32) for k, b in layers[:9] for a in (k, b)]
        k9, b9 = (np.asarray(a, dtype=np.float64) for a in layers[9])
        k10, b10 = (np.asarray(a, dtype=np.float64) for a in layers[10])
        k11, b11 = layers[11]
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(self.device)
        self.head_w = dev(k9 @ k10[:256])                   # [256, 128]
        self.head_b = dev(b9 @ k10[:256] + b10)             # [128]
        flat = np.concatenate([a.reshape(-1) for a in trunk] + [np.zeros(256 * 3 + 3, np.float32)])
        self.sigma_blob = ops.pack_weights(torch.from_numpy(flat).to(self.device), -1, posenc=self.posenc)
        self.w10e = dev(np.asarray(layers[10][0], dtype=np.float32)[256:])   # [3 + 6 deg_view, 128]
        self.w11, self.b11 = dev(k11), dev(b11)
        self._ws = None
        self._pe = posenc_struct(self.posenc)

    def _blob(self, coarse=False):
        return self.sigma_blob

    def point_stage(self, points):
        """(a_p [M, 128], raw sigma [M]) of points [M, 3], POINTS_PER_LAUNCH points per trunk pass."""
        m = points.shape[0]
        a = torch.empty((m, 128), dtype=torch.float32, device=self.device)
        sigma = torch.empty(m, dtype=torch.float32, device=self.device)
        if self._ws is None:
            n = int(lib.pob_sh_proj_points_workspace_bytes(min(m, POINTS_PER_LAUNCH)))
            self._ws = torch.empty(n, dtype=torch.uint8, device=self.device)
        for i in range(0, m, POINTS_PER_LAUNCH):
            j = min(m, i + POINTS_PER_LAUNCH)
            if int(lib.pob_sh_proj_points_workspace_bytes(j - i)) > self._ws.numel():
                self._ws = torch.empty(int(lib.pob_sh_proj_points_workspace_bytes(j - i)), dtype=torch.uint8,
                                       device=self.device)
            check(lib.pob_sh_proj_points(ptr(self.sigma_blob), posenc_ref(self._pe), ptr(points[i:j]), j - i,
                                         ptr(self.head_w), ptr(self.head_b), ptr(self._ws), ptr(a[i:j]),
                                         ptr(sigma[i:j]), stream_ptr()))
        return a, sigma


def directions(nerf, sh_deg, n_dirs, block0, n_blocks, seed=PROJ_SEED):
    """pob_sh_proj_directions: (dirs [n_blocks, D, 3], t [n_blocks, 128, D], basis [n_blocks, D, K])."""
    K = (sh_deg + 1) ** 2
    dev = nerf.device
    dirs = torch.empty((n_blocks, n_dirs, 3), dtype=torch.float32, device=dev)
    t = torch.empty((n_blocks, 128, n_dirs), dtype=torch.float32, device=dev)
    basis = torch.empty((n_blocks, n_dirs, K), dtype=torch.float32, device=dev)
    check(lib.pob_sh_proj_directions(int(seed), int(block0), int(n_blocks), int(n_dirs), nerf.deg_view,
                                     int(bool(nerf.posenc[2])), int(sh_deg), ptr(nerf.w10e),
                                     ptr(dirs), ptr(t), ptr(basis), stream_ptr()))
    return dirs, t, basis


def project_cells(nerf, a, sigma, samples_per_cell, sh_deg, tables, cells_per_block=CELLS_PER_BLOCK, out=None):
    """pob_sh_proj_cells: leaf rows [n_cells, 3K + 1] from a_p [n_cells * S, 128], raw sigma [n_cells * S] and the
    direction tables of directions() (cell i uses table block i // cells_per_block)."""
    _, t, basis = tables
    S = int(samples_per_cell)
    n_cells = a.shape[0] // S
    K = (sh_deg + 1) ** 2
    if out is None:
        out = torch.empty((n_cells, 3 * K + 1), dtype=torch.float32, device=a.device)
    check(lib.pob_sh_proj_cells(n_cells, S, int(cells_per_block), ptr(a), ptr(sigma), int(t.shape[2]), int(sh_deg),
                                ptr(t), ptr(basis), ptr(nerf.w11), ptr(nerf.b11), ptr(out), stream_ptr()))
    return out


def blocks_per_launch(samples_per_cell, n_dirs, sh_deg, cells_per_block=CELLS_PER_BLOCK):
    """leaf blocks of one projection launch: at most POINTS_PER_LAUNCH points and TABLE_BUDGET bytes of tables."""
    table = n_dirs * (128 + 3 + (sh_deg + 1) ** 2) * 4
    by_points = POINTS_PER_LAUNCH // (cells_per_block * int(samples_per_cell))
    return max(1, min(by_points, TABLE_BUDGET // table))


def project_leaves(nerf, sh_deg, n_dirs, points, samples_per_cell, block0, seed=PROJ_SEED,
                   cells_per_block=CELLS_PER_BLOCK):
    """leaf rows of the cells whose sample points are `points` [n_cells, S, 3], the first cell being cell
    block0 * cells_per_block of the tree's leaf order (so that it takes that block's directions)."""
    pts = points.reshape(-1, 3).contiguous()
    S = int(samples_per_cell)
    n_cells = pts.shape[0] // S
    n_blocks = (n_cells + cells_per_block - 1) // cells_per_block
    tables = directions(nerf, sh_deg, n_dirs, block0, n_blocks, seed)
    a, sig = nerf.point_stage(pts)
    return project_cells(nerf, a, sig, S, sh_deg, tables, cells_per_block)

"""Median-cut palette quantisation and tree compression on the device (csrc/quantize.cu: pob_quantize_median_cut).

    host (octree/compression.py)                 here
    median_cut(points, bits, weights)            median_cut(points, bits, weights): the same arrays, byte for byte
    (one basis function at a time)               median_cut_batch(points [nb, n, 3], ...): every basis function of
                                                 a tree in one launch sequence
    compress_tree(z, ...)                        compress_tree(z, ...) = compression.compress_tree(z, ..., device="cuda")

The host functions stay the definition; this module reproduces them exactly (see quantize.cu for how: the host's
(key, index) order by a stable radix sort, np.add.reduceat's pairwise order and np.cumsum's sequential fp64 sum).
The weights of the weighted cut, 1 - exp(-0.01 sigma), are computed by numpy as on the host, since the device's exp
need not round like the host's.  Deflate (np.savez_compressed) stays on the host.
"""
import numpy as np
import torch

from .._lib import check, lib, ptr, stream_ptr

MAX_BITS = 16


def median_cut_batch(points, bits, weights=None):
    """points [nb, n, 3] (numpy or torch; copied to cuda fp32), bits in 0..16, weights [n] (fp64, shared by every set)
    or None -> (palette [nb, 2^bits, 3] fp32 cuda tensor, map [nb, n] int16 cuda tensor holding the uint16 box ids)."""
    pts = torch.as_tensor(points).to(device="cuda", dtype=torch.float32).contiguous()
    if pts.dim() != 3 or pts.shape[2] != 3:
        raise ValueError(f"points must be [n_basis, n, 3], got {tuple(pts.shape)}")
    nb, n = int(pts.shape[0]), int(pts.shape[1])
    w = None
    if weights is not None and len(weights) > 0:
        w = torch.as_tensor(np.asarray(weights, dtype=np.float64)).to("cuda").contiguous()
        if w.shape != (n,):
            raise ValueError(f"weights must be [{n}], got {tuple(w.shape)}")
    ws_bytes = lib.pob_quantize_workspace_bytes(nb, n, int(w is not None))
    if ws_bytes < 0:
        raise ValueError(f"{nb} point sets of {n} points are beyond the quantiser's index range")
    palette = torch.empty((nb, 1 << max(0, min(int(bits), MAX_BITS)), 3), dtype=torch.float32, device="cuda")
    index = torch.empty((nb, n), dtype=torch.int16, device="cuda")
    ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device="cuda")
    check(lib.pob_quantize_median_cut(ptr(pts), ptr(w), nb, n, int(bits), ptr(palette), ptr(index), ptr(ws), ws_bytes,
                                      stream_ptr()))
    return palette, index


def median_cut(points, bits, weights=None):
    """compression.median_cut on the device: points [n, 3] -> (palette [2^bits, 3] float32, index [n] int64)."""
    if not 0 <= bits <= MAX_BITS:
        raise ValueError("bits must be in 0..16 (the device map is uint16)")
    palette, index = median_cut_batch(np.asarray(points, dtype=np.float32)[None], bits, weights)
    return palette[0].cpu().numpy(), index[0].cpu().numpy().view(np.uint16).astype(np.int64)


def compress_tree(z, bits=16, sigma_thresh=2.0, retain=0, weighted=False, quantize=True):
    """compression.compress_tree with the threshold, keep mask, palettes, map scatter and data_retained on the GPU."""
    out = {k: v for k, v in z.items() if k not in ("parent_depth", "geom_resize_fact", "n_free", "n_internal", "depth_limit")}
    if not quantize:
        return out
    if not 0 < bits <= MAX_BITS:
        raise ValueError("bits must be in 1..16 (the map is stored as uint16)")
    data = torch.from_numpy(np.ascontiguousarray(out.pop("data"))).to("cuda")
    N = data.shape[1]
    sigma = data[..., -1].to(torch.float32).reshape(-1).clone()
    keep = sigma > torch.tensor(np.float32(sigma_thresh), device="cuda")      # numpy compares in float32 too
    sigma[~keep] = 0.0
    basis_dim = (data.shape[-1] - 1) // 3
    coeffs = data[..., :-1].reshape(-1, 3, basis_dim).to(torch.float32)[keep]                     # [kept, 3, basis]
    weights = None
    if weighted:
        weights = 1.0 - np.exp(-0.01 * sigma[keep].cpu().numpy().astype(np.float64))
    L = keep.shape[0]
    if retain < basis_dim:
        palette, index = median_cut_batch(coeffs[:, :, retain:].permute(2, 0, 1), bits, weights)
        full = torch.zeros((basis_dim - retain, L), dtype=torch.int16, device="cuda")
        full[:, keep] = index
        # fp32 -> fp16 on the host: numpy's rounding and NaN encoding, like the host's palette.astype(np.float16)
        out["quant_colors"] = palette.cpu().numpy().astype(np.float16)
        out["quant_map"] = full.cpu().numpy().view(np.uint16).reshape(-1, L // N ** 3, N, N, N)
    else:   # np.stack of no palettes: the host raises the same error
        np.stack([], axis=0)
    out["sigma"] = sigma.cpu().numpy().reshape(-1, N, N, N)
    if retain:
        kept = torch.zeros((retain, L, 3), dtype=torch.float32, device="cuda")
        kept[:, keep] = coeffs[:, :, :retain].permute(2, 0, 1)
        out["data_retained"] = kept.cpu().numpy().astype(np.float16).reshape(retain, -1, N, N, N, 3)
    return out


def device_available():
    """True when the CUDA library loaded (importing this module) and torch sees a GPU the library can run on."""
    return torch.cuda.is_available() and lib.pob_sm_count() > 0

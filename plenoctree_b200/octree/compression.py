"""`python -m plenoctree_b200.octree.compression x.npz [y.npz ...]` — the reference's octree compressor for
in-browser viewing (octree/compression.py:39-145): voxels with sigma <= sigma_thresh are zeroed, the RGB triple of
every SH basis function is vector-quantised to a 2^bits-entry palette by median cut, and the tree is re-saved with
`quant_colors [basis_dim, 2^bits, 3] f16`, `quant_map [basis_dim, n_nodes, N, N, N] u16`, `sigma [n_nodes, N, N, N]`
(optionally `data_retained` for the first --retain basis functions) instead of `data`, deflate-compressed, without
the bookkeeping keys the viewer does not read (parent_depth, geom_resize_fact, n_free, n_internal, depth_limit).

The reference calls svox's C++ `quantize_median_cut` (third-party, not vendored, not installable here: **parity
unpinned**).  The median cut below is the textbook one in its balanced form: `bits` rounds, every round splits
every box at the (weighted) median of its longest axis, palette entry = (weighted) mean of the box; all boxes of a
round are processed together with segment reductions, so a round is a few passes over the points.
The numpy code below is the definition.  `compress_tree(..., device="cuda")` and the CLI's `--device` (default
`auto`: the GPU when the CUDA library loads and a GPU is visible) run the same computation on the device
(octree/quantize.py, csrc/quantize.cu), with byte-identical output; this module imports without the library.
"""
import argparse
import os

import numpy as np


def median_cut(points, bits, weights=None):
    """points [n,3] float, bits >= 0 -> (palette [2^bits,3] float32, index [n] int64 into the palette).
    Boxes that cannot be split further (one point, or all points equal) leave their sibling entry empty (zeros)."""
    pts = np.ascontiguousarray(points, dtype=np.float32)
    n = pts.shape[0]
    n_colors = 1 << bits
    if n == 0:
        return np.zeros((n_colors, 3), np.float32), np.zeros((0,), np.int64)
    w = None if weights is None or len(weights) == 0 else np.asarray(weights, dtype=np.float64)
    box = np.zeros(n, dtype=np.int64)
    for _ in range(bits):
        order = np.argsort(box, kind="stable")
        sb = box[order]
        starts = np.flatnonzero(np.r_[True, sb[1:] != sb[:-1]])
        ids = sb[starts]
        sp = pts[order]
        ext = np.maximum.reduceat(sp, starts, axis=0) - np.minimum.reduceat(sp, starts, axis=0)     # [boxes,3]
        axis_of_box = np.argmax(ext, axis=1)
        seg = np.repeat(np.arange(len(starts)), np.diff(np.r_[starts, n]))                           # segment of each sorted point
        key = sp[np.arange(n), axis_of_box[seg]]
        inner = np.lexsort((key, seg))                                                               # by box, then coordinate
        order, key = order[inner], key[inner]
        if w is None:
            rank = np.arange(n) - starts[seg]
            size = np.diff(np.r_[starts, n])[seg]
            upper = rank >= (size + 1) // 2                                                          # lower half keeps the median
        else:
            ws = w[order]
            cum = np.cumsum(ws)
            base = np.r_[0.0, cum[starts[1:] - 1]][seg]
            total = np.add.reduceat(ws, starts)[seg]
            upper = (cum - base) > 0.5 * total
            upper &= (np.arange(n) - starts[seg]) > 0                                                # never empty the lower box
        splittable = (ext[np.arange(len(starts)), axis_of_box] > 0)[seg]
        new_box = 2 * ids[seg] + (upper & splittable)
        box = np.empty(n, dtype=np.int64)
        box[order] = new_box
    palette = np.zeros((n_colors, 3), dtype=np.float64)
    if w is None:
        cnt = np.bincount(box, minlength=n_colors).astype(np.float64)
        for c in range(3):
            palette[:, c] = np.bincount(box, weights=pts[:, c], minlength=n_colors)
    else:
        cnt = np.bincount(box, weights=w, minlength=n_colors)
        for c in range(3):
            palette[:, c] = np.bincount(box, weights=pts[:, c] * w, minlength=n_colors)
    palette /= np.maximum(cnt, 1e-30)[:, None]
    palette[cnt == 0] = 0.0
    return palette.astype(np.float32), box


def compress_tree(z, bits=16, sigma_thresh=2.0, retain=0, weighted=False, quantize=True, device=None):
    """z: dict of a tree.npz -> dict of the compressed file (compression.py:80-139).  device None / "cpu": numpy;
    "cuda": octree.quantize.compress_tree, which returns identical arrays."""
    if device not in (None, "cpu"):
        if device != "cuda":
            raise ValueError(f"device must be None, 'cpu' or 'cuda', got {device!r}")
        from . import quantize as Q
        return Q.compress_tree(z, bits, sigma_thresh, retain, weighted, quantize)
    out = {k: v for k, v in z.items() if k not in ("parent_depth", "geom_resize_fact", "n_free", "n_internal", "depth_limit")}
    if not quantize:
        return out
    if not 0 < bits <= 16:
        raise ValueError("bits must be in 1..16 (the map is stored as uint16)")
    data = np.asarray(out.pop("data"))
    N = data.shape[1]
    sigma = data[..., -1].astype(np.float32).reshape(-1).copy()
    keep = sigma > sigma_thresh
    sigma[~keep] = 0.0
    basis_dim = (data.shape[-1] - 1) // 3
    coeffs = data[..., :-1].reshape(-1, 3, basis_dim).astype(np.float32)[keep]                      # [kept, 3, basis]
    weights = 1.0 - np.exp(-0.01 * sigma[keep].astype(np.float64)) if weighted else None
    colors, maps = [], []
    for i in range(retain, basis_dim):
        palette, index = median_cut(coeffs[:, :, i], bits, weights)
        full = np.zeros(keep.shape[0], dtype=np.uint16)
        full[keep] = index.astype(np.uint16)
        colors.append(palette.astype(np.float16))
        maps.append(full.reshape(-1, N, N, N))
    out["quant_colors"] = np.stack(colors, axis=0)
    out["quant_map"] = np.stack(maps, axis=0)
    out["sigma"] = sigma.reshape(-1, N, N, N)
    if retain:
        kept = np.zeros((retain, keep.shape[0], 3), dtype=np.float16)
        for i in range(retain):
            kept[i, keep] = coeffs[:, :, i]
        out["data_retained"] = kept.reshape(retain, -1, N, N, N, 3)
    return out


def decompress_data(c):
    """inverse of compress_tree up to quantisation: [n_nodes, N, N, N, 3*basis+1] float32 (what a viewer rebuilds)."""
    sigma = np.asarray(c["sigma"], dtype=np.float32)
    retained = np.asarray(c["data_retained"], dtype=np.float32) if "data_retained" in c else None
    retain = 0 if retained is None else retained.shape[0]
    basis_dim = retain + c["quant_colors"].shape[0]
    rgb = np.zeros(sigma.shape + (3, basis_dim), dtype=np.float32)
    for i in range(retain):
        rgb[..., i] = retained[i]
    for j in range(c["quant_colors"].shape[0]):
        rgb[..., retain + j] = np.asarray(c["quant_colors"][j], dtype=np.float32)[np.asarray(c["quant_map"][j], dtype=np.int64)]
    rgb[sigma == 0.0] = 0.0
    return np.concatenate([rgb.reshape(sigma.shape + (3 * basis_dim,)), sigma[..., None]], axis=-1)


def resolve_device(device):
    """--device auto | cpu | cuda -> "cpu" or "cuda".  auto: cuda when the CUDA library loads and a GPU it runs on is
    visible, else cpu; cuda: an error when it cannot run."""
    if device == "cpu":
        return "cpu"
    if device not in ("auto", "cuda"):
        raise ValueError(f"--device must be auto, cpu or cuda, got {device!r}")
    try:
        from . import quantize as Q
    except (ImportError, OSError) as e:
        if device == "cuda":
            raise RuntimeError(f"--device cuda: the CUDA library does not load ({e})") from e
        return "cpu"
    if Q.device_available():
        return "cuda"
    if device == "cuda":
        raise RuntimeError("--device cuda: no CUDA GPU the library can run on (sm_90) is visible")
    return "cpu"


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("input", type=str, nargs="+", help="Input npz(s)")
    ap.add_argument("--noquant", action="store_true", help="Disable quantization")
    ap.add_argument("--bits", type=int, default=16, help="Quantization bits (order)")
    ap.add_argument("--out_dir", type=str, default="min_alt", help="Where to write compressed npz")
    ap.add_argument("--overwrite", action="store_true", help="Overwrite existing compressed npz")
    ap.add_argument("--weighted", action="store_true", help="Use weighted median cut")
    ap.add_argument("--sigma_thresh", type=float, default=2.0, help="Kill voxels under this sigma")
    ap.add_argument("--retain", type=int, default=0, help="Do not compress first x SH coeffs")
    ap.add_argument("--device", choices=("auto", "cpu", "cuda"), default="auto",
                    help="Where to quantise: auto uses the GPU when the CUDA library and a GPU are available")
    args = ap.parse_args(argv)
    device = resolve_device(args.device)
    os.makedirs(args.out_dir, exist_ok=True)
    print("Quantization disabled, only applying deflate" if args.noquant else "Quantization enabled")
    for fname in args.input:
        fname_c = os.path.join(args.out_dir, os.path.basename(fname))
        print("Compressing", fname, "to", fname_c)
        if not args.overwrite and os.path.exists(fname_c):
            print(" > skip")
            continue
        z = dict(np.load(fname))
        if not args.noquant and "quant_colors" in z:
            print(" > skip since source already compressed")
            continue
        out = compress_tree(z, args.bits, args.sigma_thresh, args.retain, args.weighted, quantize=not args.noquant,
                            device=device)
        np.savez_compressed(fname_c, **out)
        print(" > Size", os.path.getsize(fname) // (1024 * 1024), "MB ->", os.path.getsize(fname_c) // (1024 * 1024), "MB")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())

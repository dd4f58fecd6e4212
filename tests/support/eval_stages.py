"""The inference forwards (render, points, grid sweep, cell means) against the training forward and fp64."""
import numpy as np
import torch

from plenoctree_b200 import layouts as L
from tests.support.mlp_stages import U24


TOL_FP16_ANY = 3e-3


# ---- bars (measured on an H100 80 GB HBM3 at a 400 W power limit; the largest value over all cases of test_eval_stages.py in
# brackets)
# fp16x3 against fp64: error of every OUT_RAW / OUT_SIGMA value in units of 2^-24 * sum_k |h_7,k w_k| of the heads GEMM
# (points 33.9, grid 28.1, render 31.1; relative to the largest magnitude: sigma 4.6e-6, rgb 3.6e-6)
X3_ALLOW = 68.0             # [33.9]


CANARY = 0x7FBADBAD         # a NaN bit pattern behind every output of the direct C-ABI calls
M_RAGGED = (1, 63, 64, 65, 127, 128, 129, 255, 257, 513)


CHUNK = 1 << 17             # rows per fp64 reference chunk


def _nbits(a, b):
    """number of 32-bit words that differ between two float32 tensors of the same shape"""
    assert a.shape == b.shape, (a.shape, b.shape)
    return int((a.contiguous().view(torch.int32) != b.contiguous().view(torch.int32)).sum())


def _canary(n, tail=4096):
    return torch.full((n + tail,), CANARY, dtype=torch.int32, device="cuda")


def _tail_ok(buf, n):
    return bool((buf[n:] == CANARY).all())


def _raw(blob, sh, pts, prec, want_rgb=True, pe=None, act=0):
    """pob_eval_points_raw -> (raw_rgb [m, 3K] reference channel-major | None, raw_sigma [m]); pe (encoder) or act
    (trunk activation, _lib.NET_*) away from the default: pob_eval_points_raw_pe with that descriptor"""
    from plenoctree_b200._lib import check, lib, posenc_ref, posenc_struct, ptr, stream_ptr
    m, C3 = pts.shape[0], 3 * L.K_of(sh)
    rb = _canary(m * C3) if want_rgb else None
    sb = _canary(m)
    d = posenc_struct(pe, act)
    if d is None:
        check(lib.pob_eval_points_raw(ptr(blob), sh, ptr(pts), m, ptr(rb), ptr(sb), prec, stream_ptr()))
    else:
        check(lib.pob_eval_points_raw_pe(ptr(blob), sh, posenc_ref(d), ptr(pts), m, ptr(rb), ptr(sb), prec,
                                         stream_ptr()))
    torch.cuda.synchronize()
    assert _tail_ok(sb, m) and (rb is None or _tail_ok(rb, m * C3)), ("write past the output", m)
    return (rb[:m * C3].view(torch.float32).view(m, C3) if want_rgb else None), sb[:m].view(torch.float32)


def _rgbs(blob, sh, pts, vd, prec):
    """pob_eval_points -> rgbs [m, 4] (sigmoid rgb, relu sigma)"""
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    m = pts.shape[0]
    ob = _canary(4 * m)
    check(lib.pob_eval_points(ptr(blob), sh, ptr(pts), ptr(vd), m, ptr(ob), prec, stream_ptr()))
    torch.cuda.synchronize()
    assert _tail_ok(ob, 4 * m), ("write past the output", m)
    return ob[:4 * m].view(torch.float32).view(m, 4)


def _grid(blob, sh, reso, off, sc, x0, nx, ny, nz, prec, want_rgb):
    import ctypes
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    m, C3 = nx * ny * nz, 3 * L.K_of(sh)
    rb = _canary(m * C3) if want_rgb else None
    sb = _canary(m)
    check(lib.pob_eval_grid(ptr(blob), sh, reso, x0, nx, ny, nz, (ctypes.c_float * 3)(*off),
                            (ctypes.c_float * 3)(*sc), ptr(rb), ptr(sb), prec, stream_ptr()))
    torch.cuda.synchronize()
    assert _tail_ok(sb, m) and (rb is None or _tail_ok(rb, m * C3)), ("write past the output", m)
    return (rb[:m * C3].view(torch.float32).view(m, C3) if want_rgb else None), sb[:m].view(torch.float32)


def _cells(blob, sh, pts, n_cells, S, prec, pe=None, act=0):
    from plenoctree_b200._lib import check, lib, posenc_ref, posenc_struct, ptr, stream_ptr
    W = 3 * L.K_of(sh) + 1
    ob = _canary(n_cells * W)
    d = posenc_struct(pe, act)
    if d is None:
        check(lib.pob_eval_cells_mean(ptr(blob), sh, ptr(pts), n_cells, S, ptr(ob), prec, stream_ptr()))
    else:
        check(lib.pob_eval_cells_mean_pe(ptr(blob), sh, posenc_ref(d), ptr(pts), n_cells, S, ptr(ob), prec,
                                         stream_ptr()))
    torch.cuda.synchronize()
    assert _tail_ok(ob, n_cells * W), ("write past the output", n_cells, S)
    return ob[:n_cells * W].view(torch.float32).view(n_cells, W)


def _blob(flat, sh):
    from plenoctree_b200 import ops
    return ops.pack_weights(torch.as_tensor(flat, dtype=torch.float32).cuda().contiguous(), sh)


def _heads_params(flat, K, dev, enc_width=L.ENC_DIM):
    """packed heads weight [256, NH] and bias [NH] (fp32) on dev, and the channel-major index of the 3K rgb columns"""
    Wh, bh = L.heads_matrix(np.asarray(flat, np.float32), K, enc_width)
    cols9 = torch.tensor([L.heads_column(K, o) for o in range(3 * K)], device=dev)
    return torch.from_numpy(Wh).to(dev), torch.from_numpy(bh).to(dev), cols9


def _raw_of_heads(heads, cols9):
    """packed heads [n, NH] -> (raw_rgb channel-major [n, 3K], raw_sigma [n])"""
    return heads[:, cols9], heads[:, 0]


def _hilo(w):
    """fp32 -> (hi, lo) fp64, the split layouts.pack_reference (and pack.cu) applies to every weight and bias"""
    hi = w.half()
    lo = (w - hi.float()).half()
    return hi.double(), lo.double()


class X3Ref:
    """fp64 evaluation of one MLP with the operands the fp16x3 forward represents: weights and biases hi + lo,
    posenc of encoder pe from the fp32 arguments (x * 2^j exact, + fp32(pi/2) as an fp32 add, fp64 sine), the trunk
    activation act in fp64 (relu exact)."""

    def __init__(self, flat, sh, dev, pe=None, act="relu"):
        from oracle import posenc_oracle as PO
        from oracle import net_activation_oracle as NA
        self.pe = PO.DEFAULT if pe is None else tuple(pe)
        self.act = NA.activation(act)
        W = PO.width(self.pe)
        K = self.K = L.K_of(sh)
        w_off, b_off, _ = L.flat_offsets(K, W)
        dims = L.layer_dims(K, W)
        fl = torch.as_tensor(np.asarray(flat, np.float32)).to(dev)
        self.Whi, self.W, self.B = [], [], []
        for l in range(8):
            hi, lo = _hilo(fl[w_off[l]:w_off[l] + dims[l][0] * 256].view(dims[l][0], 256))
            self.Whi.append(hi)
            self.W.append(hi + lo)
            bhi, blo = _hilo(fl[b_off[l]:b_off[l] + 256])
            self.B.append(bhi + blo)
        Wh, bh, self.cols9 = _heads_params(flat, K, dev, W)
        hi, lo = _hilo(Wh)
        self.Wh_hi, self.Wh = hi, hi + lo
        hi, lo = _hilo(bh)
        self.bh_hi, self.bh = hi, hi + lo

    def __call__(self, x, pert=None):
        """x fp32 [n, 3] -> (packed heads [n, NH], sum |h_7 w| + |b| [n, NH]) in fp64.  pert: one term of the error
        compensation left out (sensitivity guard)."""
        from tests.support.model_flags import _ref_features
        e = torch.cat([x.double(), _ref_features(x, self.pe)], 1)
        if pert == "posenc_unit_lo_dropped":        # one 8-column unit of the posenc tile, hi part only
            e = e.clone()
            e[:, 16:24] = e[:, 16:24].half().double()
        h = h4 = None
        for l in range(8):
            a = e if l == 0 else (torch.cat([h4, e], 1) if l == 5 else h)
            W = self.W[l]
            if pert == "weight_slot_lo_dropped" and l == 6:   # K-slot 2 of layer 6: hi part of the weights only
                W = W.clone()
                W[64:96] = self.Whi[6][64:96]
            pre = a @ W + self.B[l]
            if pert == "trunk_slot_hi_hi" and l == 3:          # K-slot 5 of layer 3 evaluated hi * hi only
                s = slice(160, 192)
                pre = pre - a[:, s] @ W[s] + a[:, s].half().double() @ self.Whi[3][s]
            h = self.act(pre)
            if l == 4:
                h4 = h
        if pert == "heads_single_pass":
            heads = h.half().double() @ self.Wh_hi + self.bh_hi
        else:
            heads = h @ self.Wh + (self.bh_hi if pert == "heads_bias_hi_only" else self.bh)
        return heads, h.abs() @ self.Wh.abs() + self.bh.abs()


def _x3_errors(ref, x, raw_rgb, raw_sig, st, key):
    """fp16x3 OUT_RAW values against the fp64 reference, chunked: running maxima of the error in units of
    2^-24 * sum |h_7 w| and of |err| / max |ref| per output, under `key`."""
    for r0 in range(0, x.shape[0], CHUNK):
        r1 = min(x.shape[0], r0 + CHUNK)
        heads, mag = ref(x[r0:r1])
        rr, rs = _raw_of_heads(heads, ref.cols9)
        mr, ms = _raw_of_heads(mag, ref.cols9)
        er = (raw_rgb[r0:r1].double() - rr).abs()
        es = (raw_sig[r0:r1].double() - rs).abs()
        st.max(f"{key}_excess", max(float((er / (U24 * mr)).max()), float((es / (U24 * ms)).max())))
        st.max(f"{key}_abs_rgb", er.max())
        st.max(f"{key}_abs_sigma", es.max())
        st.max(f"{key}_refmax_rgb", rr.abs().max())
        st.max(f"{key}_refmax_sigma", rs.abs().max())


def _level_rows(ctx, lv, z, sp, dev):
    """fp32 point (separate multiply and add, as cast_rays) and view direction of every row of one level; free
    (sparsity) rows use their own points and ray 0's direction, as the kernel does"""
    o, d, v = (torch.from_numpy(a).to(dev) for a in ctx["rays"])
    N, Mr, M = lv["N"], lv["M_rays"], lv["M"]
    s = torch.arange(M, device=dev)
    ray = (s // N).clamp_max(ctx["n"] - 1)
    x = o[ray] + z.reshape(-1)[s.clamp_max(Mr - 1)][:, None] * d[ray]
    if M > Mr:
        x = torch.where((s >= Mr)[:, None], sp[(s - Mr).clamp_min(0)], x)
    vd = v[torch.where(s < Mr, ray, torch.zeros_like(ray))]
    return x.contiguous(), vd.contiguous()


def _cell_bound(S):
    """the standard summation bound of the kernel's mean, as a multiple of 2^-24 * sum |v| / S: (n_adds + 1) roundings
    on any term's path, n_adds = 32 sequential fp32 adds per 32-row half-warpgroup + S/32 atomics of the scaled partials
    (S a multiple of 32) or S atomics (otherwise), + 1 for the product with fl(1/S); the first add onto zero is exact,
    which covers the rounding of fl(1/S).  gamma_n = n u / (1 - n u) makes it rigorous."""
    n = (32 + S // 32 if S % 32 == 0 else S) + 1
    return n / (1 - n * U24)

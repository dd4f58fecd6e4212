"""The per-ray stages of csrc/render.cu against fp64: stratified sampling, compositing, its backward, hierarchical
resampling and the sparsity gradient, standalone and inside the training and render calls.

Every reference here is built in fp64 from the kernel's own fp32 inputs, and every bar is a multiple of u = 2^-24
times an fp64 magnitude that bounds how far fp32 arithmetic in any summation order can land from the exact value
(order-independent gamma bounds: the warp-scan order does not enter).  test_train_stages.py starts from the
workspace's G; this file checks what leads up to it: z, weights, comp, disp, acc, the fine z, G and the sparsity rows.

Magnitudes (derivations; i is the sample index along the ray):
- The fp32 alpha_j = 1 - expf(-x_j) (x = sigma delta) is off by ea_j u = ((2 + 5 |x_j|) a_j [x_j != 0] +
  [a_j < 1/2] / 2) u: expf's 2 ulp and the argument's few ulp of delta, then 1 - a rounded to the 2^-24 grid below 1
  (about u absolute: 1 - fl(1 - exp) is that grid).  o_j = 1 - alpha_j + 1e-10 adds one rounding: eo_j = ea_j + o_j / 2.
  So T_i = prod_{j<i} o_j is off by at most u * sum_{j<i} eo_j prod_{k<i, k!=j} o_k = u P_i (P_0 = 0,
  P_{i+1} = o_i P_i + eo_i T_i), plus i roundings of the product chain: m_i = i T_i + P_i.  w_i = alpha_i T_i then gets
  |alpha_i| m_i + ea_i T_i.  comp, acc and depth inherit sum_i (|alpha_i| m_i + ea_i T_i) * |factor_i|, plus
  N sum_i |w_i factor_i| for the fp32 sum in any order.
- A denormal floor F = N * 2^-125 is added to every T (u * F = N * 2^-149: the absolute error of N products that
  underflow in fp32, where the fp64 value is tiny but not zero), so saturated rays are bounded too.
- dL/dalpha_i = T_i (g_i - Q_i), Q_i = sum_{k>i} g_k alpha_k prod_{i<k'<k} o_k' (the kernel's suffix / o_i; its o_i
  cancels).  Q's error: alpha_k's absolute error reaches it through A_i = sum_{k>i} |g_k| ea_k prod_{i<k'<k} o_k', each
  o's through B_i = sum_{k'>i} eo_k' |dQ_i/do_k'| (A_i = |g_{i+1}| ea_{i+1} + o_{i+1} A_{i+1}, B_i = eo_{i+1} Qa_{i+1} +
  o_{i+1} B_{i+1}, Qa the recurrence of Q on absolute values), and the chain's own rounding through N * Qa_i.  So
  dalpha gets
  (|g_i| + Qa_i) m_i + T_i (|g_i| + A_i + B_i + N Qa_i), |g_i| formed from absolute values.
- d alpha / d sigma = delta_i a_i (a_i = exp(-sigma_i delta_i)) carries a RELATIVE bar only, (1 + sigma_i delta_i) u:
  delta's few-ulp relative error moves the exponent by sigma delta ulps; below 2^-126 (sigma delta > 87) expf's output
  is an fp32 denormal, whose absolute error adds delta 2^-149.  It is not granted 1 - alpha's absolute rounding: a
  factor formed as delta (1 - alpha) is off by 2^-24 / a, which this bar is there to catch.
- The fp32 cdf of sample_pdf is within E = (2 nw + 2) u of fp64 (nw interior weights: the weight sum, the padding
  and one division give each pdf entry (nw + 2) u relative; the running sum of at most nw entries <= 1 adds nw u).
"""
import json
import os

import numpy as np
import pytest
import torch

from tests.test_train import OUT
from tests.test_train_stages import CASES, Case, _params

U24 = 2.0 ** -24
DENORM = 2.0 ** -125       # per-sample floor in magnitude units (u * DENORM = 2^-149, fp32's smallest denormal)

# ---- bars: multiples of u times the magnitudes above.  Measured on an H100 80 GB HBM3 at a 400 W power limit, the
# largest value over every case of this file in brackets (standalone kernels, in-call and render-call checks)
W_BAR = 2.0                # weights                                                              [0.89]
ACC_BAR = 1.5              # acc, comp                                                            [0.75]
DISP_BAR = 1.0             # disp, relative: acc's and depth's magnitudes over their values       [0.45]
GRGB_BAR = 4.5             # G.rgb                                                                [1.94; 2.13 emulated]
GW_BAR = 3.5               # G.w                                                                  [1.69]
SQ_BAR = 0.8               # squared-error sums, in units of (rays + 4) u * sum                   [0.39]
PDF_Z_BAR = 1.5            # a new depth away from every cdf entry: u (|b0| + |b1|) + |b1 - b0| min(1, E / (c1 - c0))
                           #                                                                      [0.70; 0.72 emulated]
PDF_FM_BAR = 2.5           # forward map of every new depth through the fp64 cdf: E + u * slope * |z|   [1.16; 1.23 emulated]
PDF_FAR = 2.0              # "away from every cdf entry": farther than PDF_FAR * E
SP_BAR = 7.0               # sparsity G.w, in units of (1 + len * s) u * |G.w| (coef's three roundings and expf)   [3.39]
EXPSUM_BAR = 0.6           # stats[2], in units of u * sum_i e_i (n + 2 + len * s_i)             [0.31]
GUARD = 10.0               # a sensitivity guard must move its reference by at least this multiple of the bar
# measured guards: the (1 - alpha) factor moves G.w by >= 43.8 units (12.5 bars) from sigma delta = 10 on and by
# 13.6 units (3.9 bars) at 8; a bracket moved by one bin moves a far sample by >= 1.4e4 units


def _record(name, payload):
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, "parity_ray_stages.json")
    data = json.load(open(path)) if os.path.exists(path) else {}
    data[name] = payload
    json.dump(data, open(path, "w"), indent=1)


def _t(x, dev="cpu"):
    return torch.as_tensor(np.ascontiguousarray(x)).to(dev)


# =====================================================================================================================
# fp64 references (torch, any device) and their magnitudes
# =====================================================================================================================
def composite_ref(rgb, sigma, z, dirs, white):
    """volumetric_rendering in fp64 from fp32 rgb [R,N,3], sigma [R,N], z [R,N], dirs [R,3]."""
    rgb, s, z, d = rgb.double(), sigma.double(), z.double(), dirs.double()
    R, N = s.shape
    dn = d.norm(dim=-1)
    gap = torch.cat([z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)], -1)
    delta = gap * dn[:, None]
    x = s * delta
    a = torch.exp(-x)
    alpha = -torch.expm1(-x)
    o = a + 1e-10
    T = torch.cat([torch.ones_like(o[:, :1]), torch.cumprod(o[:, :-1], -1)], -1)
    w = alpha * T
    # absolute errors of the fp32 alpha and o, in units of u: expf's 2 ulp and the argument's few ulp (x a each),
    # then 1 - a rounded to the 2^-24 grid below 1 when a < 1/2 (exact otherwise); exp(0) = 1 and alpha = 0 exactly.
    # 1 - alpha is exact; adding 1e-10 rounds once more.
    ea = (x != 0).double() * (2 + 5 * x.abs()) * a + 0.5 * (a < 0.5).double()
    eo = ea + 0.5 * o.abs()
    P = torch.zeros_like(T)
    for i in range(N - 1):
        P[:, i + 1] = o[:, i].abs() * P[:, i] + eo[:, i] * T[:, i].abs()
    F = N * DENORM
    m = torch.arange(N, dtype=torch.float64, device=s.device) * T.abs() + P + F
    mw = alpha.abs() * m + ea * T.abs() + F
    bg = 1.0 if white else 0.0
    acc = w.sum(-1)
    depth = (w * z).sum(-1)
    comp = (w[..., None] * rgb).sum(-2) + bg * (1.0 - acc)[:, None]
    ratio = acc / depth
    disp = torch.where((ratio > 0) & (ratio < 1e10) & (acc > 1e-10), ratio, torch.full_like(ratio, 1e10))
    wa = w.abs()
    return dict(delta=delta, x=x, a=a, alpha=alpha, o=o, ea=ea, eo=eo, T=T, m=m, w=w, mw=mw, acc=acc, depth=depth,
                comp=comp, ratio=ratio, disp=disp, bg=bg,
                mag_acc=(mw + N * wa).sum(-1), mag_depth=((mw + N * wa) * z.abs()).sum(-1),
                mag_comp=((mw + N * wa)[..., None] * (rgb.abs() + bg)).sum(-2) + bg, rgb=rgb, s=s, z=z)


def composite_bwd_ref(f, comp32, px, gscale, factor=None):
    """G of (gscale / 2) sum_c (C_c - px_c)^2 w.r.t. (pre-sigmoid rgb, raw sigma) in closed form, with the
    residual taken from the kernel's own fp32 comp.  factor: override of d alpha / d sigma (a sensitivity guard)."""
    rgb, s, bg, o, alpha, T = f["rgb"], f["s"], f["bg"], f["o"], f["alpha"], f["T"]
    N = s.shape[1]
    dc = gscale * (comp32.double() - px.double())                         # [R,3]
    g = (dc[:, None, :] * (rgb - bg)).sum(-1)
    ga = (dc.abs()[:, None, :] * (rgb - bg).abs()).sum(-1)
    Q, Qa, A, B = (torch.zeros_like(g) for _ in range(4))
    for i in range(N - 2, -1, -1):
        oo = o[:, i + 1].abs()
        Q[:, i] = g[:, i + 1] * alpha[:, i + 1] + o[:, i + 1] * Q[:, i + 1]
        Qa[:, i] = ga[:, i + 1] * alpha[:, i + 1].abs() + oo * Qa[:, i + 1]
        A[:, i] = ga[:, i + 1] * f["ea"][:, i + 1] + oo * A[:, i + 1]
        B[:, i] = f["eo"][:, i + 1] * Qa[:, i + 1] + oo * B[:, i + 1]
    dalpha = T * (g - Q)
    Tm = T.abs() + N * DENORM
    mag_da = (ga + Qa) * f["m"] + Tm * (ga + A + B + N * Qa)
    fac = f["delta"] * f["a"] if factor is None else factor
    on = (s > 0).double()
    Gw = dalpha * fac * on
    # + DENORM: the stored product itself may be an fp32 denormal (one more absolute 2^-149)
    mag_gw = (mag_da * fac.abs() + ((1.0 + f["x"].abs()) * fac.abs() + f["delta"] * DENORM) * dalpha.abs()
              + DENORM) * on
    crgb = rgb * (1.0 - rgb)
    Grgb = f["w"][..., None] * dc[:, None, :] * crgb
    mag_rgb = (f["mw"] + f["w"].abs())[..., None] * (dc.abs()[:, None, :] * crgb.abs()) + DENORM
    e2 = ((comp32.double() - px.double()) ** 2).sum(-1)
    return dict(Gw=Gw, mag_gw=mag_gw, Grgb=Grgb, mag_rgb=mag_rgb, sq=e2.sum(), n=s.shape[0], dalpha=dalpha)


def _norm(err, mag):
    """err / (u * mag), 0 where both vanish"""
    return torch.where(err == 0, torch.zeros_like(err), err / (U24 * mag).clamp_min(1e-300))


def check_composite(f, comp, disp, acc, w):
    """normalised errors of the kernel's forward outputs (fp32 tensors) against composite_ref f."""
    out = {}
    out["w"] = float(_norm((w.double() - f["w"]).abs(), f["mw"]).max())
    out["acc"] = float(_norm((acc.double() - f["acc"]).abs(), f["mag_acc"]).max())
    out["comp"] = float(_norm((comp.double() - f["comp"]).abs(), f["mag_comp"]).max())
    # disp: the where() decides on acc > 1e-10, which is ambiguous within acc's bar of the threshold; there the
    # kernel may return either branch.  Its own outputs must still obey the rule: acc <= 1e-10 -> 1e10.
    band = ACC_BAR * U24 * f["mag_acc"]
    take = (f["acc"] - band > 1e-10) & (f["ratio"] > 0) & (f["ratio"] < 1e10 * (1 - 1e-6))
    inf_ = (f["acc"] + band < 1e-10) | (f["ratio"] <= 0)
    dd = disp.double()
    rel = (f["mag_acc"] / f["acc"].abs().clamp_min(1e-300) + f["mag_depth"] / f["depth"].abs().clamp_min(1e-300))
    err = _norm((dd - f["ratio"]).abs(), rel * f["ratio"].abs())
    amb = ~(take | inf_)
    ok_amb = (dd == 1e10) | (err <= DISP_BAR)
    out["disp"] = float(err[take].max()) if bool(take.any()) else 0.0
    out["disp_rule_violations"] = int(((inf_ & (dd != np.float32(1e10))) | (amb & ~ok_amb)).sum()
                                      + ((acc <= 1e-10) & (disp != 1e10)).sum())
    out["disp_kernel_acc_in_0_1e-10"] = int(((acc > 0) & (acc <= 1e-10)).sum())
    return out


def check_composite_bwd(b, G, sq=None):
    out = {"G_rgb": float(_norm((G[..., :3].double() - b["Grgb"]).abs(), b["mag_rgb"]).max()),
           "G_w": float(_norm((G[..., 3].double() - b["Gw"]).abs(), b["mag_gw"]).max()),
           "G_nonfinite": int((~torch.isfinite(G)).sum())}
    if sq is not None:
        out["sq"] = abs(float(sq) - float(b["sq"])) / (U24 * (b["n"] + 4) * max(float(b["sq"]), 1e-300))
    return out


def assert_composite(r, bwd=True):
    assert r["w"] <= W_BAR and r["acc"] <= ACC_BAR and r["comp"] <= ACC_BAR, r
    assert r["disp"] <= DISP_BAR and r["disp_rule_violations"] == 0, r
    if bwd:
        assert r["G_nonfinite"] == 0 and r["G_rgb"] <= GRGB_BAR and r["G_w"] <= GW_BAR, r
        if "sq" in r:
            assert r["sq"] <= SQ_BAR, r


def pdf_ref(zc, w, u):
    """piecewise_constant_pdf in fp64 (the reference's find_interval: i0 = last cdf entry <= u) from fp32 zc [R,Nc],
    weights [R,Nc] (the interior ones are used) and u [R,Nf]."""
    zc, w, u = zc.double(), w.double(), u.double()
    R, Nc = zc.shape
    nw, nb = Nc - 2, Nc - 1
    bins = 0.5 * (zc[:, 1:] + zc[:, :-1])
    wl = w[:, 1:-1]
    ws = wl.sum(-1, keepdim=True)
    pad = (1e-5 - ws).clamp_min(0)
    pdf = (wl + pad / nw) / (ws + pad)
    cdf = torch.cat([torch.zeros_like(ws), torch.cumsum(pdf[:, :-1], -1).clamp_max(1), torch.ones_like(ws)], -1)
    lo = torch.searchsorted(cdf, u, right=True)          # count of entries <= u
    i0 = (lo - 1).clamp_min(0)
    i1 = lo.clamp_max(nb - 1)
    c0, c1 = cdf.gather(1, i0), cdf.gather(1, i1)
    b0, b1 = bins.gather(1, i0), bins.gather(1, i1)
    t = torch.nan_to_num((u - c0) / (c1 - c0), nan=0.0).clamp(0, 1)
    E = U24 * (2 * nw + 2)
    return dict(bins=bins, cdf=cdf, i0=i0, i1=i1, c0=c0, c1=c1, b0=b0, b1=b1, z=b0 + t * (b1 - b0), E=E, u=u)


def _split_union(zu, zc):
    """the union's entries that are not coarse depths (multiset difference, per ray), or None if a coarse depth is
    missing from the union bit for bit."""
    out = []
    for r in range(zu.shape[0]):
        uz, uc = np.unique(zu[r], return_counts=True)
        cz, cc = np.unique(zc[r], return_counts=True)
        k = np.searchsorted(uz, cz)
        if np.any(k >= uz.size) or np.any(uz[np.minimum(k, uz.size - 1)] != cz) or np.any(uc[k] < cc):
            return None
        rem = uc.copy()
        rem[k] -= cc
        out.append(np.repeat(uz, rem))
    return np.stack(out)


def check_pdf(zu, zc, w, u, dev="cpu", shift=0):
    """checks of one sample_pdf result zu [R, Nc+Nf] (fp32 numpy) for zc, w [R,Nc] and u [R,Nf] (fp32 numpy).
    shift: move the reference's bracket by this many bins (the sensitivity guard)."""
    R, Nc = zc.shape
    out = {"unsorted": int((zu[:, 1:] < zu[:, :-1]).sum())}
    new = _split_union(zu, zc)
    out["coarse_missing"] = int(new is None)
    if new is None:
        return out
    order = np.argsort(u, axis=1, kind="stable")
    us = np.take_along_axis(u, order, 1)
    p = pdf_ref(_t(zc, dev), _t(w, dev), _t(us, dev))
    nb = Nc - 1
    if shift:
        i0 = (p["i0"] + shift).clamp(0, nb - 1)
        i1 = (p["i1"] + shift).clamp(0, nb - 1)
        c0, c1 = p["cdf"].gather(1, i0), p["cdf"].gather(1, i1)
        b0, b1 = p["bins"].gather(1, i0), p["bins"].gather(1, i1)
        tt = torch.nan_to_num((p["u"] - c0) / (c1 - c0), nan=0.0).clamp(0, 1)
        p["z_shift"] = b0 + tt * (b1 - b0)
    z = _t(new, dev).double()
    uu, cdf, bins, E = p["u"], p["cdf"], p["bins"], p["E"]
    far = ((uu - p["c0"]).abs() > PDF_FAR * E) & ((p["c1"] - uu).abs() > PDF_FAR * E)
    width = (p["b1"] - p["b0"]).abs()
    zbar = U24 * (p["b0"].abs() + p["b1"].abs()) + width * torch.clamp(E / (p["c1"] - p["c0"]).clamp_min(1e-300), max=1)
    zerr = (z - p["z"]).abs() / zbar.clamp_min(1e-300)
    out["far"] = int(far.sum())
    out["z_far"] = float(zerr[far].max()) if bool(far.any()) else 0.0
    if shift:
        serr = (p["z_shift"] - p["z"]).abs() / zbar.clamp_min(1e-300)
        out["shift_guard"] = float(serr[far].max()) if bool(far.any()) else 0.0
    lo_b, hi_b = p["b0"] - 2 * U24 * p["b0"].abs(), p["b1"] + 2 * U24 * p["b1"].abs()
    out["bracket_violations"] = int((far & ((z < lo_b) | (z > hi_b))).sum())
    # exact ties: u equal to an fp64 cdf entry that fp32 also holds exactly (a multiple of 1/64: the zero plateaus and
    # the unit weights of Nc = 66), the sample must be the tie rule's bin in fp32, fl(0.5 * fl(z[i0+1] + z[i0]))
    c0 = p["c0"]
    tie = (uu == c0) & ((c0 * 64) == torch.round(c0 * 64))
    b32 = (np.float32(0.5) * (zc[:, 1:] + zc[:, :-1])).astype(np.float32)
    want = np.take_along_axis(b32, p["i0"].cpu().numpy(), 1)
    tie_np = tie.cpu().numpy()
    out["ties"] = int(tie_np.sum())
    out["tie_mismatches"] = int((tie_np & (new != want)).sum())
    # forward map of every new depth through the fp64 cdf: the set of u that maps onto z (an interval where z is a
    # bin edge shared by several entries), its distance to u, against E + u * slope * |z| with the steepest slope of
    # the bracket z lands in and its neighbours
    kl = torch.searchsorted(bins, z, right=False)
    kr = torch.searchsorted(bins, z, right=True)
    k = kl.clamp(1, nb - 1)
    x0, x1 = bins.gather(1, k - 1), bins.gather(1, k)
    y0, y1 = cdf.gather(1, k - 1), cdf.gather(1, k)
    span = (x1 - x0)
    ub = torch.where(span > 0, y0 + (z - x0).clamp_min(0) / span.clamp_min(1e-300) * (y1 - y0), y0).clamp(y0, y1)
    lo_set = torch.where(kr > kl, cdf.gather(1, kl.clamp_max(nb - 1)), ub)
    hi_set = torch.where(kr > kl, cdf.gather(1, (kr - 1).clamp(0, nb - 1)), ub)
    dist = torch.maximum(lo_set - uu, uu - hi_set).clamp_min(0)
    slope = (cdf[:, 1:] - cdf[:, :-1]) / (bins[:, 1:] - bins[:, :-1]).clamp_min(1e-300)
    slope = torch.where(bins[:, 1:] > bins[:, :-1], slope, torch.zeros_like(slope))
    sl = torch.stack([slope.gather(1, (k - 1 + j).clamp(0, nb - 2)) for j in (-1, 0, 1)]).amax(0)
    out["fm"] = float((dist / (E + U24 * sl * z.abs())).max())
    return out


def assert_pdf(r):
    assert r["unsorted"] == 0 and r["coarse_missing"] == 0, r
    assert r["bracket_violations"] == 0 and r["tie_mismatches"] == 0, r
    assert r["z_far"] <= PDF_Z_BAR and r["fm"] <= PDF_FM_BAR, r


def sample_coarse_np(z_base, t_rand, R):
    """sample_coarse_kernel's arithmetic in numpy fp32 (separately rounded, like the kernel's __f*_rn)"""
    f = np.float32
    zb = np.asarray(z_base, f)
    N = zb.size
    if t_rand is None:
        return np.broadcast_to(zb, (R, N)).copy()
    mids = (f(0.5) * (zb[1:] + zb[:-1])).astype(f)
    lower = np.concatenate([zb[:1], mids]).astype(f)
    upper = np.concatenate([mids, zb[-1:]]).astype(f)
    return (lower + ((upper - lower).astype(f) * t_rand).astype(f)).astype(f)


# =====================================================================================================================
# numpy fp32 emulations of the kernels (rehearse the bars without a GPU)
# =====================================================================================================================
def emu_composite(rgb, sigma, z, dirs, white, px=None, gscale=None, one_minus_alpha=False):
    """composite_fwd_kernel / composite_bwd_kernel in fp32 (sequential order).  one_minus_alpha: the d alpha / d sigma
    factor as dist * (1 - alpha), as the kernel formed it before it kept exp's output."""
    f = np.float32
    with np.errstate(all="ignore"):
        R, N = sigma.shape
        dn = np.sqrt(((dirs[:, 0] * dirs[:, 0] + dirs[:, 1] * dirs[:, 1]).astype(f) + dirs[:, 2] * dirs[:, 2]).astype(f))
        gap = np.concatenate([(z[:, 1:] - z[:, :-1]).astype(f), np.full((R, 1), 1e10, f)], 1)
        dist = (gap * dn[:, None].astype(f)).astype(f)
        ex = np.exp(-(sigma * dist).astype(f).astype(np.float64)).astype(f)    # expf, correctly rounded
        alpha = (f(1) - ex).astype(f)
        om = ((f(1) - alpha).astype(f) + f(1e-10)).astype(f)
        T = np.ones(R, f)
        w = np.empty((R, N), f)
        Tpre = np.empty((R, N), f)
        for i in range(N):
            Tpre[:, i] = T
            w[:, i] = alpha[:, i] * T
            T = (T * om[:, i]).astype(f)
        acc = w.sum(-1, dtype=f)
        depth = (w * z).astype(f).sum(-1, dtype=f)
        comp = (w[..., None] * rgb).astype(f).sum(1, dtype=f)
        if white:
            comp = (comp + (f(1) - acc)[:, None]).astype(f)
        disp = (acc / depth).astype(f)
        disp = np.where((disp > 0) & (disp < f(1e10)) & (acc > f(1e-10)), disp, f(1e10)).astype(f)
        if px is None:
            return comp, disp, acc, w
        bg = f(1) if white else f(0)
        dc = (f(gscale) * (comp - px).astype(f)).astype(f)
        gi = ((dc[:, None, :] * (rgb - bg).astype(f)).astype(f)).sum(-1, dtype=f)
        G = np.zeros((R, N, 4), f)
        suffix = np.zeros(R, f)
        fac = (dist * ((f(1) - alpha).astype(f) if one_minus_alpha else ex)).astype(f)
        for i in range(N - 1, -1, -1):
            dalpha = ((gi[:, i] * Tpre[:, i]).astype(f) - (suffix / om[:, i]).astype(f)).astype(f)
            G[:, i, 3] = np.where(sigma[:, i] > 0, (dalpha * fac[:, i]).astype(f), f(0))
            G[:, i, :3] = (w[:, i, None] * dc * rgb[:, i] * (f(1) - rgb[:, i])).astype(f)
            suffix = (suffix + (gi[:, i] * w[:, i]).astype(f)).astype(f)
        sq = float((((comp - px).astype(f)) ** 2).astype(f).sum(dtype=f))
        return comp, disp, acc, w, G, sq


def emu_pdf(zc, w, u, strict=False):
    """sample_pdf_kernel in fp32; strict: the bracket search with cdf[mid] < u instead of <= u."""
    f = np.float32
    R, Nc = zc.shape
    nb, nw = Nc - 1, Nc - 2
    out = np.empty((R, Nc + u.shape[1]), f)
    with np.errstate(all="ignore"):
        for r in range(R):
            bins = (f(0.5) * (zc[r, 1:] + zc[r, :-1])).astype(f)
            wl = w[r, 1:-1].astype(f)
            ws = f(wl.sum(dtype=f))
            pad = max(f(0), f(f(1e-5) - ws))
            padw = f(pad / f(nw))
            ws = f(ws + pad)
            pdf = ((wl + padw) / ws).astype(f)
            cdf = np.empty(nb, f)
            cdf[0], cdf[-1] = 0, 1
            cdf[1:nw] = np.minimum(f(1), np.cumsum(pdf, dtype=f)[:nw - 1])
            lo = np.searchsorted(cdf, u[r], side="left" if strict else "right")
            i0, i1 = np.maximum(lo - 1, 0), np.minimum(lo, nb - 1)
            t = ((u[r] - cdf[i0]).astype(f) / (cdf[i1] - cdf[i0]).astype(f)).astype(f)
            t = np.clip(np.nan_to_num(t, nan=0.0), 0, 1).astype(f)
            new = (bins[i0] + (t * (bins[i1] - bins[i0]).astype(f)).astype(f)).astype(f)
            out[r] = np.sort(np.concatenate([zc[r], new]))
    return out


# =====================================================================================================================
# input families
# =====================================================================================================================
def ray_families(N, seed):
    """rays [R,N] of every family: (rgb, sigma, z, dirs, px, family index per ray).  R is not a multiple of 4."""
    f = np.float32
    rs = np.random.RandomState(1000 + N + seed)
    rays = []

    def base(zdup=False):
        z = np.sort(rs.uniform(2, 6, N)).astype(f)
        if zdup and N > 2:
            k = rs.randint(0, N - 1, size=max(1, N // 4))
            z[k + 1] = z[k]
            z = np.sort(z)
        d = rs.normal(size=3).astype(f)
        d = (d / np.linalg.norm(d) * rs.uniform(0.25, 4)).astype(f)
        rgb = rs.uniform(0, 1, (N, 3)).astype(f)
        return rgb, z, d

    def gap(z, d, i):
        return float((z[i + 1] - z[i]) if i + 1 < N else 1e10) * float(np.linalg.norm(d))

    def add(fam, rgb, s, z, d):
        rays.append((rgb, np.asarray(s, f), z, d, rs.uniform(0, 1, 3).astype(f), fam))

    for _ in range(3):                                                          # 0: random densities
        rgb, z, d = base()
        add(0, rgb, rs.uniform(-1, 3, N).clip(0) * rs.choice([0.2, 5.0, 50.0]), z, d)
    rgb, z, d = base()
    add(1, rgb, np.zeros(N), z, d)                                              # 1: empty
    for acc in (1e-11, 3e-11, 1e-10, 3e-10, 1e-9):                              # 2: near-empty
        rgb, z, d = base()
        add(2, rgb, np.full(N, acc / ((z[-1] - z[0] + 1e10) * np.linalg.norm(d))), z, d)
    for x in OPAQUE_X:                                                          # 3: opaque first sample, empty
        for behind in (0.0, 2.0):                                               #    space or content behind it
            rgb, z, d = base()
            s = rs.uniform(0, behind, N).astype(f)
            s[0] = x / gap(z, d, 0)
            add(3 if behind == 0 else 11, rgb, s, z, d)
    if N > 4:                                                                   # 4: saturation mid-ray (T underflows)
        rgb, z, d = base()
        s = np.zeros(N)
        s[N // 4:3 * N // 4] = 2e3
        add(4, rgb, s, z, d)
    for x in (0.1, 1.0, 5.0, 12.0, 17.0, 30.0, 100.0):                         # 5: last sample, sigma * 1e10 * |d|
        rgb, z, d = base()
        s = np.zeros(N)
        s[-1] = x / gap(z, d, N - 1)
        add(5, rgb, s, z, d)
    rgb, z, d = base()                                                          # 6: exact zeros between positives
    s = rs.uniform(0.1, 3, N)
    s[1::2] = 0
    add(6, rgb, s, z, d)
    rgb, z, d = base(zdup=True)                                                 # 7: repeated depths (delta = 0)
    add(7, rgb, rs.uniform(0, 3, N), z, d)
    for c in (0.0, 1.0, 1.0 - 2.0 ** -24):                                      # 8: colours at the sigmoid's ends
        rgb, z, d = base()
        add(8, np.full((N, 3), c, f), rs.uniform(0, 2, N), z, d)
    for sc in (0.25, 4.0):                                                      # 9: |d| at both ends
        rgb, z, d = base()
        add(9, rgb, rs.uniform(0, 2, N), z, (d / np.linalg.norm(d) * sc).astype(f))
    if N > 1:                                                                   # 10: cancelling signed densities:
        for x0 in (1.25, 2.25):                                                 #     alpha_1 steps along the 2^-24
            for k in np.arange(1, 10, 0.25):                                    #     grid past -alpha_0 (expf is
                rgb, z, d = base()                                              #     within 2 ulp there), so that
                s = np.zeros(N)                                                 #     some ray has 0 < acc <= 1e-10
                s[0] = -x0 * 2.0 ** -23 / gap(z, d, 0)
                s[1] = k * 2.0 ** -24 / gap(z, d, 1)
                add(10, rgb, s, z, d)
    if len(rays) % 4 == 0:
        rgb, z, d = base()
        add(0, rgb, rs.uniform(0, 2, N), z, d)
    rgb, s, z, d, px, fam = (np.stack([r[i] for r in rays]) for i in range(6))
    return rgb.astype(f), s.astype(f), z.astype(f), d.astype(f), px.astype(f), fam


def pdf_families(Nc, Nf, seed):
    """(zc [R,Nc], weights [R,Nc], u [R,Nf]) over every weight family and three kinds of u."""
    f = np.float32
    rs = np.random.RandomState(2000 + Nc + 7 * Nf + seed)
    nw = Nc - 2
    Ws = [np.zeros(Nc)]                                                         # padding path
    for tot in (1e-5 * (1 - 1e-3), 1e-5 * (1 + 1e-3)):                          # sum just below / above eps
        Ws.append(np.r_[0, rs.uniform(0.5, 1.5, nw) * tot / nw * 1.0, 0])
    for k in (1, nw):                                                           # single spike, first / last interior
        v = np.zeros(Nc)
        v[k] = 0.9
        Ws.append(v)
    p = max(1, nw // 3)
    v = rs.uniform(0, 1, Nc); v[1:1 + p] = 0; Ws.append(v)                      # leading zero plateau
    v = rs.uniform(0, 1, Nc); v[Nc - 1 - p:] = 0; Ws.append(v)                  # trailing
    v = rs.uniform(0, 1, Nc); v[nw // 3:nw // 3 + p] = 0; Ws.append(v)          # interior
    Ws.append(np.full(Nc, 1.0 / Nc))                                            # flat
    Ws.append(rs.uniform(0, 1, Nc) ** 8)                                        # peaky
    Ws.append(np.ones(Nc))                                                      # unit (exact cdf when nw = 64)
    w = np.stack(Ws).astype(f)
    R = w.shape[0]
    zc = np.sort(rs.uniform(2, 6, (R, Nc)), axis=1).astype(f)
    table = torch.linspace(0.0, 1.0 - float(np.finfo(np.float32).eps), Nf).numpy()   # NerfModel.u_table
    ties = (np.arange(Nf) % 65 / 64.0).astype(f)                                # every k/64, 0 included
    us = [np.broadcast_to(table, (R, Nf)).copy(), rs.uniform(0, 1, (R, Nf)).astype(f),
          np.broadcast_to(ties, (R, Nf)).copy()]
    return zc, w, us


# =====================================================================================================================
# CPU: the references against autograd of the oracle, the emulated kernel against the bars, the guards
# =====================================================================================================================
def test_composite_reference_matches_oracle_autograd():
    """composite_ref / composite_bwd_ref equal fp64 torch autograd of oracle.volumetric_rendering, on random and edge
    rays (every family; G.w in the closed form with Q, rgb through the sigmoid)."""
    from oracle import nerf_sh_oracle as O
    for N in (1, 2, 33, 64, 97):
        rgb, s, z, d, px, fam = ray_families(N, 0)
        keep = fam != 10                                        # the oracle's sigma is a relu output
        rgb, s, z, d, px = rgb[keep], s[keep], z[keep], d[keep], px[keep]
        for white in (True, False):
            rt = torch.from_numpy(rgb).double().requires_grad_(True)
            st = torch.from_numpy(s).double()[..., None].requires_grad_(True)
            comp, disp, acc, w = O.volumetric_rendering(rt, st, torch.from_numpy(z).double(),
                                                        torch.from_numpy(d).double(), white)
            f = composite_ref(_t(rgb), _t(s), _t(z), _t(d), white)
            # the oracle's 1 - exp(-x) cancels in fp64 (absolute error ~1e-16 where the reference takes -expm1(-x)):
            # that is all that separates the two on the near-empty rays
            for a, b in ((comp, f["comp"]), (acc, f["acc"]), (w, f["w"])):
                np.testing.assert_allclose(a.detach().numpy(), b.numpy(), rtol=1e-12, atol=1e-15)
            rtol = 1e-12 + 1e-15 / f["acc"].abs().clamp_min(1e-300).numpy()
            assert np.all(np.abs(disp.detach().numpy() - f["disp"].numpy()) <= rtol * f["disp"].abs().numpy())
            gscale = 0.37
            comp32 = comp.detach().float()
            # the closed form takes the residual as given (the kernel's comp): autograd of the same quadratic form
            loss = 0.5 * gscale * (2 * ((comp - comp.detach()) * (comp32.double() - torch.from_numpy(px).double()))
                                   ).sum()
            g_rgb, g_sig = torch.autograd.grad(loss, [rt, st])
            b = composite_bwd_ref(f, comp32, _t(px), gscale)
            want_rgb = (g_rgb * rt * (1 - rt)).detach()
            want_w = (g_sig[..., 0] * (st[..., 0] > 0)).detach()
            np.testing.assert_allclose(b["Grgb"].numpy(), want_rgb.numpy(), rtol=1e-10, atol=1e-15)
            scale = want_w.abs().amax(-1, keepdim=True).clamp_min(1e-300)
            # fp64 rounding of the magnitudes (g cancels on the colours at 1 - 2^-24 under a white background)
            err = (((b["Gw"] - want_w).abs() - 1e-6 * U24 * b["mag_gw"]).clamp_min(0) / scale).amax(-1)
            near_empty = torch.from_numpy(fam[keep] == 2)     # the oracle's alpha there: ~1e-16 / x relative
            assert float(err[~near_empty].max()) < 1e-9 and float(err[near_empty].max()) < 1e-4, (N, white)


def test_pdf_reference_matches_oracle():
    """pdf_ref's samples equal oracle.piecewise_constant_pdf run in fp64 on every weight family, ties included.  (The
    oracle, like the reference's zeros_like(cdf[..., :1]), cannot build a cdf from one interior weight: Nc >= 4.)"""
    from oracle import nerf_sh_oracle as O
    for Nc, Nf in ((4, 4), (5, 1), (34, 94), (66, 64), (200, 56)):
        zc, w, us = pdf_families(Nc, Nf, 0)
        zc64 = torch.from_numpy(zc).double()
        mids = 0.5 * (zc64[:, 1:] + zc64[:, :-1])
        for u in us:
            want = O.piecewise_constant_pdf(mids, torch.from_numpy(w).double()[:, 1:-1], Nf,
                                            torch.from_numpy(u).double())
            got = pdf_ref(_t(zc), _t(w), _t(u))["z"]
            np.testing.assert_array_equal(got.numpy(), want.numpy())


def _emu_bars(N, white, one_minus_alpha=False):
    rgb, s, z, d, px, fam = ray_families(N, 1)
    gscale = 0.37
    comp, disp, acc, w, G, sq = emu_composite(rgb, s, z, d, white, px, gscale, one_minus_alpha)
    f = composite_ref(_t(rgb), _t(s), _t(z), _t(d), white)
    r = check_composite(f, _t(comp), _t(disp), _t(acc), _t(w))
    b = composite_bwd_ref(f, _t(comp), _t(px), gscale)
    r.update(check_composite_bwd(b, _t(G), sq))
    gw = _norm((_t(G)[..., 3].double() - b["Gw"]).abs(), b["mag_gw"])[torch.from_numpy(fam == 3), 0]
    r["G_w_opaque_first"] = gw.tolist()          # sigma delta = OPAQUE_X in order
    return r, f, b, fam


OPAQUE_X = (8, 10, 12, 14, 16, 20, 40)


@pytest.mark.parametrize("N", [1, 2, 33, 97, 160, 256])
def test_emulated_composite_within_bars(N):
    """the numpy fp32 model of the fixed kernels passes every bar; the (1 - alpha) factor fails G.w on every ray
    with an opaque first sample, by >= GUARD x the bar from sigma delta = 10 on (at 8 its factor is off by ~400 u
    relative, against the bar's (1 + 8) u * GW_BAR)."""
    for white in (True, False):
        r, _, _, _ = _emu_bars(N, white)
        assert_composite(r)
        if N > 1:
            assert r["disp_kernel_acc_in_0_1e-10"] > 0, r        # the disp rule is exercised
        bad, _, _, _ = _emu_bars(N, white, one_minus_alpha=True)
        assert min(bad["G_w_opaque_first"]) > GW_BAR, bad
        assert min(bad["G_w_opaque_first"][1:]) > GUARD * GW_BAR, bad


@pytest.mark.parametrize("N", [1, 33, 192])
def test_composite_guards(N):
    """each guard moves the fp64 reference by >= GUARD x its bar: the (1 - alpha) factor (fp32 alpha) on opaque first
    samples, the white background's 1 - acc term."""
    rgb, s, z, d, px, fam = ray_families(N, 2)
    f = composite_ref(_t(rgb), _t(s), _t(z), _t(d), True)
    comp32 = f["comp"].float()
    b = composite_bwd_ref(f, comp32, _t(px), 0.37)
    alpha32 = (1 - np.exp(-(s * emu_delta(z, d)).astype(np.float32))).astype(np.float32)
    bad = composite_bwd_ref(f, comp32, _t(px), 0.37, factor=f["delta"] * (1 - _t(alpha32).double()))
    move = _norm((bad["Gw"] - b["Gw"]).abs(), b["mag_gw"])[torch.from_numpy(fam == 3), 0]
    assert float(move.min()) > GW_BAR and float(move[1:].min()) > GUARD * GW_BAR, move    # OPAQUE_X order
    black = composite_ref(_t(rgb), _t(s), _t(z), _t(d), False)
    move = _norm((black["comp"] - f["comp"]).abs(), f["mag_comp"]).amax(-1)
    assert float(move.max()) > GUARD * ACC_BAR
    assert float(move[torch.from_numpy(fam == 1)].min()) > GUARD * ACC_BAR     # an empty ray is all background


def emu_delta(z, d):
    f = np.float32
    R = z.shape[0]
    dn = np.sqrt(((d * d).astype(f)).sum(-1, dtype=f)).astype(f)
    gap = np.concatenate([(z[:, 1:] - z[:, :-1]).astype(f), np.full((R, 1), 1e10, f)], 1)
    return (gap * dn[:, None]).astype(f)


@pytest.mark.parametrize("Nc,Nf", [(3, 1), (4, 4), (34, 94), (64, 128), (66, 64), (255, 1)])
def test_emulated_pdf_within_bars(Nc, Nf):
    """the fp32 model of sample_pdf_kernel passes every check; the cdf[mid] < u bracket fails the tie check; a
    reference bracket moved by one bin moves far samples by >= GUARD x the bar."""
    zc, w, us = pdf_families(Nc, Nf, 1)
    caught = 0
    for u in us:
        r = check_pdf(emu_pdf(zc, w, u), zc, w, u, shift=1)
        assert_pdf(r)
        if r["far"]:
            assert r["shift_guard"] > GUARD * PDF_Z_BAR, r
        bad = check_pdf(emu_pdf(zc, w, u, strict=True), zc, w, u)
        caught += bad["tie_mismatches"]
    if Nc > 3:
        assert caught > 0                       # the leading plateau at u = 0 tells the two brackets apart


# =====================================================================================================================
# GPU: the standalone kernels
# =====================================================================================================================
def _lib():
    from plenoctree_b200._lib import check, lib, ptr
    return check, lib, ptr


def gpu_composite(rgb, s, z, d, white, px=None, gscale=None):
    check, lib, ptr = _lib()
    R, N = s.shape
    rgbs = torch.from_numpy(np.concatenate([rgb, s[..., None]], -1)).cuda().contiguous()
    zt, dt = torch.from_numpy(z).cuda(), torch.from_numpy(d).cuda()
    comp = torch.empty((R, 3), device="cuda")
    disp, acc = torch.empty(R, device="cuda"), torch.empty(R, device="cuda")
    w = torch.empty((R, N), device="cuda")
    check(lib.pob_composite(ptr(rgbs), ptr(zt), ptr(dt), R, N, int(white), ptr(comp), ptr(disp), ptr(acc), ptr(w),
                            None))
    out = dict(comp=comp, disp=disp, acc=acc, w=w)
    if px is not None:
        pxt = torch.from_numpy(px).cuda()
        G = torch.empty((R, N, 4), device="cuda")
        sq = torch.zeros(1, device="cuda")
        check(lib.pob_composite_bwd(ptr(rgbs), ptr(zt), ptr(dt), ptr(comp), ptr(pxt), R, N, int(white), gscale,
                                    ptr(G), ptr(sq), None))
        out.update(G=G, sq=sq)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


def gpu_sample_pdf(zc, w, u, per_ray):
    check, lib, ptr = _lib()
    R, Nc = zc.shape
    Nf = u.shape[-1]
    zt, wt, ut = (torch.as_tensor(x).cuda().contiguous() for x in (zc, w, u))
    out = torch.empty((R, Nc + Nf), device="cuda")
    check(lib.pob_sample_pdf(ptr(zt), ptr(wt), ptr(ut), int(per_ray), R, Nc, Nf, ptr(out), None))
    torch.cuda.synchronize()
    return out.cpu().numpy()


_STANDALONE_N = [1, 2, 31, 32, 33, 64, 65, 96, 97, 128, 129, 160, 161, 192, 193, 224, 225, 255, 256]


@pytest.mark.gpu
@pytest.mark.parametrize("N", _STANDALONE_N)
def test_composite_kernels_vs_fp64(N):
    """pob_composite and pob_composite_bwd per element against fp64, every S = ceil(N / 32) with both of its
    boundaries, both backgrounds, every ray family; R not a multiple of 4, and R = 1."""
    rgb, s, z, d, px, fam = ray_families(N, 3)
    gscale = 0.37
    rec = {}
    for white in (True, False):
        for sl in (slice(None), slice(0, 1)):
            g = gpu_composite(rgb[sl], s[sl], z[sl], d[sl], white, px[sl], gscale)
            f = composite_ref(_t(rgb[sl]), _t(s[sl]), _t(z[sl]), _t(d[sl]), white)
            r = check_composite(f, g["comp"], g["disp"], g["acc"], g["w"])
            b = composite_bwd_ref(f, g["comp"], _t(px[sl]), gscale)
            r.update(check_composite_bwd(b, g["G"], g["sq"]))
            if sl.stop is None:
                gw = _norm((g["G"][..., 3].double() - b["Gw"]).abs(), b["mag_gw"])
                # the parent's factor: dist * (1 - alpha) with the fp32 alpha, as a reference move
                alpha32 = (1 - np.exp(-(s * emu_delta(z, d)).astype(np.float32))).astype(np.float32)
                bad = composite_bwd_ref(f, g["comp"], _t(px), gscale, factor=f["delta"] * (1 - _t(alpha32).double()))
                mv = _norm((bad["Gw"] - b["Gw"]).abs(), b["mag_gw"])[torch.from_numpy(fam == 3), 0]
                r["guard_one_minus_alpha_x8"] = float(mv[0])
                r["guard_one_minus_alpha_min"] = float(mv[1:].min())
                r["G_w_per_family"] = {int(k): float(gw[torch.from_numpy(fam == k)].max()) for k in np.unique(fam)}
            rec[f"white{int(white)}_R{len(s[sl])}"] = r
    _record(f"composite_N{N}", rec)
    for k, r in rec.items():
        assert_composite(r)
        if "guard_one_minus_alpha_min" in r:
            assert r["guard_one_minus_alpha_min"] > GUARD * GW_BAR and r["guard_one_minus_alpha_x8"] > GW_BAR, (k, r)
            if N > 1:
                assert r["disp_kernel_acc_in_0_1e-10"] > 0, (k, r)


_PDF_SIZES = [(3, 1), (3, 253), (4, 4), (33, 31), (34, 94), (64, 128), (64, 192), (65, 64), (66, 64), (128, 128),
              (200, 56), (255, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("Nc,Nf", _PDF_SIZES)
def test_sample_pdf_kernel_vs_fp64(Nc, Nf):
    """pob_sample_pdf on every weight family and three kinds of u (the linspace table through the shared-table path,
    per-ray uniforms, exact k/64 ties): sorted, the coarse depths bit for bit, far samples in the fp64 bracket and
    within the bar, ties on the tie rule's bin, every sample's forward map within its bound."""
    zc, w, us = pdf_families(Nc, Nf, 3)
    rec = {}
    for i, u in enumerate(us):
        zu = gpu_sample_pdf(zc, w, u[0] if i == 0 else u, per_ray=i != 0)
        r = check_pdf(zu, zc, w, u)
        rec[["table", "uniform", "ties"][i]] = r
    _record(f"pdf_{Nc}_{Nf}", rec)
    for r in rec.values():
        assert_pdf(r)
    if Nc == 66:
        assert rec["ties"]["ties"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 2, 33, 256])
@pytest.mark.parametrize("lindisp", [False, True])
def test_sample_coarse_bit_exact(N, lindisp):
    check, lib, ptr = _lib()
    t = torch.linspace(0.0, 1.0, N, dtype=torch.float32)
    zb = 1.0 / (1.0 / 2.0 * (1.0 - t) + 1.0 / 6.0 * t) if lindisp else 2.0 * (1.0 - t) + 6.0 * t
    R = 37
    tr = np.random.RandomState(N).uniform(0, 1, (R, N)).astype(np.float32)
    for t_rand in (None, tr):
        zg = torch.empty((R, N), device="cuda")
        tt = None if t_rand is None else torch.from_numpy(t_rand).cuda()
        zbt = zb.cuda()
        check(lib.pob_sample_coarse(ptr(zbt), ptr(tt), R, N, ptr(zg), None))
        torch.cuda.synchronize()
        np.testing.assert_array_equal(zg.cpu().numpy(), sample_coarse_np(zb.numpy(), t_rand, R))


# =====================================================================================================================
# GPU: inside the training and render calls
# =====================================================================================================================
class RayCase(Case):
    """a training call of test_train_stages.py, plus background, lindisp, per-ray direction scale, a call over fewer
    rays than max_rays and the precision"""

    def __init__(self, *a, white=True, lindisp=False, dir_scale=False, n_call=None, precision=1, **k):
        super().__init__(*a, **k)
        self.white, self.lindisp, self.dir_scale, self.n_call, self.precision = white, lindisp, dir_scale, n_call, precision

    @property
    def name(self):
        return (super().name + ("" if self.white else "_black") + ("_lindisp" if self.lindisp else "")
                + ("_dirscale" if self.dir_scale else "") + (f"_n{self.n_call}" if self.n_call else "")
                + ("_x3" if self.precision == 3 else ""))

    def inputs(self, n):
        (o, d, v, px), t_rand, u, sp, noise = super().inputs(n)
        if self.dir_scale:
            d = (d * np.random.RandomState(self.seed + 2).uniform(0.3, 3, (n, 1))).astype(np.float32)
        return (o, d, v, px), t_rand, u, sp, noise

    def model(self, max_rays=None):
        from plenoctree_b200.nerf.models import NerfModel
        m = NerfModel(sh_deg=self.sh, num_coarse_samples=self.nc, num_fine_samples=self.nf, white_bkgd=self.white,
                      lindisp=self.lindisp, max_rays=max_rays or self.R, sparsity_npoints=self.nsp)
        fc, ff = _params(self.sh, self.seed)
        m.set_params(np.concatenate([fc, ff]) if self.nf else fc)
        return m


def _as_ray_case(c, **k):
    return RayCase(c.sh, c.R, c.nc, c.nf, c.nsp, noise=c.noise, seed=c.seed, sparsity_weight=c.sparsity_weight,
                   sp_radius=c.sp_radius, **k)


IN_CALL = [_as_ray_case(c) for c in CASES] + [
    RayCase(3, 96, 64, 128, 300, white=False),
    RayCase(3, 96, 64, 128, 300, dir_scale=True),
    RayCase(3, 96, 64, 128, 300, lindisp=True),
    RayCase(3, 96, 64, 128, 300, n_call=37),
    RayCase(3, 96, 64, 128, 300, precision=3),
    RayCase(3, 64, 64, 0, 200, white=False, n_call=29, precision=3),
]


def _check_levels(model, views, ws, rays, z_base, t_rand, u, upr, st, px=None, gscale=None):
    """forward (and with px: backward) ray-stage checks of every level of one call's workspace."""
    o, d, v = rays
    n = o.shape[0]
    dev = ws.device
    from plenoctree_b200 import layouts as L
    dt = torch.from_numpy(d).to(dev)
    res = {}
    levels = views["levels"]
    for i, lv in enumerate(levels):
        N, Mr = lv["N"], lv["M_rays"]
        z = L.workspace_view(ws, lv, "z")
        rgbs = L.workspace_view(ws, lv, "rgbs")[:Mr].view(n, N, 4)
        w = L.workspace_view(ws, lv, "weights")
        comp, disp, acc = (L.workspace_view(ws, lv, k) for k in ("comp", "disp", "acc"))
        if i == 0:
            want = sample_coarse_np(z_base, t_rand, n)
            st["coarse_z_bit_mismatches"] = int((z.cpu().numpy() != want).sum())
        else:
            c0 = levels[0]
            zc, wc = L.workspace_view(ws, c0, "z").cpu().numpy(), L.workspace_view(ws, c0, "weights").cpu().numpy()
            alone = gpu_sample_pdf(zc, wc, u, upr)
            st["fine_z_vs_standalone_bit_mismatches"] = int((alone != z.cpu().numpy()).sum())
            uu = np.broadcast_to(u, (n, u.shape[-1])).astype(np.float32)
            r = check_pdf(z.cpu().numpy(), zc, wc, uu, dev)
            res["pdf"] = r
        f = composite_ref(rgbs[..., :3], rgbs[..., 3], z, dt, model.white_bkgd)
        r = check_composite(f, comp, disp, acc, w)
        if px is not None:
            G = L.workspace_view(ws, lv, "G")[:Mr].view(n, N, 4)
            if model.sigma_activation == "softplus":
                # d sigma / d raw sigma = sigmoid(raw) = -expm1(-sigma) in G.w (test_sigma_activation.py: GW_SP_EXTRA)
                from tests.test_sigma_activation import GW_SP_EXTRA
                fac = f["delta"] * f["a"] * (-torch.expm1(-rgbs[..., 3].double()))
                b = composite_bwd_ref(f, comp, torch.from_numpy(px).to(dev), gscale, factor=fac)
                b["mag_gw"] = b["mag_gw"] + GW_SP_EXTRA * b["Gw"].abs()
                b_relu = composite_bwd_ref(f, comp, torch.from_numpy(px).to(dev), gscale)
                r["relu_factor_guard"] = float(_norm((b_relu["Gw"] - b["Gw"]).abs(), b["mag_gw"]).max())
            else:
                b = composite_bwd_ref(f, comp, torch.from_numpy(px).to(dev), gscale)
            r.update(check_composite_bwd(b, G))
            r["sq64"] = float(b["sq"])
        res[f"level{i}"] = r
    return res


def _in_call(case):
    from tests.test_train_x3 import _run
    model = case.model()
    n = case.n_call or case.R
    state, _ = _run(case, model, case.precision, n=n, fill=0xFF)
    return _in_call_checks(case, model, state, n)


def _in_call_checks(case, model, state, n):
    """the ray-stage checks of a training call over n rays of `case` already in the model's workspace"""
    from plenoctree_b200 import layouts as L
    from plenoctree_b200.nerf.train import default_loss_scale
    (o, d, v, px), t_rand, u, sp, _ = case.inputs(n)
    ws = model.workspace(True, case.precision)
    views = L.train_workspace_views(model.cfg, n, case.nsp > 0, precision=case.precision)
    assert views["total"] == ws.numel()
    ls = default_loss_scale(n, case.precision)
    gscale = ls * 2.0 / (3.0 * n)
    st = {}
    res = _check_levels(model, views, ws, (o, d, v), model.z_base.cpu().numpy(), t_rand, u, 1, st, px, gscale)
    stats = state.stats_raw.double().cpu()
    lvls = [k for k in res if k.startswith("level")]
    for slot, lk in zip((1, 0) if len(lvls) == 2 else (0,), lvls):     # fine in stats[0], coarse in stats[1]
        sq64 = res[lk].pop("sq64")
        res[lk]["sq"] = abs(float(stats[slot]) - sq64) / (U24 * (n + 4) * max(sq64, 1e-300))
    if case.nsp:
        lv = views["levels"][-1]
        Mr, M = lv["M_rays"], lv["M"]
        sgm = L.workspace_view(ws, lv, "rgbs")[Mr:M, 3].double().cpu()
        G = L.workspace_view(ws, lv, "G")[Mr:M].double().cpu()
        length = float(np.float32(0.05))
        coef = float(np.float32(ls)) * float(np.float32(case.sparsity_weight)) * length / case.nsp
        e = torch.exp(-length * sgm)
        want = coef * e * (sgm > 0)
        sp = dict(xyz_nonzero=int((G[:, :3] != 0).sum()), zero_sigma_rows=int((sgm <= 0).sum()),
                  w_at_zero_sigma_nonzero=int((G[sgm <= 0, 3] != 0).sum()),
                  w=float(_norm((G[:, 3] - want).abs(), (1 + length * sgm.abs()) * want.abs()).max()))
        mag = float((e * (case.nsp + 2 + length * sgm.abs())).sum())
        sp["exp_sum"] = abs(float(stats[2]) - float(e.sum())) / (U24 * mag)
        res["sparsity"] = sp
    res["stage"] = st
    return res


def _assert_in_call(res):
    for k, r in res.items():
        if k.startswith("level"):
            assert_composite(r, bwd="G_w" in r)
        elif k == "pdf":
            assert_pdf(r)
        elif k == "sparsity":
            assert r["xyz_nonzero"] == 0 and r["w_at_zero_sigma_nonzero"] == 0, r
            assert r["w"] <= SP_BAR and r["exp_sum"] <= EXPSUM_BAR, r
        elif k == "stage":
            assert all(x == 0 for x in r.values()), r


@pytest.mark.gpu
@pytest.mark.parametrize("case", IN_CALL, ids=lambda c: c.name)
def test_ray_stages_in_training_call(case):
    """z, weights, comp, disp, acc, the fine z, G, the sparsity rows and stats[0..2] of one pob_loss_and_grad call,
    read back from its workspace, against fp64 from the call's own inputs"""
    res = _in_call(case)
    _record(case.name, res)
    _assert_in_call(res)
    if case.nsp >= 64:
        assert res["sparsity"]["zero_sigma_rows"] > 0        # the [s > 0] rule is exercised


@pytest.mark.gpu
def test_ray_stages_production_step():
    case = RayCase(3, 4096, 64, 128, 10000)
    from plenoctree_b200._lib import RenderConfig, lib
    from plenoctree_b200.nerf.models import ctypes_ref
    need = int(lib.pob_workspace_bytes(ctypes_ref(RenderConfig(3, 64, 128, 1, 4096, 10000)), 1))
    free, _ = torch.cuda.mem_get_info()
    if free < need + (4 << 30):
        pytest.skip(f"the production step needs {need / 2**30:.1f} GB of workspace + ~4 GB; "
                    f"{free / 2**30:.1f} GB free on this (shared) device")
    res = _in_call(case)
    _record(case.name, res)
    _assert_in_call(res)


@pytest.mark.gpu
@pytest.mark.parametrize("randomized", [False, True])
def test_ray_stages_render_call(randomized):
    """NerfModel.__call__: the render workspace's stages against fp64 (the u table at randomized=False: its u = 0
    ties at every ray whose first interior weights are exactly zero), and the [n, 5] outputs equal the workspace's
    comp / disp / acc bit for bit"""
    from plenoctree_b200 import layouts as L
    from plenoctree_b200.nerf.models import Rays
    case = RayCase(3, 200, 64, 128, 0, dir_scale=True)
    model = case.model()
    n = 177
    (o, d, v, px), t_rand, u, _, _ = case.inputs(n)
    model.workspace(False).fill_(0xFF)
    out = model(Rays(o, d, v), randomized=randomized, t_rand=t_rand if randomized else None,
                u=u if randomized else None)
    torch.cuda.synchronize()
    ws = model.workspace(False)
    views = L.train_workspace_views(model.cfg, n, False, training=False)
    uu = u if randomized else model.u_table.cpu().numpy()[None]
    st = {}
    res = _check_levels(model, views, ws, (o, d, v), model.z_base.cpu().numpy(), t_rand if randomized else None,
                        uu, int(randomized), st)
    for i, lv in enumerate(views["levels"]):
        got = torch.cat([out[i][0], out[i][1][:, None], out[i][2][:, None]], 1)
        want = torch.cat([L.workspace_view(ws, lv, "comp"), L.workspace_view(ws, lv, "disp")[:, None],
                          L.workspace_view(ws, lv, "acc")[:, None]], 1)
        st[f"out_bit_mismatches_{i}"] = int((got.view(torch.int32) != want.view(torch.int32)).sum())
    res["stage"] = st
    _record(f"render_rand{int(randomized)}", res)
    _assert_in_call(res)
    if not randomized:
        assert res["pdf"]["ties"] > 0

"""The grid-weight render of extraction against fp64: its scene, sigma, shading reference and launch checks."""
import functools

import numpy as np

from oracle import octree_oracle as OO


f32, f64 = np.float32, np.float64
U24 = 2.0 ** -24

# ---- bars (measured on an H100 80 GB HBM3 at a 400 W power limit; the largest value in brackets)
# weight: |wmax - fp64| per voxel in units of max over the voxel's visits of
#   2^-24 * T_j * (att_j * (1 + tau_j) + (1 - att_j) * (1 + n_j + S_j))
# att_j = e^-tau_j, T_j = e^-S_j, S_j / n_j the optical depth / number of hits before visit j.  The first term is
# `__expf`'s error (2 + 1.17 |x| ulp) and the rounding of tau, both absolute in 1 - att; the second the rounding of
# 1 - att and of the weight, and the relative error `light` accumulates over the earlier visits.
WEIGHT_ALLOW = 4.0          # [2.03]


CUT = 100.0 * np.log(2.0)   # S_j beyond this: T_j < 2^-100, the kernel may already have stopped


STEP = 1e-5                 # --renderer_step_size of the reference's configs (octree/config/syn_sh16.json)
WEIGHT_THRESH = 1e-3


RADIUS = (1.3, 1.1, 1.45)
CENTER = (0.12, -0.08, 0.05)


@functools.lru_cache(maxsize=None)
def geometry():
    t = OO.N3Tree(radius=RADIUS, center=CENTER)
    return t.offset.copy(), t.invradius.copy()


M32 = 0xFFFFFFFF
BODY = (0.47, 0.53, 0.5, 0.17)      # centre, radius (unit cube)
SHELL = 0.33


def _hash(i):
    """32-bit mix of an int64 array (numpy or torch); every product stays below 2^63"""
    h = (i * 0x2C1B3C6D + 0x297A2D39) & M32
    h = h ^ (h >> 15)
    h = (h * 0x5BD1E995) & M32
    h = h ^ (h >> 13)
    h = (h * 0x297A2D39) & M32
    return h ^ (h >> 16)


def _sigma_expr(idx, reso, where, to_f64):
    """sigma of flat voxels idx (int64) as float64: every operation is an exact integer one or a single IEEE fp64
    operation, so numpy and torch (one kernel per operation) produce the same bits"""
    h = _hash(idx)
    u1 = to_f64(h >> 16) / 65536.0
    u2 = to_f64(h & 0xFFFF) / 65536.0
    i, j, k = idx // (reso * reso), (idx // reso) % reso, idx % reso
    dx = (to_f64(i) + 0.5) / reso - BODY[0]
    dy = (to_f64(j) + 0.5) / reso - BODY[1]
    dz = (to_f64(k) + 0.5) / reso - BODY[2]
    r2 = dx * dx + dy * dy + dz * dz
    scale = reso / (RADIUS[0] + RADIUS[1] + RADIUS[2]) * 1.5     # tau across one cell -> sigma
    body = r2 < BODY[3] * BODY[3]
    shell = (r2 > (SHELL - 1.0 / reso) ** 2) & (r2 < (SHELL + 1.0 / reso) ** 2)
    tau = where(body, 0.02 + 2.5 * u1, 0.0)
    tau = where(shell, where(u2 < 0.06, 95.0 + 300.0 * u1, 0.3 + 1.5 * u1), tau)
    occ = body | shell
    tau = where(occ & (u2 >= 0.8) & (u2 < 0.9), -tau, tau)
    tau = where(occ & (u2 >= 0.9), 0.0, tau)
    tau = where(~occ & (u2 < 0.01), 1e-6 * (1.0 + u1), tau)
    return tau * scale


def sigma_host(idx, reso):
    idx = np.asarray(idx, dtype=np.int64)
    return _sigma_expr(idx, reso, np.where, lambda a: a.astype(f64)).astype(f32)


def sigma_device(reso, chunk=1 << 25):
    import torch
    n = reso ** 3
    out = torch.empty(n, dtype=torch.float32, device="cuda")
    for lo in range(0, n, chunk):
        idx = torch.arange(lo, min(n, lo + chunk), dtype=torch.int64, device="cuda")
        out[lo:lo + idx.numel()] = _sigma_expr(idx, reso, torch.where, lambda a: a.double()).float()
    return out


def cam_rows(cams):
    rows = np.zeros((len(cams), 16), dtype=f32)
    for n, (c2w, W, H, f) in enumerate(cams):
        rows[n, :12] = np.asarray(c2w, f32)[:3, :4].reshape(12)
        rows[n, 12:] = (f, f, W, H)
    return rows


def _first(vis):
    R = vis["miss"].shape[0]
    count = np.bincount(vis["ray"], minlength=R)
    return np.cumsum(count) - count, count


def _excl_cumsum(x, vis, first, count, chunk=2048):
    """per-ray exclusive prefix sums in march order, summed within each ray only (a global cumsum would carry the
    other rays' magnitude into every S)"""
    out = np.zeros_like(x)
    ray = vis["ray"]
    R = count.size
    for r0 in range(0, R, chunk):
        r1 = min(R, r0 + chunk)
        v0, v1 = first[r0], first[r1 - 1] + count[r1 - 1]
        if v1 == v0:
            continue
        rr = ray[v0:v1]
        kk = np.arange(v0, v1) - first[rr]
        P = np.zeros((r1 - r0, int(count[r0:r1].max())))
        P[rr - r0, kk] = x[v0:v1]
        out[v0:v1] = (np.cumsum(P, axis=1) - P)[rr - r0, kk]
    return out


def shade64(vis, sig, delta_t=None, delta_scale=None):
    """fp64 weights of every visit of `vis` over the float32 sigma of its voxels (sig [V]) -> dict of per-visit
    hit, w, unit (the bar unit / 2^-24) and pre (the fp64 transmittance before the visit is >= 2^-100)"""
    first, count = _first(vis)
    dt = (vis["delta_t"] if delta_t is None else delta_t).astype(f64)
    ds = (vis["delta_scale"] if delta_scale is None else delta_scale).astype(f64)[vis["ray"]]
    hit = sig > 0
    tau = np.where(hit, dt * ds * sig.astype(f64), 0.0)
    S = _excl_cumsum(tau, vis, first, count)
    n = _excl_cumsum(hit.astype(f64), vis, first, count)
    T = np.exp(-S)
    att = np.exp(-tau)
    om = -np.expm1(-tau)
    w = np.where(hit, T * om, 0.0)
    unit = np.where(hit, T * (att * (1.0 + tau) + om * (1.0 + n + S)), 0.0)
    return dict(hit=hit, w=w, unit=unit, pre=S <= CUT, tau=tau)


def per_voxel(vox, w, unit, pre):
    """per voxel over the given (hit) visits -> keys, max w over the visits before the cut, max w over all, the
    unit (max over all visits; a visit past the cut adds an absolute 2^-100 / 2^-24), any visit before the cut"""
    unit = unit + np.where(pre, 0.0, 2.0 ** -100 / U24)
    order = np.argsort(vox, kind="stable")
    v = vox[order]
    keys, start = np.unique(v, return_index=True)
    if keys.size == 0:
        z = np.zeros(0)
        return dict(keys=keys, lo=z, hi=z, unit=z, pre=np.zeros(0, bool))
    return dict(keys=keys, lo=np.maximum.reduceat(np.where(pre, w, 0.0)[order], start),
                hi=np.maximum.reduceat(w[order], start), unit=np.maximum.reduceat(unit[order], start),
                pre=np.maximum.reduceat(pre[order].astype(np.uint8), start).astype(bool))


def merge(parts):
    vox = np.concatenate([p["keys"] for p in parts])
    order = np.argsort(vox, kind="stable")
    keys, start = np.unique(vox[order], return_index=True)
    out = dict(keys=keys)
    for k in ("lo", "hi", "unit"):
        out[k] = np.maximum.reduceat(np.concatenate([p[k] for p in parts])[order], start) if keys.size else np.zeros(0)
    out["pre"] = (np.maximum.reduceat(np.concatenate([p["pre"] for p in parts]).astype(np.uint8)[order], start)
                  .astype(bool) if keys.size else np.zeros(0, bool))
    return out


def weight_err(ref, keys_got, vals_got):
    """-> per-voxel error in units (0 inside [lo, hi]); keys_got must be a subset of ref['keys']"""
    pos = np.searchsorted(ref["keys"], keys_got)
    got = np.zeros(ref["keys"].size)
    got[pos] = vals_got
    err = np.maximum(ref["lo"] - got, got - ref["hi"])
    return np.maximum(err, 0.0) / (U24 * ref["unit"]), got


@functools.lru_cache(maxsize=1)
def device_sigma(reso):
    return sigma_device(reso)


def take(wmax, hit):
    """nonzero voxels of wmax (indices, values) and of hit (indices), and zero them again"""
    import torch
    kw = torch.nonzero(wmax).reshape(-1)
    vw = wmax[kw].cpu().numpy()
    kh = torch.nonzero(hit).reshape(-1)
    wmax[kw] = 0.0
    hit[kh] = 0
    return kw.cpu().numpy(), vw, kh.cpu().numpy()


def check_launch(ref, kw, vw, kh, tag):
    """path and values of one launch against its fp64 reference -> (largest error in units, mask margin count)"""
    required = ref["keys"][ref["pre"]]
    assert np.isin(kh, ref["keys"]).all(), (tag, "kernel hit a voxel no listed hit reaches")
    assert np.isin(required, kh).all(), (tag, "a listed hit before the cut is missing", np.setdiff1d(required, kh)[:8])
    assert np.isin(kw, ref["keys"]).all(), (tag, "nonzero weight on a voxel no positive-sigma visit reaches")
    err, got = weight_err(ref, kw, vw)
    worst = float(err.max()) if err.size else 0.0
    assert worst <= WEIGHT_ALLOW, (tag, worst, int(ref["keys"][np.argmax(err)]))
    # the mask outside the margin
    m = ref["hi"]
    margin = np.abs(m - WEIGHT_THRESH) <= WEIGHT_ALLOW * U24 * ref["unit"]
    bad = ((got >= f32(WEIGHT_THRESH)) != (m >= WEIGHT_THRESH)) & ~margin
    assert not bad.any(), (tag, int(bad.sum()))
    return worst, int(margin.sum()), int((m >= WEIGHT_THRESH).sum())

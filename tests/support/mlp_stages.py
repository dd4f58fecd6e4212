"""The fp16 training MLP against fp64, stage by stage: cases, inputs, models, the stage checker and its budgets."""
import functools
import time

import numpy as np
import torch

from plenoctree_b200 import layouts as L
from tests.support.records import record

_record = functools.partial(record, "parity_train_stages.json")


def _setup(sh_deg, R, nf, nsp, seed):
    from oracle import nerf_sh_oracle as O
    fc = O.init_flat_params(sh_deg, seed, bias_scale=0.05)
    ff = O.init_flat_params(sh_deg, seed + 1, bias_scale=0.05)
    K = (sh_deg + 1) ** 2
    for f in (fc, ff):
        off = O.param_count(sh_deg) - 3 * K - 1 - 256 * 3 * K - 256
        f[off:off + 256] *= 30.0
    o, d, v = _rays(R, seed)
    rs = np.random.RandomState(seed)
    px = rs.uniform(0, 1, size=(R, 3)).astype(np.float32)
    t_rand = rs.uniform(0, 1, size=(R, 64)).astype(np.float32)
    u = rs.uniform(0, 1, size=(R, nf)).astype(np.float32) if nf else None
    sp = rs.uniform(-1.5, 1.5, size=(nsp, 3)).astype(np.float32) if nsp else None
    return fc, ff, (o, d, v), px, t_rand, u, sp


def _rays(n, seed, radius=4.0):
    """rays of random spherical poses through random pixels of an 800x800 / focal 1111 camera."""
    from oracle import nerf_sh_oracle as O
    rs = np.random.RandomState(seed)
    o = np.zeros((n, 3), np.float32)
    d = np.zeros((n, 3), np.float32)
    for i in range(n):
        c2w = O.pose_spherical(rs.uniform(-180, 180), rs.uniform(-90, 0), radius)
        x, y = rs.randint(0, 800), rs.randint(0, 800)
        cam = np.array([(x - 400) / 1111.1, -(y - 400) / 1111.1, -1.0], np.float32)
        d[i] = c2w[:3, :3] @ cam
        o[i] = c2w[:3, 3]
    v = d / np.linalg.norm(d, axis=-1, keepdims=True)
    return o, d, v.astype(np.float32)


U24 = 2.0 ** -24

# ---- bars (measured on an H100 80 GB HBM3 at a 400 W power limit; the largest value over all cases of test_train_stages.py in
# brackets)
# forward / dgrad GEMMs: error beyond the rounding of the stored fp16 value, in units of 2^-24 * sum_k |a_k w_k|
FWD_ALLOW = 8.0             # [3.74]
BWD_ALLOW = 12.0            # [6.35, production step]
# positional encoding: sine columns within one fp16 ulp plus the reduced SFU sine's absolute error (2^-20)
SIN_ABS = 2.0 ** -20        # [0.5 of it beyond the ulp]; xyz columns bit-exact; rgbs: sigma [0.50], rgb [0.15] of their allowance
# weight gradient + reduce, per tensor: max |err| <= WG_EPS_W / WG_EPS_B * sum_s |a_s b_s| and relative L2 <= WG_EPS2_W /
# WG_EPS2_B (kernels / biases).  The kernels' error grows with the tiles one CTA sums in fp32 (~1 200 per Dense_0 CTA
# in the production step)
WG_EPS_W = 1e-4             # [3.0e-5, production Dense_9.w]
WG_EPS_B = 2e-6             # [5.3e-7, production Dense_9.b]
WG_EPS2_W = 3e-4            # [1.7e-4, production Dense_9.w; <= 4.3e-5 for every other kernel]
WG_EPS2_B = 1e-5            # [5.6e-6, the sigma-noise case's Dense_8.b: a scalar sum with cancellation]
# a left-out tile must move the reference by at least this multiple of the tensor's bar (every case but the
# production step, where one of ~6 200 tiles moves Dense_0.w by 5e-4 relative: 1.7x its bar; recorded, not asserted)
SENSITIVITY = 10.0
CHUNK_TILES = 256           # tiles of one reference chunk (32 Ki rows: ~2 GB of fp64 temporaries)


def _params(sh_deg, seed):
    """two MLPs of the oracle's initialisation with biases, Dense_8 (sigma) scaled by 30 so that a good share of the
    samples is opaque and the gradient reaches every layer (as in test_train.py)."""
    from oracle import nerf_sh_oracle as O
    K = L.K_of(sh_deg)
    w_off, _, _ = L.flat_offsets(K)
    out = []
    for s in (seed, seed + 1):
        f = O.init_flat_params(sh_deg, s, bias_scale=0.05)
        f[w_off[8]:w_off[8] + 256] *= 30.0
        out.append(f)
    return out


class Case:
    # sparsity_weight: 100x the training default, so that the sparsity rows (which ride in the last tiles of the last
    # level) carry gradients of the same order as the ray samples and a lost sparsity tile is visible in every tensor
    # sp_radius: the sparsity points are drawn in [-sp_radius, sp_radius]^3 (train.py's sparsity_radius)
    def __init__(self, sh, R, nc, nf, nsp, noise=False, seed=17, sparsity_weight=0.1, sp_radius=1.5):
        self.sh, self.R, self.nc, self.nf, self.nsp, self.noise = sh, R, nc, nf, nsp, noise
        self.seed, self.sparsity_weight, self.sp_radius = seed, sparsity_weight, sp_radius

    @property
    def name(self):
        return (f"sh{self.sh}_R{self.R}_{self.nc}+{self.nf}_nsp{self.nsp}" + ("_noise" if self.noise else "")
                + (f"_r{self.sp_radius:g}" if self.sp_radius != 1.5 else ""))

    def inputs(self, n):
        from plenoctree_b200.nerf.rays import random_rays_np
        o, d, v, px = random_rays_np(n, self.seed)
        rs = np.random.RandomState(self.seed + 1)
        t_rand = rs.uniform(0, 1, size=(n, self.nc)).astype(np.float32)
        u = rs.uniform(0, 1, size=(n, self.nf)).astype(np.float32) if self.nf else None
        r = self.sp_radius
        sp = rs.uniform(-r, r, size=(self.nsp, 3)).astype(np.float32) if self.nsp else None
        noise = None
        if self.noise:
            noise = (rs.normal(size=(n, self.nc)).astype(np.float32) * 0.5,
                     rs.normal(size=(n, self.nc + self.nf)).astype(np.float32) * 0.5 if self.nf else None)
        return (o, d, v, px), t_rand, u, sp, noise

    def model(self, max_rays=None):
        from plenoctree_b200.nerf.models import NerfModel
        m = NerfModel(sh_deg=self.sh, num_coarse_samples=self.nc, num_fine_samples=self.nf,
                      max_rays=max_rays or self.R, sparsity_npoints=self.nsp)
        fc, ff = _params(self.sh, self.seed)
        m.set_params(np.concatenate([fc, ff]) if self.nf else fc)
        return m

    def run(self, model, n=None, fill=None):
        """one loss_and_grad call over n rays on the model's workspace (pre-filled with byte `fill` if given)."""
        from plenoctree_b200.nerf import train as T
        from plenoctree_b200.nerf.models import Rays
        n = n or self.R
        (o, d, v, px), t_rand, u, sp, noise = self.inputs(n)
        state = T.TrainState(model)
        if fill is not None:
            model.workspace(True).fill_(fill)
        T.loss_and_grad(model, state, {"rays": Rays(o, d, v), "pixels": px},
                        sparsity_weight=self.sparsity_weight if self.nsp else 0.0, sparsity_length=0.05,
                        randomized=True, t_rand=t_rand, u=u, sp_points=sp, sigma_noise=noise)
        torch.cuda.synchronize()
        return state, dict(rays=(o, d, v), sp=sp, noise=noise, n=n)


def _ulp16_log2(x):
    """fp16 ulp at |x| (fp64 tensor); 2^-24 in the subnormal range."""
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14))) - 10)


def _sh_basis(deg, v):
    """real SH basis of the reference (sh.py; common.cuh: sh_basis) in fp64, v [n, 3] -> [n, K]."""
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    b = [torch.full_like(x, 0.28209479177387814)]
    if deg > 0:
        b += [-0.4886025119029199 * y, 0.4886025119029199 * z, -0.4886025119029199 * x]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        b += [1.0925484305920792 * xy, -1.0925484305920792 * yz, 0.31539156525252005 * (2 * zz - xx - yy),
              -1.0925484305920792 * xz, 0.5462742152960396 * (xx - yy)]
    if deg > 2:
        b += [-0.5900435899266435 * y * (3 * xx - yy), 2.890611442640554 * xy * z,
              -0.4570457994644658 * y * (4 * zz - xx - yy), 0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy),
              -0.4570457994644658 * x * (4 * zz - xx - yy), 1.445305721320277 * z * (xx - yy),
              -0.5900435899266435 * x * (xx - 3 * yy)]
    if deg > 3:
        b += [2.5033429417967046 * xy * (xx - yy), -1.7701307697799304 * yz * (3 * xx - yy),
              0.9461746957575601 * xy * (7 * zz - 1), -0.6690465435572892 * yz * (7 * zz - 3),
              0.10578554691520431 * (zz * (35 * zz - 30) + 3), -0.6690465435572892 * xz * (7 * zz - 3),
              0.47308734787878004 * (xx - yy) * (7 * zz - 1), -1.7701307697799304 * xz * (xx - 3 * yy),
              0.6258357354491761 * (xx * (xx - 3 * yy) - yy * (3 * xx - yy))]
    return torch.stack(b, 1)


class Stats:
    """running maxima, minima and counts of one level's stage checks"""

    def __init__(self):
        self.d = {}

    def max(self, key, val):
        val = float(val)
        self.d[key] = max(self.d.get(key, float("-inf")), val)

    def min(self, key, val):
        self.d[key] = min(self.d.get(key, float("inf")), float(val))

    def add(self, key, val):
        self.d[key] = self.d.get(key, 0) + int(val)


def _gemm_excess(got16, ref, mag):
    """error of the stored fp16 value beyond its rounding, in units of 2^-24 * mag (fp64 tensors).  The rounding is
    half an fp16 ulp, or one whole subnormal step (2^-24) below 2^-14: there the loss-scaled gradients of the data
    gradient chain land on either neighbour of the exact value (measured up to 0.5003 steps from it while the fp32
    sum is within 2^-24 * mag of it), so a tie of the fp16 grid is no evidence either way."""
    got = got16.double()
    big = torch.maximum(ref.abs(), got.abs())
    err = (got - ref).abs() - torch.where(big < 2.0 ** -14, U24, 0.5 * _ulp16_log2(big))
    return (err.clamp_min(0) / (U24 * mag).clamp_min(1e-300)).max()


def _check_level(ws, lv, flat, grad, case, ctx, st, lvl_idx, last_level):
    """stages A (saving forward), B (data gradient) and C (weight gradient + reduce) of one level."""
    dev = ws.device
    K = L.K_of(case.sh)
    NH = L.heads_width(K)
    C3 = 3 * K
    w_off, b_off, P = L.flat_offsets(K)
    dims = L.layer_dims(K)
    scale = ctx["loss_scale"]
    fl = torch.from_numpy(flat).to(dev)
    # fp16 operands ("hi" images of pack_weights; the biases travel through the tensor cores in fp16 too)
    W = [fl[w_off[l]:w_off[l] + dims[l][0] * 256].view(dims[l][0], 256).half().double() for l in range(8)]
    B = [fl[b_off[l]:b_off[l] + 256].half().double() for l in range(8)]
    Wh_np, bh_np = L.heads_matrix(flat, K)
    Wh = torch.from_numpy(Wh_np).to(dev).half().double()       # [256, NH]
    bh = torch.from_numpy(bh_np).to(dev).half().double()
    cols9 = torch.tensor([L.heads_column(K, o) for o in range(C3)], device=dev)

    N, M, Mr, rows, tiles = lv["N"], lv["M"], lv["M_rays"], lv["rows"], lv["tiles"]
    z = L.workspace_view(ws, lv, "z").reshape(-1)
    rgbs = L.workspace_view(ws, lv, "rgbs")
    G = L.workspace_view(ws, lv, "G")
    H, E, DZ, DO = (L.workspace_view(ws, lv, k) for k in ("H", "E", "DZ", "DO"))
    MASK = L.workspace_view(ws, lv, "mask")
    o, d, v = (torch.from_numpy(a).to(dev) for a in ctx["rays"])
    sp = torch.from_numpy(ctx["sp"]).to(dev) if (ctx["sp"] is not None and last_level and M > Mr) else None
    noise = None
    if ctx["noise"] is not None and ctx["noise"][lvl_idx] is not None:
        noise = torch.from_numpy(ctx["noise"][lvl_idx]).to(dev).reshape(-1)

    # weight-gradient references: fp64 sums over all padded rows and their |a*b| sums; per-tile contributions of the
    # last tile holding a real sample and of one in the middle (sensitivity guard)
    real_tiles = (M + L.TILE_M - 1) // L.TILE_M
    probe = sorted({real_tiles - 1, (Mr + L.TILE_M - 1) // L.TILE_M - 1, real_tiles // 2})
    shapes = {**{f"w{l}": (dims[l][0], 256) for l in range(8)}, **{f"b{l}": (256,) for l in range(8)},
              "wh": (256, NH), "bh": (NH,)}
    acc = {k: torch.zeros(s, dtype=torch.float64, device=dev) for k, s in shapes.items()}
    mag = {k: torch.zeros(s, dtype=torch.float64, device=dev) for k, s in shapes.items()}
    tile_d = {t: {k: torch.zeros(s, dtype=torch.float64, device=dev) for k, s in shapes.items()} for t in probe}

    def wsum(key, a, b, r0):
        """acc[key] += a^T b over the chunk's rows (a, b fp64 [n, *]); b None: column sums of a."""
        if b is None:
            acc[key] += a.sum(0)
            mag[key] += a.abs().sum(0)
        else:
            acc[key] += a.T @ b
            mag[key] += a.abs().T @ b.abs()
        for t in probe:
            lo = t * L.TILE_M - r0
            if 0 <= lo < a.shape[0]:
                aa = a[lo:lo + L.TILE_M]
                tile_d[t][key] += aa.sum(0) if b is None else aa.T @ b[lo:lo + L.TILE_M]

    for t0 in range(0, tiles, CHUNK_TILES):
        t1 = min(tiles, t0 + CHUNK_TILES)
        r0, r1 = t0 * L.TILE_M, t1 * L.TILE_M
        s = torch.arange(r0, r1, device=dev)
        real = s < M
        sc = s.clamp_max(M - 1)                      # load_point clamps the row: padded rows repeat row M-1
        e16 = L.decode_e(E[t0:t1])
        h16 = [L.decode_h(H[t0:t1], l) for l in range(8)]
        dz16 = [L.decode_dz(DZ[t0:t1], l) for l in range(8)]
        do16 = L.decode_do(DO[t0:t1])
        mask = [L.decode_mask(MASK[l, r0:r1]) for l in range(8)]

        # ---------------- A. saving forward ----------------
        ray = (sc // N).clamp_max(ctx["n"] - 1)
        x = o[ray] + z[sc.clamp_max(Mr - 1)][:, None] * d[ray]          # fp32: separate multiply and add
        if sp is not None:
            x = torch.where((sc >= Mr)[:, None], sp[(sc - Mr).clamp_min(0)], x)
        st.add("posenc_xyz_bit_mismatches", (e16[:, :3].view(torch.int16) != x.half().view(torch.int16)).sum())
        st.add("posenc_col63_not_one", (e16[:, 63] != 1).sum())
        j = torch.arange(10, device=dev, dtype=torch.float32)
        xb = (x[:, None, :] * torch.exp2(j)[None, :, None]).reshape(-1, 30)          # j-major, exact
        arg = torch.cat([xb, xb + torch.tensor(np.float32(np.pi / 2), device=dev)], 1)   # fp32 add
        ref_sin = torch.sin(arg.double())
        err = (e16[:, 3:63].double() - ref_sin.half().double()).abs()
        st.max("posenc_sin_err_ulps", (err / _ulp16_log2(ref_sin)).max())
        st.max("posenc_sin_err_abs", err.max())
        st.max("posenc_sin_excess", ((err - _ulp16_log2(ref_sin)).clamp_min(0) / SIN_ABS).max())
        e63 = e16[:, :63].double()
        hd = [h.double() for h in h16]
        for l in range(8):
            a = e63 if l == 0 else (torch.cat([hd[4], e63], 1) if l == 5 else hd[l - 1])
            pre = a @ W[l] + B[l]
            amag = a.abs() @ W[l].abs() + B[l].abs()
            ref = pre.clamp_min(0)
            st.max("fwd_excess", _gemm_excess(h16[l], ref, amag))
            st.add("fwd_fp16_bit_mismatches", (ref.half().view(torch.int16) != h16[l].view(torch.int16)).sum())
            st.add("mask_mismatches", (mask[l] != (h16[l] != 0)).sum())
            st.add("h_nonfinite", (~torch.isfinite(h16[l])).sum())
        heads = hd[7] @ Wh + bh
        hmag = hd[7].abs() @ Wh.abs() + bh.abs()
        rr = s[real]
        got = rgbs[r0:r0 + rr.numel()].double()
        sig = heads[real, 0]
        sig_tol = FWD_ALLOW * U24 * hmag[real, 0]
        if noise is not None:
            nz = torch.where(rr < Mr, noise[rr.clamp_max(Mr - 1)].double(), torch.zeros_like(sig))
            sig = sig + nz
            sig_tol = sig_tol + U24 * sig.abs()
        st.max("rgbs_sigma_excess", ((got[:, 3] - sig.clamp_min(0)).abs() / sig_tol.clamp_min(1e-300)).max())
        onray = rr < Mr
        if onray.any():
            Y = _sh_basis(case.sh, v[(rr[onray] // N)].double()) if case.sh >= 0 else \
                torch.ones(int(onray.sum()), 1, dtype=torch.float64, device=dev)
            hr = heads[real][onray][:, 1:1 + C3].view(-1, K, 3)
            hm = hmag[real][onray][:, 1:1 + C3].view(-1, K, 3)
            prer = (Y[:, :, None] * hr).sum(1)
            tol = 0.25 * ((Y.abs()[:, :, None] * (FWD_ALLOW * U24 * hm + 4 * U24 * hr.abs())).sum(1)) + 2 ** -21
            err = (got[onray, :3] - torch.sigmoid(prer)).abs()
            st.max("rgbs_rgb_excess", (err / tol).max())

        # ---------------- B. data gradient ----------------
        g = torch.zeros(r1 - r0, 4, dtype=torch.float32, device=dev)
        g[:int(real.sum())] = G[r0:r0 + int(real.sum())]
        st.add("dO_sigma_bit_mismatches", (do16[:, 0].view(torch.int16) != g[:, 3].half().view(torch.int16)).sum())
        ray_rows = s < Mr
        Yall = torch.zeros(r1 - r0, K, dtype=torch.float64, device=dev)
        if ray_rows.any():
            Yall[ray_rows] = (_sh_basis(case.sh, v[s[ray_rows] // N].double()) if case.sh >= 0 else 1.0)
        ref_do = (g[:, None, :3].double() * Yall[:, :, None]).reshape(-1, C3)
        err = (do16[:, 1:1 + C3].double() - ref_do).abs()
        st.max("dO_rgb_err_ulps", (err / _ulp16_log2(ref_do)).max())
        st.add("dO_free_or_padded_rgb_nonzero", (do16[~ray_rows, 1:1 + C3] != 0).sum())
        st.add("dO_padded_sigma_nonzero", (do16[~real, 0] != 0).sum())
        st.add("dO_pad_columns_nonzero", (do16[:, 1 + C3:64 * ((NH + 63) // 64)] != 0).sum())
        dod = do16[:, :NH].double()
        dzd = [x.double() for x in dz16]
        for l in range(7, -1, -1):
            a, Wt = (dod, Wh.T) if l == 7 else (dzd[l + 1], W[l + 1][:256].T)
            ref = (a @ Wt) * mask[l]
            amag = (a.abs() @ Wt.abs()) * mask[l]
            st.max("bwd_excess", _gemm_excess(dz16[l], ref, amag))
            st.add("dz_nonzero", (dz16[l] != 0).sum())
            st.add("dz_subnormal", ((dz16[l] != 0) & (dz16[l].abs() < 2 ** -14)).sum())
            st.add("bwd_fp16_bit_mismatches", (ref.half().view(torch.int16) != dz16[l].view(torch.int16)).sum())
            bits = dz16[l].view(torch.int16)
            st.add("dz_masked_nonzero_bits", (bits[~mask[l]] != 0).sum())
            st.add("dz_padded_nonzero_bits", (bits[~real] != 0).sum())
            st.add("dz_nonfinite", (~torch.isfinite(dz16[l])).sum())
            st.max("dz_headroom", dz16[l].abs().max() / 65504.0)

        # ---------------- C. weight-gradient sums ----------------
        for l in range(1, 8):
            wsum(f"w{l}", hd[l - 1] if l != 5 else torch.cat([hd[4], e63], 1), dzd[l], r0)
        wsum("w0", e63, dzd[0], r0)
        for l in range(8):
            wsum(f"b{l}", dzd[l], None, r0)
        wsum("wh", hd[7], dod, r0)
        wsum("bh", dod, None, r0)

    # reference tensors in flat (flax) order, over the loss scale
    def flat_of(dct):
        out = torch.zeros(P, dtype=torch.float64, device=dev)
        for l in range(8):
            out[w_off[l]:w_off[l] + dims[l][0] * 256] = dct[f"w{l}"].reshape(-1)
            out[b_off[l]:b_off[l] + 256] = dct[f"b{l}"]
        out[w_off[8]:w_off[8] + 256] = dct["wh"][:, 0]
        out[w_off[9]:w_off[9] + 256 * C3] = dct["wh"][:, cols9].reshape(-1)
        out[b_off[8]] = dct["bh"][0]
        out[b_off[9]:b_off[9] + C3] = dct["bh"][cols9]
        return out / scale

    ref, rmag = flat_of(acc), flat_of(mag)
    deltas = {t: flat_of(tile_d[t]) for t in probe}
    gg = grad.double()
    report = {}
    for l in range(10):
        for nm, a, n in (("w", w_off[l], dims[l][0] * dims[l][1]), ("b", b_off[l], dims[l][1])):
            sl = slice(a, a + n)
            err = (gg[sl] - ref[sl]).abs()
            eps, eps2 = (WG_EPS_B, WG_EPS2_B) if nm == "b" else (WG_EPS_W, WG_EPS2_W)
            elem = float((err / rmag[sl].clamp_min(1e-300)).max())
            rnorm = float(ref[sl].norm())
            rel = float(err.norm() / max(rnorm, 1e-300))
            # sensitivity: leaving out a real tile the tensor depends on (the last tile with a sample, the last with a
            # ray sample, a middle one; a sparsity-only tile does not reach the rgb heads) moves the reference by
            # >= SENSITIVITY x the bar
            sens = min([max(float((deltas[t][sl].abs() / (eps * rmag[sl]).clamp_min(1e-300)).max()),
                            float(deltas[t][sl].norm()) / max(rnorm, 1e-300) / eps2)
                        for t in probe if bool((deltas[t][sl] != 0).any())] or [0.0])
            report[f"Dense_{l}.{nm}"] = dict(max_err_over_abs_sum=elem, rel_l2=rel, bars=(eps, eps2), sensitivity=sens)
    for k, r in report.items():
        st.max("wgrad_max_err_over_abs_sum", r["max_err_over_abs_sum"])
        st.max("wgrad_rel_l2", r["rel_l2"])
        st.max("wgrad_sensitivity_min_neg", -r["sensitivity"])
    return report


def _check_all(case, model, state, ctx, sparsity_on):
    from plenoctree_b200.nerf.train import default_loss_scale
    ws = model.workspace(True)
    views = L.train_workspace_views(model.cfg, ctx["n"], sparsity_on)
    assert views["total"] == ws.numel()
    ctx["loss_scale"] = default_loss_scale(ctx["n"])
    params = model.params.cpu().numpy()
    out = {}
    for i, lv in enumerate(views["levels"]):
        st = Stats()
        P = model.P
        rep = _check_level(ws, lv, params[i * P:(i + 1) * P], state.grads[i * P:(i + 1) * P], case, ctx, st, i,
                           i == len(views["levels"]) - 1)
        out[f"MLP_{i}"] = dict(stages=st.d, wgrad=rep, M=lv["M"], tiles=lv["tiles"])
    return out


def _assert_stages(res, guard=True):
    for mlp, r in res.items():
        s = r["stages"]
        for k in ("posenc_xyz_bit_mismatches", "posenc_col63_not_one", "mask_mismatches", "h_nonfinite",
                  "dO_sigma_bit_mismatches", "dO_free_or_padded_rgb_nonzero", "dO_padded_sigma_nonzero",
                  "dO_pad_columns_nonzero", "dz_masked_nonzero_bits", "dz_padded_nonzero_bits", "dz_nonfinite"):
            assert s[k] == 0, (mlp, k, s[k])
        assert s["posenc_sin_excess"] <= 1.0, (mlp, s)
        assert s["fwd_excess"] <= FWD_ALLOW, (mlp, s["fwd_excess"])
        assert s["rgbs_sigma_excess"] <= 1.0, (mlp, s["rgbs_sigma_excess"])
        assert s.get("rgbs_rgb_excess", 0.0) <= 1.0, (mlp, s["rgbs_rgb_excess"])
        assert s["dO_rgb_err_ulps"] <= 1.0, (mlp, s["dO_rgb_err_ulps"])
        assert s["bwd_excess"] <= BWD_ALLOW, (mlp, s["bwd_excess"])
        assert s["dz_headroom"] < 1.0
        for name, w in r["wgrad"].items():
            assert w["max_err_over_abs_sum"] <= w["bars"][0], (mlp, name, w)
            assert w["rel_l2"] <= w["bars"][1], (mlp, name, w)
            if guard:
                assert w["sensitivity"] >= SENSITIVITY, (mlp, name, w)


CASES = [
    Case(3, 96, 64, 128, 300),                                   # the shape test_train.py uses
    *[Case(sh, 40, 64, 128, 64) for sh in (-1, 0, 1, 2, 4)],     # every heads width: NH 16/16/16/32/80
    Case(3, 64, 64, 0, 0), Case(3, 64, 64, 0, 200),              # single level; sparsity rows on MLP_0
    Case(3, 1, 3, 0, 0), Case(3, 1, 3, 0, 1), Case(3, 1, 3, 5, 0), Case(3, 1, 3, 5, 1),   # one real tile
    Case(3, 8, 64, 0, 0), Case(3, 8, 64, 0, 1),                  # M = 512 exactly, and 513
    Case(3, 32, 64, 192, 64),                                    # N = 256
    Case(3, 64, 64, 128, 0, noise=True),                         # noised sigma in the rgbs epilogue
]


def _stage_case(case, guard=True):
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    model = case.model()
    state, ctx = case.run(model, fill=0xFF)      # NaN in every byte the call does not write
    res = _check_all(case, model, state, ctx, case.nsp > 0)
    res["wall_s"] = time.time() - t0
    res["peak_alloc_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    _record(case.name, res)
    _assert_stages({k: v for k, v in res.items() if k.startswith("MLP")}, guard)

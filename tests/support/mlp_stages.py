"""The training MLP against fp64, stage by stage: cases, inputs, models, the one stage checker of fp16 and fp16x3 for
every model flag, and its bars."""
import copy
import time

import numpy as np
import torch

from oracle import net_activation_oracle as NA, posenc_oracle as PO
from plenoctree_b200 import layouts as L
from tests.support.model_flags import SP_BAR, SP_FLOOR, _act64, _ref_features, softplus64

FP16, X3 = 1, 3


def _setup(sh_deg, R, nf, nsp, seed):
    """the oracle's inputs of one training call: params(sh_deg, seed), rays, pixels and the draws"""
    fc, ff = params(sh_deg, seed)
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

# ---- bars, per precision.  Forward / data-gradient GEMMs: error beyond the rounding of the stored value (fp16: half an
# fp16 ulp; fp16x3: the representation error of hi + lo), in units of 2^-24 * sum_k |a_k w_k|.  An x3 bar must stay at
# least 2^7 below fp16's operand rounding (2^-11 = 2^13 units), or the mode is not what it claims.  The largest value
# measured on an H100 80 GB HBM3 in brackets (fp16; fp16x3): over the cases of test_train_stages.py at a 400 W power
# limit (fp16), of test_train_x3.py at 400 W (fp16x3), and of test_net_activation.py and test_flag_matrix.py at 700 W
# (DO_ALLOW, SIN_ALLOW's fp16x3 value).
FWD_ALLOW = {FP16: 8.0, X3: 32.0}            # [3.74; 16.2]
BWD_ALLOW = {FP16: 12.0, X3: 32.0}           # [6.35, production step; 22.1]
# fp16x3 dZ entries whose contraction reads an fp16-subnormal operand (|a| < 2^-14 in the loss-scaled chain: hi then
# carries fewer than 11 bits and lo is 0): the tensor cores' fp32 sum is up to ~390 units from fp64 there (coarse MLP
# of the production step), so those rows are held to this bar instead of BWD_ALLOW.  fp16 sets no such rows apart.
BWD_SUBNORMAL_ALLOW = {FP16: BWD_ALLOW[FP16], X3: 512.0}    # [6.35; 391]
# positional encoding: xyz columns bit-exact; sine columns against fp64 of the kernel's fp32 arguments.  fp16: beyond
# one fp16 ulp, in units of the reduced SFU sine's absolute error SIN_ABS = 2^-20; fp16x3: hi + lo beyond lo's
# representation error, in units of 2^-24 (|sin| <= 1)
SIN_ABS = 2.0 ** -20
SIN_ALLOW = {FP16: 1.0, X3: 3.0}             # [0.5; 1.41]
# dO's rgb columns (the fp32 product G.rgb * Y_k with the fp32 SH basis, stored in fp16 or hi + lo) beyond the rounding
# of the stored value, in units of 2^-24 * |G.rgb|.  With the relu trunk, fp16 dO is also within one fp16 ulp of fp64
# (dO_rgb_err_ulps); the production step with an elu or a tanh trunk reaches 1.07 ulp, fp16x3 1.27 (recorded only)
DO_ALLOW = {FP16: 6.0, X3: 6.0}              # [1.74; 2.84]
# weight gradient + reduce, per tensor: max |err| <= WG_EPS_W / WG_EPS_B * sum_s |a_s b_s| and, at fp16, relative L2
# <= WG_EPS2_W / WG_EPS2_B (kernels / biases).  The kernels' error grows with the tiles one CTA sums in fp32 (~1 200 per
# Dense_0 CTA in the production step).  At fp16x3 the relative L2 is recorded, and WG_EPS2 only scales the recorded
# sensitivity: the scalar Dense_8.b of an fp16x3 flag-matrix row (elu trunk, softplus density, noise) reaches 5.3e-5
# relative, a sum with cancellation, while its max |err| / sum |a b| is 5.1e-9
WG_EPS_W = {FP16: 1e-4, X3: 1e-4}            # [3.0e-5, production Dense_9.w; 1.9e-5]
WG_EPS_B = {FP16: 2e-6, X3: 2e-6}            # [5.3e-7, production Dense_9.b; 2.5e-7]
WG_EPS2_W = {FP16: 3e-4, X3: 3e-4}           # [1.7e-4, production Dense_9.w, <= 4.3e-5 for every other kernel]
WG_EPS2_B = {FP16: 1e-5, X3: 1e-5}           # [5.6e-6, the sigma-noise case's Dense_8.b]
ACT_BOUND = 4.0             # a smooth trunk activation's fp32 error, in units of 2^-24 * |f(z)| (kernels.h: net_act_f32)
# a left-out tile must move the weight-gradient reference by at least this multiple of the tensor's bar (asserted under
# guard: the fp16 cases with the default flags but the production step, where one of ~6 200 tiles moves Dense_0.w by
# 5e-4 relative, 1.7x its bar)
SENSITIVITY = 10.0
CHUNK_TILES = 128           # tiles of one reference chunk (16 Ki rows)

# End to end (fp16x3).  The loss statistics within LOSS_REL of the fp64 oracle.  The gradient (and a six-step Adam
# update) against two oracles on the same inputs: fp64, and the oracle evaluated in fp32 (the reference's own
# precision).  The fp32 oracle is itself some 5e-4 (relative L2) from fp64 on these inputs: fp32 sample positions
# o + t d, amplified up to 2^9 by the positional encoding.  No fp32-class step can come closer to fp64 than that, so the
# x3 step must sit at that floor (within FLOOR_SLACK of the fp32 oracle's distance to fp64) and be GRAD_GAIN times
# closer to the fp32 oracle than the fp16 step is.
LOSS_REL = 1e-5             # [1.5e-6]
GRAD_GAIN = 10.0            # [780x gradient, 21x six-step update]
FLOOR_SLACK = 1.1           # [1.000 gradient, 0.995 update]


def params(sh_deg, seed, pe=PO.DEFAULT):
    """two MLPs of the oracle's initialisation for encoder pe (seeds seed, seed + 1) with biases, Dense_8 (sigma)
    scaled by 30 so that a good share of the samples is opaque and the gradient reaches every layer (as in
    test_train.py)."""
    w_off = L.flat_offsets(L.K_of(sh_deg), PO.width(pe))[0]
    out = []
    for s in (seed, seed + 1):
        f = PO.init_flat_params(sh_deg, s, bias_scale=0.05, pe=pe)
        f[w_off[8]:w_off[8] + 256] *= 30.0
        out.append(f)
    return out


def _centre_sigma(flat, sh, act, pe=PO.DEFAULT):
    """centre every trunk layer's pre-activations and raw sigma over the scene box (each bias minus the mean, raw
    sigma's minus the median), the state a trained network sits in.  With the relu trunk's initial parameters a
    softplus trunk's pre-activations drift up layer by layer (softplus >= 0 adds a common positive part) until raw
    sigma is negative everywhere: an empty scene, a zero gradient."""
    _, b_off, _ = L.flat_offsets(L.K_of(sh), PO.width(pe))
    box = torch.from_numpy(np.random.RandomState(5).uniform(-1.5, 1.5, (4000, 3)).astype(np.float32))
    f = NA.activation(act)
    with torch.no_grad():
        p = PO.unflatten(flat, sh, pe)
        enc = PO.encode(box, pe)
        h = enc
        for i in range(8):
            z = h @ p[i][0] + p[i][1]
            shift = z.mean(0).numpy().astype(np.float32)
            flat[b_off[i]:b_off[i] + 256] -= shift
            h = f(z - torch.from_numpy(shift))
            if i == 4:
                h = torch.cat([h, enc], -1)
        _, sig = NA.mlp(PO.unflatten(flat, sh, pe), enc, act)
    flat[b_off[8]] -= np.float32(np.median(sig.numpy()))


class Case:
    """one training call: its shape, draws and model flags.
    sparsity_weight: 100x the training default, so that the sparsity rows (which ride in the last tiles of the last
    level) carry gradients of the same order as the ray samples and a lost sparsity tile is visible in every tensor.
    sp_radius: the sparsity points are drawn in [-sp_radius, sp_radius]^3 (train.py's sparsity_radius).
    centre: the parameters pass through _centre_sigma (the flag-model cases)."""

    def __init__(self, sh, R, nc, nf, nsp, noise=False, seed=17, sparsity_weight=0.1, sp_radius=1.5, precision=FP16,
                 act="relu", pe=PO.DEFAULT, sigma_act="relu", centre=False, white=True, lindisp=False):
        self.sh, self.R, self.nc, self.nf, self.nsp, self.noise = sh, R, nc, nf, nsp, noise
        self.seed, self.sparsity_weight, self.sp_radius = seed, sparsity_weight, sp_radius
        self.precision, self.act, self.pe, self.sigma_act, self.centre = precision, act, pe, sigma_act, centre
        self.white, self.lindisp = white, lindisp

    @property
    def name(self):
        return (f"sh{self.sh}_R{self.R}_{self.nc}+{self.nf}_nsp{self.nsp}" + ("_noise" if self.noise else "")
                + (f"_r{self.sp_radius:g}" if self.sp_radius != 1.5 else ""))

    def replace(self, **kw):
        """a copy of the case with the attributes kw changed"""
        c = copy.copy(self)
        c.__dict__.update(kw)
        return c

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
        mn, mx, legacy = self.pe
        m = NerfModel(sh_deg=self.sh, num_coarse_samples=self.nc, num_fine_samples=self.nf, white_bkgd=self.white,
                      lindisp=self.lindisp, max_rays=max_rays or self.R, sparsity_npoints=self.nsp,
                      net_activation=self.act, sigma_activation=self.sigma_act, min_deg_point=mn, max_deg_point=mx,
                      legacy_posenc_order=legacy)
        fc, ff = params(self.sh, self.seed, self.pe)
        if self.centre:
            for f in (fc, ff):
                _centre_sigma(f, self.sh, self.act, self.pe)
        m.set_params(np.concatenate([fc, ff]) if self.nf else fc)
        return m

    def run(self, model, n=None, fill=None, z_fine=None, inputs=None):
        """one loss_and_grad call at the case's precision over n rays on the model's workspace (pre-filled with byte
        `fill` if given)."""
        from plenoctree_b200.nerf import train as T
        from plenoctree_b200.nerf.models import Rays
        n = n or self.R
        (o, d, v, px), t_rand, u, sp, noise = inputs or self.inputs(n)
        state = T.TrainState(model)
        if fill is not None:
            model.workspace(True, self.precision).fill_(fill)
        T.loss_and_grad(model, state, {"rays": Rays(o, d, v), "pixels": px},
                        sparsity_weight=self.sparsity_weight if self.nsp else 0.0, sparsity_length=0.05,
                        randomized=True, t_rand=t_rand, u=u, sp_points=sp, sigma_noise=noise, z_fine=z_fine,
                        precision=self.precision)
        torch.cuda.synchronize()
        return state, dict(rays=(o, d, v), sp=sp, noise=noise, n=n, t_rand=t_rand, u=u)


def ulp16(x):
    """fp16 ulp at |x| (fp64 tensor), 2^-24 in the subnormal range.  The exponent comes from frexp: log2 on the GPU is
    not exact at every power of two (log2(8) < 3 there), which would halve the ulp of 8, 64, ..."""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -14))
    return torch.ldexp(torch.ones_like(x), (e - 11).to(torch.int64))


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


def operands(flat, K, dev, x3, enc_width=L.ENC_DIM):
    """fp64 images of the operands pack_weights makes (hi; fp16x3: + pack_wt_lo's lo): W[l] [in, 256], B[l],
    Wh [256, NH], bh [NH].  The biases travel through the tensor cores in fp16 too."""
    w_off, b_off, _ = L.flat_offsets(K, enc_width)
    dims = L.layer_dims(K, enc_width)
    fl = torch.from_numpy(flat).to(dev)

    def hl(x):
        return x.half().double() + ((x - x.half().float()).half().double() if x3 else 0.0)
    W = [hl(fl[w_off[l]:w_off[l] + dims[l][0] * 256].view(dims[l][0], 256)) for l in range(8)]
    B = [hl(fl[b_off[l]:b_off[l] + 256]) for l in range(8)]
    Wh_np, bh_np = L.heads_matrix(flat, K, enc_width)
    return W, B, hl(torch.from_numpy(Wh_np).to(dev)), hl(torch.from_numpy(bh_np).to(dev))


def excess(hi, lo, ref, amag, x3, extra=0.0):
    """error of the stored value hi (+ lo) beyond its rounding and `extra`, in units of 2^-24 * amag (fp64 tensors).
    fp16x3: the representation error of hi + lo, half an ulp of lo (2^-25 once lo is subnormal).  fp16: half an fp16
    ulp, or one whole subnormal step (2^-24) below 2^-14: there the loss-scaled gradients of the data gradient chain
    land on either neighbour of the exact value (measured up to 0.5003 steps from it while the fp32 sum is within
    2^-24 * mag of it), so a tie of the fp16 grid is no evidence either way."""
    got = hi.double() + lo.double()
    if x3:
        rnd = 0.5 * ulp16(lo.double())
    else:
        big = torch.maximum(ref.abs(), got.abs())
        rnd = torch.where(big < 2.0 ** -14, U24, 0.5 * ulp16(big))
    err = (got - ref).abs() - rnd - extra
    return float((err.clamp_min(0) / (U24 * amag).clamp_min(1e-300)).max())


def _split_violations(hi, lo):
    """pairs with |lo| > half an ulp of hi, or lo != 0 where hi = 0"""
    return int(((lo.double().abs() > 0.5 * ulp16(hi.double()) * (hi != 0)) | ((hi == 0) & (lo != 0))).sum())


def _sin_excess(e_hi, e_lo, ref, x3):
    """sine columns against fp64 of the kernel's fp32 arguments, in SIN_ALLOW's units"""
    if x3:
        err = (e_hi.double() + e_lo.double() - ref).abs() - 0.5 * ulp16(e_lo.double())
        return float((err.clamp_min(0) / U24).max())
    err = (e_hi.double() - ref.half().double()).abs()
    return float(((err - ulp16(ref)).clamp_min(0) / SIN_ABS).max())


def _grad_of_output(act, h):
    """fp64 f'(z) from h = f(z) (kernels.h: net_act_grad_of_output)"""
    if act == "elu":
        return torch.where(h > 0, torch.ones_like(h), h + 1.0)
    if act == "softplus":
        return -torch.expm1(-h)
    if act == "tanh":
        return (1.0 - h) * (1.0 + h)
    return (h > 0).double()


def _sigma_want(sig, onray, sigma_act):
    """the rgbs epilogue's density from fp64 raw sigma (+ noise): the model's activation on ray rows, relu on the
    free sparsity rows; and the extra allowance of softplus (test_sigma_activation.py: SP_BAR, SP_FLOOR)"""
    if sigma_act == "softplus":
        sp = softplus64(sig)
        return (torch.where(onray, sp, sig.clamp_min(0)),
                torch.where(onray, SP_BAR * U24 * sp + SP_FLOOR, torch.zeros_like(sig)))
    return sig.clamp_min(0), torch.zeros_like(sig)


def check_level(ws, lv, flat, grad, sh, scale, st, *, precision, call, act="relu", pe=PO.DEFAULT, sigma_act="relu",
                alt=None):
    """stages A (saving forward: posenc tile, trunk, rgbs epilogue), B (data gradient: dO, dZ) and C (weight gradient
    + reduce) of one level, each against fp64 whose inputs are the kernel's own previous-stage tiles: fp16 (its lo
    parts are zeros) or fp16x3 (hi + lo), for any encoder pe, trunk activation act and density sigma_act.  call: the
    rays, free points, noise and ray count of the training call.  alt: a flag replaced ({"pe", "act", "sigma_act"}):
    the same stages against the reference of the wrong flag, under guard_*.  Returns the weight-gradient report per
    tensor."""
    x3 = precision == X3
    alt = alt or {}
    dev = ws.device
    K = L.K_of(sh)
    NH = L.heads_width(K)
    C3 = 3 * K
    EW = PO.width(pe)
    relu = act == "relu"
    nd = 64 * ((NH + 63) // 64)                 # columns of the dO image mlp_bwd writes
    w_off, b_off, P = L.flat_offsets(K, EW)
    dims = L.layer_dims(K, EW)
    W, B, Wh, bh = operands(flat, K, dev, x3, EW)
    cols9 = torch.tensor([L.heads_column(K, o) for o in range(C3)], device=dev)
    N, M, Mr, tiles = lv["N"], lv["M"], lv["M_rays"], lv["tiles"]
    view = lambda k: L.workspace_view(ws, lv, k)
    images = {s: [view(k + s) for k in ("H", "E", "DZ", "DO")] for s in (("", "_lo") if x3 else ("",))}
    MASK, z, rgbs, G = view("mask"), view("z").reshape(-1), view("rgbs"), view("G")
    o, d, v = (torch.from_numpy(a).to(dev) for a in call["rays"])
    sp = torch.from_numpy(call["sp"]).to(dev) if call["sp"] is not None and M > Mr else None
    noise = torch.from_numpy(call["noise"]).to(dev).reshape(-1) if call["noise"] is not None else None

    # weight-gradient references: fp64 sums over all padded rows and their |a*b| sums; per-tile contributions of the
    # last tile holding a real sample, the last holding a ray sample and one in the middle (sensitivity guard)
    real_tiles = (M + L.TILE_M - 1) // L.TILE_M
    probe = sorted({real_tiles - 1, (Mr + L.TILE_M - 1) // L.TILE_M - 1, real_tiles // 2})
    shapes = {**{f"w{l}": (dims[l][0], 256) for l in range(8)}, **{f"b{l}": (256,) for l in range(8)},
              "wh": (256, NH), "bh": (NH,)}
    zeros = lambda: {k: torch.zeros(s, dtype=torch.float64, device=dev) for k, s in shapes.items()}
    acc, mag = zeros(), zeros()
    tile_d = {t: zeros() for t in probe}

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

    def bits(t):
        return t.view(torch.int16)

    def decode(s, t0, t1):
        H, E, DZ, DO = images[s]
        return ([L.decode_h(H[t0:t1], l) for l in range(8)], [L.decode_dz(DZ[t0:t1], l) for l in range(8)],
                L.decode_do(DO[t0:t1])[:, :nd], L.decode_e(E[t0:t1]))

    for t0 in range(0, tiles, CHUNK_TILES):
        t1 = min(tiles, t0 + CHUNK_TILES)
        r0, r1 = t0 * L.TILE_M, t1 * L.TILE_M
        s = torch.arange(r0, r1, device=dev)
        real = s < M
        h_hi, dz_hi, do_hi, e_hi = decode("", t0, t1)
        if x3:
            h_lo, dz_lo, do_lo, e_lo = decode("_lo", t0, t1)
        else:
            h_lo, dz_lo = [torch.zeros_like(x) for x in h_hi], [torch.zeros_like(x) for x in dz_hi]
            do_lo, e_lo = torch.zeros_like(do_hi), torch.zeros_like(e_hi)
        st.add("split_violations_e", _split_violations(e_hi, e_lo))
        st.add("split_violations_do", _split_violations(do_hi, do_lo))
        st.add("split_violations_h", sum(_split_violations(a, b) for a, b in zip(h_hi, h_lo)))
        st.add("split_violations_dz", sum(_split_violations(a, b) for a, b in zip(dz_hi, dz_lo)))
        eW = (e_hi.double() + e_lo.double())[:, :EW]
        hd = [a.double() + b.double() for a, b in zip(h_hi, h_lo)]

        # ---------------- A. saving forward ----------------
        # posenc tile: xyz bit-exact, sines against fp64 of the fp32 arguments, pad columns [W, 63) zero, col 63 the
        # constant one (lo 0)
        st.add("posenc_pad_nonzero_bits", int(((bits(e_hi[:, EW:63]) != 0) | (bits(e_lo[:, EW:63]) != 0)).sum()))
        st.add("posenc_col63_not_one", int(((e_hi[:, 63] != 1) | (e_lo[:, 63] != 0)).sum()))
        sc = s.clamp_max(M - 1)                      # load_point clamps the row: padded rows repeat row M-1
        ray = (sc // N).clamp_max(call["n"] - 1)
        x = o[ray] + z[sc.clamp_max(Mr - 1)][:, None] * d[ray]          # fp32: separate multiply and add
        if sp is not None:
            x = torch.where((sc >= Mr)[:, None], sp[(sc - Mr).clamp_min(0)], x)
        xh = x.half()
        st.add("posenc_xyz_bit_mismatches", int((bits(e_hi[:, :3]) != bits(xh)).sum()))
        if x3:
            st.add("posenc_xyz_bit_mismatches", int((bits(e_lo[:, :3]) != bits((x - xh.float()).half())).sum()))
        if EW > 3:
            ref_sin = _ref_features(x, pe)
            st.max("posenc_sin_excess", _sin_excess(e_hi[:, 3:EW], e_lo[:, 3:EW], ref_sin, x3))
            err = (e_hi[:, 3:EW].double() - ref_sin.half().double()).abs()
            st.max("posenc_sin_err_ulps", (err / ulp16(ref_sin)).max())
            st.max("posenc_sin_err_abs", err.max())
            if "pe" in alt:
                st.max("guard_posenc_sin", _sin_excess(e_hi[:, 3:EW], e_lo[:, 3:EW], _ref_features(x, alt["pe"]), x3))
        # trunk: h_l = f(pre) within the rounding of the stored value + f's fp32 bound + the GEMM allowance
        mask = [L.decode_mask(MASK[l, r0:r1]) for l in range(8)] if relu else None
        for l in range(8):
            a = eW if l == 0 else (torch.cat([hd[4], eW], 1) if l == 5 else hd[l - 1])
            pre = a @ W[l] + B[l]
            amag = a.abs() @ W[l].abs() + B[l].abs()
            ref = _act64(act, pre)
            st.max("fwd_excess", excess(h_hi[l], h_lo[l], ref, amag, x3, 0.0 if relu else ACT_BOUND * U24 * ref.abs()))
            st.add("fwd_fp16_bit_mismatches", (bits(ref.half()) != bits(h_hi[l])).sum())
            if "act" in alt:
                alt_ref = _act64(alt["act"], pre)
                st.max(f"guard_fwd_l{l}", excess(h_hi[l], h_lo[l], alt_ref, amag, x3,
                                                 0.0 if alt["act"] == "relu" else ACT_BOUND * U24 * alt_ref.abs()))
            st.add("h_nonfinite", int((~torch.isfinite(hd[l])).sum()))
            st.max("pre_min", float(pre[real].min()))
            st.max("pre_max_neg", -float(pre[real].max()))
            if relu:
                # fp16x3: relu(v) < 2^-25 stores hi = lo = 0 under a set mask bit
                pos = hd[l] > 0
                st.add("mask_mismatches", int((mask[l] != (hd[l] != 0)).sum()))
                st.add("mask_clear_but_positive", int((pos & ~mask[l]).sum()))
                st.add("mask_set_value_zero", int((mask[l] & ~pos).sum()))
                st.add("mask_set_value_zero_not_tiny", int((mask[l] & ~pos & (pre > 2.0 ** -20)).sum()))
        # rgbs epilogue: density activation (+ noise) on ray rows, relu on sparsity rows, sigmoid of the SH sum
        heads = hd[7] @ Wh + bh
        hmag = hd[7].abs() @ Wh.abs() + bh.abs()
        rr = s[real]
        onray = rr < Mr
        got = rgbs[r0:r0 + rr.numel()].double()
        sig = heads[real, 0]
        sig_tol = FWD_ALLOW[precision] * U24 * hmag[real, 0]
        if noise is not None:
            sig = sig + torch.where(onray, noise[rr.clamp_max(Mr - 1)].double(), torch.zeros_like(sig))
            sig_tol = sig_tol + U24 * sig.abs()
        want, extra = _sigma_want(sig, onray, sigma_act)
        st.max("rgbs_sigma_excess", ((got[:, 3] - want).abs() / (sig_tol + extra).clamp_min(1e-300)).max())
        if "sigma_act" in alt:
            want, extra = _sigma_want(sig, onray, alt["sigma_act"])
            st.max("guard_rgbs_sigma", ((got[:, 3] - want).abs() / (sig_tol + extra).clamp_min(1e-300)).max())
        if onray.any():
            Y = _sh_basis(sh, v[rr[onray] // N].double()) if sh >= 0 else \
                torch.ones(int(onray.sum()), 1, dtype=torch.float64, device=dev)
            hr = heads[real][onray][:, 1:1 + C3].view(-1, K, 3)
            hm = hmag[real][onray][:, 1:1 + C3].view(-1, K, 3)
            prer = (Y[:, :, None] * hr).sum(1)
            tol = 0.25 * ((Y.abs()[:, :, None] * (FWD_ALLOW[precision] * U24 * hm + 4 * U24 * hr.abs())).sum(1)) \
                + 2 ** -21
            st.max("rgbs_rgb_excess", ((got[onray, :3] - torch.sigmoid(prer)).abs() / tol).max())

        # ---------------- B. data gradient ----------------
        # dO: G.w in column 0, G.rgb x SH basis in the heads columns, zero on free / padded rows and pads
        g = torch.zeros(r1 - r0, 4, dtype=torch.float32, device=dev)
        g[:int(real.sum())] = G[r0:r0 + int(real.sum())]
        gh = g[:, 3].half()
        st.add("dO_sigma_bit_mismatches", int((bits(do_hi[:, 0]) != bits(gh)).sum()))
        if x3:
            st.add("dO_sigma_bit_mismatches", int((bits(do_lo[:, 0]) != bits((g[:, 3] - gh.float()).half())).sum()))
        ray_rows = s < Mr
        Yall = torch.zeros(r1 - r0, K, dtype=torch.float64, device=dev)
        if ray_rows.any():
            Yall[ray_rows] = (_sh_basis(sh, v[s[ray_rows] // N].double()) if sh >= 0 else 1.0)
        ref_do = (g[:, None, :3].double() * Yall[:, :, None]).reshape(-1, C3)
        # beyond the rounding of the stored value, in units of 2^-24 * |G.rgb|: the fp32 SH basis cancels (e.g.
        # 2zz - xx - yy), so its error is absolute, on the scale of |G.rgb|, not relative to G.rgb * Y_k
        gmag = g[:, None, :3].double().abs().expand(-1, K, 3).reshape(-1, C3)
        st.max("dO_rgb_excess", excess(do_hi[:, 1:1 + C3], do_lo[:, 1:1 + C3], ref_do, gmag, x3))
        err = (do_hi[:, 1:1 + C3].double() + do_lo[:, 1:1 + C3].double() - ref_do).abs()
        st.max("dO_rgb_err_ulps", (err / ulp16(ref_do)).max())
        nzr = (do_hi != 0) | (do_lo != 0)
        st.add("dO_free_or_padded_rgb_nonzero", int(nzr[~ray_rows, 1:1 + C3].sum()))
        st.add("dO_padded_sigma_nonzero", int(nzr[~real, 0].sum()))
        st.add("dO_pad_columns_nonzero", int(nzr[:, 1 + C3:nd].sum()))
        st.add("padded_rows_nonzero", int(nzr[~real].sum()))
        # dZ_l = dH_l * f'(h_l) with f' from the kernel's own saved h_l (relu: its mask words)
        dod = (do_hi.double() + do_lo.double())[:, :NH]
        dzd = [a.double() + b.double() for a, b in zip(dz_hi, dz_lo)]
        for l in range(7, -1, -1):
            a, Wt = (dod, Wh.T) if l == 7 else (dzd[l + 1], W[l + 1][:256].T)
            dh = a @ Wt
            gp = mask[l].double() if relu else _grad_of_output(act, hd[l])
            ref = dh * gp
            amag = (a.abs() @ Wt.abs()) * gp.abs()
            ex_all = excess(dz_hi[l], dz_lo[l], ref, amag, x3)
            ex = ex_all
            if x3:
                # rows whose contraction reads an fp16-subnormal operand: BWD_SUBNORMAL_ALLOW, not BWD_ALLOW
                sub_row = ((a != 0) & (a.abs() < 2.0 ** -14)).any(1, keepdim=True)
                ex = excess(dz_hi[l], dz_lo[l], torch.where(sub_row, dzd[l], ref), amag, x3)
            st.max("bwd_excess", ex)
            st.max(f"bwd_excess_dz{l}", ex)
            st.max("bwd_excess_subnormal_operand_rows", ex_all)
            st.add("bwd_fp16_bit_mismatches", (bits(ref.half()) != bits(dz_hi[l])).sum())
            if "act" in alt:
                gpa = _grad_of_output(alt["act"], hd[l])
                st.max(f"guard_bwd_l{l}", excess(dz_hi[l], dz_lo[l], dh * gpa, (a.abs() @ Wt.abs()) * gpa.abs(), x3))
            if not relu:
                # mutation: the relu mask of h_l in place of f'(h_l)
                st.min("bwd_excess_relu_mask_mutation", excess(dz_hi[l], dz_lo[l], dh * (hd[l] > 0).double(), amag,
                                                               x3))
            nzb = (bits(dz_hi[l]) != 0) | (bits(dz_lo[l]) != 0)
            if relu:
                st.add("dz_masked_nonzero_bits", int(nzb[~mask[l]].sum()))
            st.add("dz_padded_nonzero_bits", int(nzb[~real].sum()))
            st.add("dz_padded_nonzero", int(nzb[~real].sum()))        # the flag-model records' name of the same count
            st.add("padded_rows_nonzero", int(nzb[~real].sum()))
            st.add("dz_nonfinite", int((~torch.isfinite(dzd[l])).sum()))
            st.max("dz_headroom", float(dz_hi[l].abs().max()) / 65504.0)
            nz = dz_hi[l] != 0
            st.add("dz_nonzero", int(nz.sum()))
            st.add("dz_subnormal", int((nz & (dz_hi[l].abs() < 2 ** -14)).sum()))
            st.add("dz_lo_subnormal", int((nz & (dz_lo[l].abs() < 2 ** -14)).sum()))
            st.max("dz_abs_max", float(dz_hi[l].abs().max()))

        # ---------------- C. weight-gradient sums ----------------
        for l in range(1, 8):
            wsum(f"w{l}", hd[l - 1] if l != 5 else torch.cat([hd[4], eW], 1), dzd[l], r0)
        wsum("w0", eW, dzd[0], r0)
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
            eps, eps2 = eps[precision], eps2[precision]
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
            if elem > st.d.get(f"wgrad_{nm}_max_err_over_abs_sum", float("-inf")):
                st.d[f"wgrad_{nm}_worst_tensor"] = f"Dense_{l}.{nm}"
            st.max(f"wgrad_{nm}_max_err_over_abs_sum", elem)
            st.max(f"wgrad_{nm}_rel_l2", rel)
            st.max("wgrad_max_err_over_abs_sum", elem)
            st.max("wgrad_rel_l2", rel)
            st.max("wgrad_sensitivity_min_neg", -sens)
    return report


def check_call(model, state, ctx, precision, alt=None):
    """check_level on every level of the training call in the model's workspace, with the model's flags ->
    {MLP_i: {stages, wgrad, M, tiles}}"""
    from plenoctree_b200.nerf.train import default_loss_scale
    ws = model.workspace(True, precision)
    views = L.train_workspace_views(model.cfg, ctx["n"], ctx["sp"] is not None, precision=precision)
    assert views["total"] == ws.numel()
    scale = default_loss_scale(ctx["n"], precision)
    flat = model.params.cpu().numpy()
    P = model.P
    noise = ctx.get("noise")
    res = {}
    for i, lv in enumerate(views["levels"]):
        st = Stats()
        last = i == len(views["levels"]) - 1
        call = dict(rays=ctx["rays"], n=ctx["n"], sp=ctx["sp"] if last else None,
                    noise=noise[i] if noise is not None else None)
        rep = check_level(ws, lv, flat[i * P:(i + 1) * P], state.grads[i * P:(i + 1) * P], model.sh_deg, scale, st,
                          precision=precision, call=call, act=model.net_activation, pe=model.posenc,
                          sigma_act=model.sigma_activation, alt=alt)
        res[f"MLP_{i}"] = dict(stages=st.d, wgrad=rep, M=lv["M"], tiles=lv["tiles"])
    return res


def assert_stages(res, precision, act, guard=True, wg_w_bar=None):
    """the bars of check_call's result; guard: also the sensitivity of every weight-gradient tensor; wg_w_bar: the
    kernels' max |err| / sum |a b| bar in place of WG_EPS_W"""
    zero = ["posenc_xyz_bit_mismatches", "posenc_pad_nonzero_bits", "posenc_col63_not_one", "h_nonfinite",
            "split_violations_e", "split_violations_h", "split_violations_do", "split_violations_dz",
            "dO_sigma_bit_mismatches", "dO_free_or_padded_rgb_nonzero", "dO_padded_sigma_nonzero",
            "dO_pad_columns_nonzero", "padded_rows_nonzero", "dz_padded_nonzero_bits", "dz_nonfinite"]
    if act == "relu":
        zero += ["mask_clear_but_positive", "mask_set_value_zero_not_tiny", "dz_masked_nonzero_bits"]
        if precision == FP16:
            zero.append("mask_mismatches")
    for mlp, r in res.items():
        s = r["stages"]
        for k in zero:
            assert s[k] == 0, (act, mlp, k, s[k])
        assert s.get("posenc_sin_excess", 0.0) <= SIN_ALLOW[precision], (act, mlp, s)
        assert s["fwd_excess"] <= FWD_ALLOW[precision], (act, mlp, s["fwd_excess"])
        assert s["rgbs_sigma_excess"] <= 1.0, (act, mlp, s["rgbs_sigma_excess"])
        assert s.get("rgbs_rgb_excess", 0.0) <= 1.0, (act, mlp, s["rgbs_rgb_excess"])
        assert s["dO_rgb_excess"] <= DO_ALLOW[precision], (act, mlp, s["dO_rgb_excess"])
        if precision == FP16 and act == "relu":
            assert s["dO_rgb_err_ulps"] <= 1.0, (act, mlp, s["dO_rgb_err_ulps"])
        assert s["bwd_excess"] <= BWD_ALLOW[precision], (act, mlp, s["bwd_excess"])
        assert s["bwd_excess_subnormal_operand_rows"] <= BWD_SUBNORMAL_ALLOW[precision], (act, mlp, s)
        assert s["dz_headroom"] < 1.0, (act, mlp, s["dz_headroom"])
        for name, w in r["wgrad"].items():
            eps = WG_EPS_B[precision] if name.endswith(".b") else wg_w_bar or WG_EPS_W[precision]
            eps2 = (WG_EPS2_B if name.endswith(".b") else WG_EPS2_W)[precision]
            assert w["max_err_over_abs_sum"] <= eps, (act, mlp, name, w)
            if precision == FP16:
                assert w["rel_l2"] <= eps2, (act, mlp, name, w)
            if guard:
                assert w["sensitivity"] >= SENSITIVITY, (act, mlp, name, w)


CASES = [
    Case(3, 96, 64, 128, 300),                                   # the shape test_train.py uses
    *[Case(sh, 40, 64, 128, 64) for sh in (-1, 0, 1, 2, 4)],     # every heads width: NH 16/16/16/32/80
    Case(3, 64, 64, 0, 0), Case(3, 64, 64, 0, 200),              # single level; sparsity rows on MLP_0
    Case(3, 1, 3, 0, 0), Case(3, 1, 3, 0, 1), Case(3, 1, 3, 5, 0), Case(3, 1, 3, 5, 1),   # one real tile
    Case(3, 8, 64, 0, 0), Case(3, 8, 64, 0, 1),                  # M = 512 exactly, and 513
    Case(3, 32, 64, 192, 64),                                    # N = 256
    Case(3, 64, 64, 128, 0, noise=True),                         # noised sigma in the rgbs epilogue
]


def _render_mismatches(model, ctx, precision):
    """bits in which the training forward's rgbs / comp / disp / acc differ from the render of the same draws and
    noise at the same precision, per level"""
    from plenoctree_b200.nerf.models import Rays
    o, d, v = ctx["rays"]
    out = model(Rays(o, d, v), randomized=True, t_rand=ctx["t_rand"], u=ctx["u"], precision=precision,
                sigma_noise=ctx["noise"])
    torch.cuda.synchronize()
    ws, rws = model.workspace(True, precision), model.workspace(False)
    views = L.train_workspace_views(model.cfg, ctx["n"], ctx["sp"] is not None, precision=precision)
    rviews = L.train_workspace_views(model.cfg, ctx["n"], False, training=False)
    mism = {}
    for i, (lv, rlv) in enumerate(zip(views["levels"], rviews["levels"])):
        Mr = lv["M_rays"]
        mism[f"rgbs_{i}"] = int((L.workspace_view(ws, lv, "rgbs")[:Mr].view(torch.int32)
                                 != L.workspace_view(rws, rlv, "rgbs")[:Mr].view(torch.int32)).sum())
        got = torch.cat([L.workspace_view(ws, lv, "comp"), L.workspace_view(ws, lv, "disp")[:, None],
                         L.workspace_view(ws, lv, "acc")[:, None]], 1)
        want = torch.cat([out[i][0], out[i][1][:, None], out[i][2][:, None]], 1)
        mism[f"comp_disp_acc_{i}"] = int((got.view(torch.int32) != want.view(torch.int32)).sum())
    return mism


def stage_case(case, record, guard=True, wg_w_bar=None):
    """one training call of `case` on a 0xFF-filled workspace (NaN in every byte the call does not write): the
    training forward's outputs bit-identical to the render of the same draws, then every stage against fp64 and its
    bars.  The result goes to record(case.name, result)."""
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    model = case.model()
    state, ctx = case.run(model, fill=0xFF)
    res = check_call(model, state, ctx, case.precision)
    mism = _render_mismatches(model, ctx, case.precision)
    res.update(render_bit_mismatches=mism, wall_s=time.time() - t0,
               peak_alloc_gb=torch.cuda.max_memory_allocated() / 2 ** 30)
    record(case.name, res)
    assert all(x == 0 for x in mism.values()), mism
    assert_stages({k: v for k, v in res.items() if k.startswith("MLP")}, case.precision, case.act, guard, wg_w_bar)
    return res

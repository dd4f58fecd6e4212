"""The vanilla NeRF (use_viewdirs) model flags combined: trunk activation (net_activation), point encoder
(min_deg_point, max_deg_point, legacy_posenc_order, which also orders the view encoder), deg_view, density activation
(sigma_activation), ray length and level count, draws (jitter, resampled fine depths, sigma noise), background, ray
family (Blender or forward-facing NDC) and a call over fewer rays than the workspace was carved for, over a covering
matrix of rows.

tests/test_vanilla_render.py varies one flag at a time, while check_vanilla_scope accepts every combination, and some
compiled paths run only when flags are combined: the elu, softplus and tanh OUT_VANILLA forwards with the runtime
("generic") point encoder, the render path's table row s / n_per_ray where a ray boundary falls inside a warpgroup's
rows (n_per_ray 33, 127) or a ray spans several tiles (n_per_ray 1024), a smooth trunk under the softplus density.

CPU: the matrix's covering properties, the OUT_VANILLA instantiations it reaches, and the host mirror of the vanilla
render workspace (layouts.train_workspace_views(..., vanilla=True)) against pob_vanilla_workspace_bytes.
GPU, per row: one VanillaNerfModel call on a 0xFF-filled workspace, then, per level and from the workspace's own
inputs: the depths (coarse bit-exact, fine bit-equal to a standalone pob_sample_pdf and against fp64), the per-ray view
table against fp64, the density against the sigma blob's raw sigma, the colour against an fp64 view branch from the
kernel's own fp16 h7 and the workspace's table row of the sample's ray, the compositing against fp64, and the render
path against the point path bit for bit; each check again against a reference with one thing wrong (mutation
guards).  Then the point path (pob_eval_points_vanilla) of both MLPs at ragged point counts with canaries.
Once: the SM split, the workspace fill and a smaller call after a larger one leave every bit unchanged.
"""
import functools
import os
import re

import numpy as np
import pytest
import torch

from plenoctree_b200 import layouts as L
from tests.support.covering import assert_covers_every_pair
from tests.support.model_flags import SP_BAR, SP_FLOOR, _alt_pe
from tests.support.records import ROOT, record
from tests.support.vanilla_ref import C_BRANCH, U, _h7_fp16, _rays, _view_features

GUARD = 10.0        # a check must miss its bar by at least this factor against a reference with one thing wrong
# the logistic 1 / (1 + expf(-r)) at the kernel's fp32 r, relative to its value: expf within 2 ulp (4 u), the add and
# the division one rounding each
LOGISTIC_ULPS = 6.0
# the view table against fp64 at the fp32 sine arguments (test_vanilla_render.test_view_branch_against_fp64_from_the_
# kernels_h7): 64 u sum |terms| + 1e-6 max |feature| (sinf of arguments up to 2^31)
TABLE_ULPS, TABLE_ABS = 64.0, 1e-6

DEF_PE = (0, 10, False)
TRUNKS = ("relu", "elu", "softplus", "tanh")
ENCODERS = (DEF_PE, (0, 10, True), (2, 8, True), (0, 0, False), (9, 10, True))
DEG_VIEWS = (0, 1, 10, 32)
DENSITIES = ("relu", "softplus")
# (rays, coarse, fine)
SHAPES = ((40, 64, 128),                   # both levels
          (64, 64, 0),                     # one level
          (16, 128, 384),                  # N = 512: the one-block-per-ray compositing
          (1, 3, 5),                       # one partial tile
          (7, 33, 94),                     # n_per_ray 33 and 127: ray boundaries at many rows inside a tile
          (2, 1000, 24))                   # one ray spans 8 tiles
DRAWS = ("det", "rand", "noise")           # deterministic; jitter + resampled fine depths; the same + sigma noise
WHITE = (True, False)
# blender: near 2, far 6.  ndc: forward-facing rays through nerf.rays.convert_to_ndc, near 0, far 1 with depths linear
# in z (the reference's LLFF setting: lindisp would divide by near = 0)
RAY_FAMILIES = ("blender", "ndc")
SPARE = (False, True)                      # max_rays = R, or R + SPARE_RAYS: a call over fewer rays than were carved
SPARE_RAYS = 13
DIMS = (TRUNKS, ENCODERS, DEG_VIEWS, DENSITIES, SHAPES, DRAWS, WHITE, RAY_FAMILIES, SPARE)

# trunk, encoder, deg_view, density, shape, draws, white_bkgd, rays, spare rays
MATRIX = [
    ("tanh", DEF_PE, 32, "relu", (40, 64, 128), "rand", False, "blender", True),
    ("elu", (0, 10, True), 32, "relu", (40, 64, 128), "det", True, "ndc", False),
    ("softplus", (2, 8, True), 10, "relu", (40, 64, 128), "det", False, "ndc", True),
    ("relu", (0, 0, False), 0, "softplus", (40, 64, 128), "det", False, "ndc", False),
    ("elu", (9, 10, True), 1, "softplus", (40, 64, 128), "noise", False, "ndc", True),
    ("elu", DEF_PE, 0, "softplus", (64, 64, 0), "noise", False, "blender", True),
    ("softplus", (0, 10, True), 0, "relu", (64, 64, 0), "rand", True, "ndc", True),
    ("relu", (2, 8, True), 1, "relu", (64, 64, 0), "rand", True, "ndc", False),
    ("elu", (0, 0, False), 32, "softplus", (64, 64, 0), "rand", False, "blender", True),
    ("tanh", (9, 10, True), 10, "relu", (64, 64, 0), "det", False, "blender", False),
    ("tanh", DEF_PE, 0, "relu", (16, 128, 384), "det", True, "blender", True),
    ("relu", (0, 10, True), 1, "softplus", (16, 128, 384), "det", False, "blender", False),
    ("elu", (2, 8, True), 32, "relu", (16, 128, 384), "noise", False, "blender", True),
    ("softplus", (0, 0, False), 1, "relu", (16, 128, 384), "det", True, "blender", True),
    ("relu", (9, 10, True), 10, "relu", (16, 128, 384), "rand", False, "ndc", False),
    ("relu", DEF_PE, 10, "softplus", (1, 3, 5), "noise", False, "ndc", False),
    ("tanh", (0, 10, True), 10, "relu", (1, 3, 5), "noise", True, "ndc", True),
    ("softplus", (2, 8, True), 32, "softplus", (1, 3, 5), "det", True, "blender", False),
    ("elu", (0, 0, False), 0, "softplus", (1, 3, 5), "rand", True, "ndc", False),
    ("tanh", (9, 10, True), 1, "relu", (1, 3, 5), "rand", True, "blender", False),
    ("elu", DEF_PE, 1, "softplus", (7, 33, 94), "rand", True, "blender", True),
    ("elu", (0, 10, True), 10, "relu", (7, 33, 94), "det", True, "blender", False),
    ("tanh", (2, 8, True), 32, "relu", (7, 33, 94), "rand", False, "blender", False),
    ("relu", (0, 0, False), 1, "relu", (7, 33, 94), "noise", False, "blender", False),
    ("softplus", (9, 10, True), 0, "relu", (7, 33, 94), "det", True, "ndc", False),
    ("softplus", DEF_PE, 32, "relu", (2, 1000, 24), "noise", False, "ndc", False),
    ("elu", (0, 10, True), 1, "relu", (2, 1000, 24), "rand", True, "blender", False),
    ("tanh", (2, 8, True), 0, "softplus", (2, 1000, 24), "noise", False, "ndc", True),
    ("tanh", (0, 0, False), 10, "relu", (2, 1000, 24), "rand", False, "blender", True),
    ("relu", (9, 10, True), 32, "softplus", (2, 1000, 24), "det", True, "blender", True),
]
OFF_DEFAULT = MATRIX[4]            # every flag away from its default (deg_view 4, relu, relu, white, Blender, R)
POINT_COUNTS = (1, 127, 128, 129, 4097)


def _tag(row):
    act, pe, dv, dens, (R, nc, nf), draw, white, rays, spare = row
    return (f"{act}_{pe[0]}_{pe[1]}_{'legacy' if pe[2] else 'std'}_dv{dv}_{dens}_R{R}_{nc}+{nf}_{draw}"
            + ("" if white else "_black") + f"_{rays}" + ("_spare" if spare else ""))


def _max_rays(row):
    R = row[4][0]
    return R + SPARE_RAYS if row[8] else R


_record = functools.partial(record, "parity_vanilla_flags.json")


# =====================================================================================================================
# CPU
# =====================================================================================================================
def test_matrix_covers_every_pair():
    """every pair of values of any two dimensions appears in some row"""
    assert_covers_every_pair(MATRIX, DIMS)


def _compiled_vanilla_trunks():
    src = open(os.path.join(ROOT, "plenoctree_b200", "csrc", "mlp_fwd.cu")).read()
    body = src[src.index("cudaError_t launch_mlp_fwd_vanilla("):]
    return {a.lower() for a in re.findall(r"mlp_fwd_kernel<1, OUT_VANILLA, false, NET_(\w+)>", body)}


def test_matrix_reaches_every_vanilla_instantiation_with_both_encoder_branches():
    """the OUT_VANILLA forward is compiled once per trunk activation; each one runs in some row with the default
    encoder and in some row with the runtime ("generic") encoder"""
    assert _compiled_vanilla_trunks() == set(TRUNKS)
    seen = {(r[0], r[1] == DEF_PE) for r in MATRIX}
    want = {(a, d) for a in TRUNKS for d in (True, False)}
    assert seen == want, want - seen


def _cfg(nc, nf, white, max_rays):
    from plenoctree_b200._lib import RenderConfig
    return RenderConfig(-1, nc, nf, int(white), max_rays, 0)


def test_vanilla_workspace_mirror_matches_library():
    """train_workspace_views(..., training=False, vanilla=True) reproduces carve(..., vanilla=true): the total of
    pob_vanilla_workspace_bytes for every row's configuration at its own max_rays and at 1, 7 and 4096; the render
    buffers where the render workspace has them, a view table [n_rays, 128] per level behind them, no overlap"""
    from plenoctree_b200._lib import lib
    from plenoctree_b200.nerf.models import ctypes_ref
    n = 0
    for row in MATRIX:
        (_, nc, nf), white = row[4], row[6]
        for R in sorted({_max_rays(row), 1, 7, 4096}):
            cfg = _cfg(nc, nf, white, R)
            want = int(lib.pob_vanilla_workspace_bytes(ctypes_ref(cfg)))
            render = int(lib.pob_workspace_bytes(ctypes_ref(cfg), 0))
            for n_rays in sorted({1, (R + 1) // 2, R}):
                v = L.train_workspace_views(cfg, n_rays, False, training=False, vanilla=True)
                r = L.train_workspace_views(cfg, n_rays, False, training=False)
                assert v["total"] == want, (row, R)
                assert len(v["levels"]) == (2 if nf else 1) and v["partials"] == []
                ext = []
                for lv, lr in zip(v["levels"], r["levels"]):
                    assert sorted(k for k in lv if isinstance(lv[k], tuple)) == \
                        ["acc", "comp", "disp", "rgbs", "view_t", "weights", "z"]
                    assert lv["view_t"][1] == (n_rays, 128) and lv["view_t"][0] >= render
                    for k in ("z", "rgbs", "weights", "comp", "disp", "acc"):
                        assert lv[k] == lr[k], (row, R, k)
                    for val in lv.values():
                        if isinstance(val, tuple):
                            ext.append((val[0], val[0] + 4 * int(np.prod(val[1]))))
                ext.sort()
                for (a0, a1), (b0, _) in zip(ext, ext[1:]):
                    assert a0 % 1024 == 0 and a1 <= b0
                assert ext[-1][1] <= want
                n += 1
    assert n > 200
    with pytest.raises(ValueError, match="render workspace"):
        L.train_workspace_views(_cfg(64, 128, True, 8), 8, False, training=True, vanilla=True)


# =====================================================================================================================
# GPU
# =====================================================================================================================
def _row_inputs(row, seed):
    """(o, d, v) [R, 3], t_rand [R, nc] | None, u [R, nf] | None, sigma_noise (coarse, fine) | None: fp32 numpy"""
    from plenoctree_b200.nerf.rays import convert_to_ndc
    f = np.float32
    (R, nc, nf), draw, family = row[4], row[5], row[7]
    rs = np.random.RandomState(seed)
    if family == "blender":
        o, d, v = _rays(R, seed)
    else:
        # a forward-facing camera at the origin looking down -z, its rays through the NDC transform; the view
        # directions stay the world-space ones (nerf/datasets.py)
        cam_o = rs.uniform(-0.05, 0.05, (R, 3)).astype(f)
        cam_d = np.concatenate([rs.uniform(-0.8, 0.8, (R, 2)), -np.ones((R, 1))], 1).astype(f)
        v = (cam_d / np.linalg.norm(cam_d, axis=1, keepdims=True)).astype(f)
        o, d = (np.asarray(x, f) for x in convert_to_ndc(cam_o, cam_d, 60.0, 64, 64, near=1.0))
    if draw == "det":
        return (o, d, v), None, None, None
    t_rand = rs.uniform(0, 1, (R, nc)).astype(f)
    u = rs.uniform(0, 1, (R, nf)).astype(f) if nf else None
    noise = None
    if draw == "noise":
        noise = (rs.normal(size=(R, nc)).astype(f), rs.normal(size=(R, nc + nf)).astype(f) if nf else None)
    return (o, d, v), t_rand, u, noise


def _scene_mlps(seed, pe, deg_view, act):
    """{"MLP_0", "MLP_1"} of projection_oracle.init_params with every trunk layer's pre-activations centred over the
    scene box (each bias minus its mean) and raw sigma scaled by 8 around its median there: raw sigma of both signs,
    half the box dense, under every trunk activation.  Uncentred, a softplus trunk's raw sigma is large and positive at
    every point (softplus >= 0 adds a common positive part layer by layer), so every ray is opaque and relu and
    softplus of raw sigma agree to a few ulp."""
    from oracle import net_activation_oracle as NA
    from oracle import posenc_oracle as PO
    from oracle.projection_oracle import init_params
    f = NA.activation(act)
    box = torch.from_numpy(np.random.RandomState(5).uniform(-1.5, 1.5, (4000, 3)))
    enc = PO.encode(box, pe)
    mlps = {}
    for i, name in enumerate(("MLP_0", "MLP_1")):
        layers = init_params(seed + i, pe, deg_view)
        h = enc
        with torch.no_grad():
            for l in range(8):
                k, b = layers[l]
                z = h @ torch.from_numpy(k).double() + torch.from_numpy(b).double()
                shift = z.mean(0)
                layers[l] = (k, (b - shift.numpy()).astype(np.float32))
                h = f(z - shift)
                if l == 4:
                    h = torch.cat([h, enc], -1)
            k, b = layers[8]
            sig = h @ torch.from_numpy(k).double() + float(b[0])
        med = float(np.median(sig.numpy()))
        layers[8] = ((k * np.float32(8)).astype(np.float32), ((b - np.float32(med)) * np.float32(8)).astype(np.float32))
        mlps[name] = layers
    return mlps


def _row_model(row, mlps):
    from plenoctree_b200.nerf.vanilla import VanillaNerfModel
    act, pe, dv, dens, (R, nc, nf), _, white, family, _ = row
    near, far = (2.0, 6.0) if family == "blender" else (0.0, 1.0)
    return VanillaNerfModel(mlps, deg_view=dv, num_coarse_samples=nc, num_fine_samples=nf, near=near, far=far,
                            white_bkgd=white, max_rays=_max_rays(row), sigma_activation=dens, min_deg_point=pe[0],
                            max_deg_point=pe[1], legacy_posenc_order=pe[2], net_activation=act)


def _call(model, rays, t_rand, u, noise):
    from plenoctree_b200.nerf.models import Rays
    out = model(Rays(*rays), randomized=t_rand is not None, t_rand=t_rand, u=u, sigma_noise=noise)
    torch.cuda.synchronize()
    return out


def _act_code(act):
    from plenoctree_b200.nerf.flags import net_activation_code
    return net_activation_code(act)


def _act64(act, z):
    from tests.support.model_flags import _act64 as A
    return A(act, torch.from_numpy(z)).numpy()


def _softplus64(x):
    from tests.support.model_flags import softplus64
    return softplus64(torch.from_numpy(np.asarray(x, np.float64))).numpy()


def _sigma_blob(layers, pe):
    """the plain-RGB (sh_deg -1) blob of the trunk and Dense_8 with zero rgb columns: column 0 of its heads is the
    raw sigma extraction evaluates (octree/projection.py: VanillaNerf.sigma_blob)"""
    from plenoctree_b200 import ops
    flat = np.concatenate([np.asarray(a, np.float32).reshape(-1) for k, b in layers[:9] for a in (k, b)]
                          + [np.zeros(256 * 3 + 3, np.float32)])
    return ops.pack_weights(torch.from_numpy(flat).cuda(), -1, posenc=pe)


def _raw_sigma(layers, pe, act, pts):
    """raw sigma [m] (fp32 numpy) of the sigma blob at the points (CUDA [m, 3]) with the encoder and the trunk"""
    from plenoctree_b200 import ops
    _, s = ops.eval_points_raw(_sigma_blob(layers, pe), -1, pts, want_rgb=False, posenc=pe,
                               net_activation=_act_code(act))
    return s[:, 0].cpu().numpy()


def _density_err(got, x32, dens):
    """max of |got - act(x)| / (SP_BAR u act(x) + SP_FLOOR) over the rows (x = raw sigma + noise in fp32): relu is
    exact, softplus_f32 within SP_BAR u (kernels.h); and the count of relu rows that differ in any bit"""
    if dens == "relu":
        want = np.maximum(x32, np.float32(0)).astype(np.float32)
        bits = int((got.view(np.int32) != want.view(np.int32)).sum())
        want = want.astype(np.float64)
    else:
        want, bits = _softplus64(x32), 0
    err = np.abs(got.astype(np.float64) - want) / (SP_BAR * U * np.abs(want) + SP_FLOOR)
    return float(err.max()), bits


def _table_ref(layers, enc):
    """(fp64 W10_e posenc(v) + c [m, 128], the bound TABLE_ULPS u sum|terms| + TABLE_ABS max|feature|)"""
    from plenoctree_b200.nerf import vanilla as V
    w10e = np.asarray(layers[10][0][256:], np.float64)
    _, c = V.fold_view_branch(layers)
    t64 = enc @ w10e + c
    bound = TABLE_ULPS * U * (np.abs(enc) @ np.abs(w10e) + np.abs(c)) + TABLE_ABS * np.abs(enc).max(1, keepdims=True)
    return t64, bound


def _table_err(t, layers, enc):
    t64, bound = _table_ref(layers, enc)
    return float((np.abs(t - t64) / bound).max())


class Branch:
    """the fp64 view branch W11 act(h7 fold + t) + b11 from the kernel's fp16 h7 [m, 256], the packed fp16 fold and
    per-row tables t [m, 128]; raw rgb within C_BRANCH u sum|terms| (test_vanilla_render)"""

    def __init__(self, layers, h):
        from plenoctree_b200.nerf import vanilla as V
        self.fold = V.folded_flat(layers)[-256 * 128:].reshape(256, 128).astype(np.float64)
        self.w11, self.b11 = (np.asarray(x, np.float64) for x in layers[11])
        self.h = h
        self.a = h @ self.fold
        self.a_abs = np.abs(h) @ np.abs(self.fold)

    def raw(self, t, act):
        z = _act64(act, self.a + t)
        want = z @ self.w11 + self.b11
        terms = ((self.a_abs + np.abs(t)) @ np.abs(self.w11)) + np.abs(z) @ np.abs(self.w11) + np.abs(self.b11)
        return want, C_BRANCH * U * terms

    def raw_err(self, got, t, act):
        want, bound = self.raw(t, act)
        return float((np.abs(got - want) / bound).max())

    def rgb_err(self, got, t, act):
        """sigmoid of the fp64 branch: the raw bound through the logistic's slope, plus the logistic's own error"""
        want, bound = self.raw(t, act)
        s = 1.0 / (1.0 + np.exp(-want))
        den = s * (1.0 - s) * bound + LOGISTIC_ULPS * U * s
        return float((np.abs(got - s) / den).max())

    def prefix(self, m):
        """the branch of the first m rows"""
        b = object.__new__(Branch)
        b.fold, b.w11, b.b11 = self.fold, self.w11, self.b11
        b.h, b.a, b.a_abs = self.h[:m], self.a[:m], self.a_abs[:m]
        return b


def _other(act, dens):
    return "softplus" if act == "relu" else "relu", "softplus" if dens == "relu" else "relu"


def _check_level(row, model, mlps, views, ws, i, rays, noise):
    """checks 2, 3, 4 and 6 of level i, with their mutation guards"""
    from plenoctree_b200 import _lib
    from tests.support.eval_stages import _nbits
    from tests.support.model_flags import CANARY, _canary
    act, pe, dv, dens = row[:4]
    o, d, v = rays
    n = o.shape[0]
    lv = views["levels"][i]
    N, M = lv["N"], lv["M_rays"]
    layers, other = mlps[f"MLP_{i}"], mlps[f"MLP_{1 - i}"]
    alt_act, alt_dens = _other(act, dens)
    res = {}

    # 2. the per-ray view table against fp64 at the fp32 sine arguments
    t = L.workspace_view(ws, lv, "view_t").cpu().numpy().astype(np.float64)
    enc = _view_features(v, dv, pe[2])
    res["table"] = _table_err(t, layers, enc)
    res["guard_table_other_mlp"] = _table_err(t, other, enc)
    if dv >= 2:      # at deg_view 1 both orders give the same features [v, sin(v), cos(v)]
        res["guard_table_legacy_flipped"] = _table_err(t, layers, _view_features(v, dv, not pe[2]))

    # 3. density: the sample points as load_point forms them, o + fl(t d) with a separate multiply and add
    z = L.workspace_view(ws, lv, "z").cpu().numpy()
    ray = np.repeat(np.arange(n), N)
    pts = (o[ray] + (z.reshape(-1)[:, None] * d[ray]).astype(np.float32)).astype(np.float32)
    pts_t = torch.from_numpy(pts).cuda()
    rgbs = L.workspace_view(ws, lv, "rgbs")[:M].cpu().numpy()
    nz = None if noise is None else noise[i].reshape(-1)
    sig = _raw_sigma(layers, pe, act, pts_t)

    def dens_err(s, de=dens, with_noise=True):
        x = s if nz is None or not with_noise else (s + nz).astype(np.float32)
        return _density_err(rgbs[:, 3], x, de)

    res["density"], res["density_relu_bit_mismatches"] = dens_err(sig)
    res["guard_density_trunk"] = dens_err(_raw_sigma(layers, pe, alt_act, pts_t))[0]
    res["guard_density_other_density"] = dens_err(sig, alt_dens)[0]
    if _alt_pe(pe) is not None:
        res["guard_density_encoder"] = dens_err(_raw_sigma(layers, _alt_pe(pe), act, pts_t))[0]
    if nz is not None:
        res["guard_density_noise_dropped"] = dens_err(sig, with_noise=False)[0]

    # 4. colour: the kernel's fp16 h7 at the same points, the packed fold and the workspace's table row of the ray
    br = Branch(layers, _h7_fp16(layers, pts_t, pe, _act_code(act)))
    res["colour"] = br.rgb_err(rgbs[:, :3], t[ray], act)
    if n > 1:
        nb = np.where(ray + 1 < n, ray + 1, ray - 1)
        res["guard_colour_neighbour_ray_row"] = br.rgb_err(rgbs[:, :3], t[nb], act)
    t_other, _ = _table_ref(other, enc)
    bo = Branch(other, br.h)
    res["guard_colour_other_mlp"] = bo.rgb_err(rgbs[:, :3], t_other[ray], act)
    res["guard_colour_trunk"] = br.rgb_err(rgbs[:, :3], t[ray], alt_act)

    # 6. the point path at the same fp32 points, each with its ray's view direction: the same per-row arithmetic
    vd = torch.from_numpy(np.ascontiguousarray(v[ray])).cuda()
    tb, table = _canary((M, 128))
    ob, out = _canary((M, 4))
    _lib.check(_lib.lib.pob_eval_points_vanilla(_lib.ptr(model.blobs[i]), _lib.posenc_ref(model._pe),
                                                _lib.ctypes.addressof(model.view), i, _lib.ptr(pts_t), _lib.ptr(vd),
                                                M, _lib.ptr(table), None, None, _lib.ptr(out), model.sigma_act_code,
                                                _lib.stream_ptr()))
    torch.cuda.synchronize()
    got = torch.from_numpy(rgbs).cuda()
    if noise is None:
        res["points_vs_render_rgbs_bit_mismatches"] = _nbits(out, got)
    else:
        res["points_vs_render_rgb_bit_mismatches"] = _nbits(out[:, :3].contiguous(), got[:, :3].contiguous())
    res["points_vs_render_table_bit_mismatches"] = _nbits(table, torch.from_numpy(t[ray].astype(np.float32)).cuda())
    res["points_canary_mismatches"] = int((tb[M * 128:] != CANARY).sum()) + int((ob[M * 4:] != CANARY).sum())
    res["rgbs_nonfinite"] = int((~np.isfinite(rgbs)).sum())
    res["acc_mean"] = float(L.workspace_view(ws, lv, "acc").mean())
    return res


def _check_points(row, model, mlps, seed):
    """pob_eval_points_vanilla of every MLP of the model at POINT_COUNTS in raw and rgbs modes, canaries behind every
    output and behind the scratch table"""
    from plenoctree_b200 import _lib
    from tests.support.model_flags import CANARY, _canary
    act, pe, dv, dens = row[:4]
    rs = np.random.RandomState(seed)
    mmax = max(POINT_COUNTS)
    pts = torch.from_numpy(rs.uniform(-1.5, 1.5, (mmax, 3)).astype(np.float32)).cuda()
    vdn = rs.normal(size=(mmax, 3))
    vd32 = (vdn / np.linalg.norm(vdn, axis=1, keepdims=True)).astype(np.float32)
    vd = torch.from_numpy(vd32).cuda()
    enc = _view_features(vd32, dv, pe[2])
    res = {}
    for mlp in range(model.num_mlps):
        layers = mlps[f"MLP_{mlp}"]
        sig = _raw_sigma(layers, pe, act, pts)
        br = Branch(layers, _h7_fp16(layers, pts, pe, _act_code(act)))
        r = dict(table=0.0, raw_rgb=0.0, colour=0.0, density=0.0, raw_sigma_bit_mismatches=0,
                 density_relu_bit_mismatches=0, canary_violations=0)
        for m in POINT_COUNTS:
            for raw in (True, False):
                tb, table = _canary((m, 128))
                if raw:
                    bufs = [_canary((m, 3)), _canary((m,))]
                    outs = (bufs[0][1], bufs[1][1], None)
                else:
                    bufs = [_canary((m, 4))]
                    outs = (None, None, bufs[0][1])
                _lib.check(_lib.lib.pob_eval_points_vanilla(
                    _lib.ptr(model.blobs[mlp]), _lib.posenc_ref(model._pe), _lib.ctypes.addressof(model.view), mlp,
                    _lib.ptr(pts), _lib.ptr(vd), m, _lib.ptr(table), _lib.ptr(outs[0]), _lib.ptr(outs[1]),
                    _lib.ptr(outs[2]), model.sigma_act_code, _lib.stream_ptr()))
                torch.cuda.synchronize()
                r["canary_violations"] += sum(int((b[int(np.prod(x.shape)):] != CANARY).sum())
                                              for b, x in [(tb, table)] + bufs)
                t = table.cpu().numpy().astype(np.float64)
                r["table"] = max(r["table"], _table_err(t, layers, enc[:m]))
                if raw:
                    rgb, s = (x.cpu().numpy() for x in outs[:2])
                    r["raw_sigma_bit_mismatches"] += int((s.view(np.int32) != sig[:m].view(np.int32)).sum())
                    r["raw_rgb"] = max(r["raw_rgb"], br.prefix(m).raw_err(rgb, t, act))
                else:
                    o = outs[2].cpu().numpy()
                    e, bits = _density_err(o[:, 3], sig[:m], dens)
                    r["density"] = max(r["density"], e)
                    r["density_relu_bit_mismatches"] += bits
                    r["colour"] = max(r["colour"], br.prefix(m).rgb_err(o[:, :3], t, act))
        res[f"mlp{mlp}"] = r
    return res


def _run_row(row, seed, fill=0xFF):
    """the row's model and one call on a workspace filled with `fill`: (model, mlps, inputs, outputs, views)"""
    act, pe, dv = row[:3]
    mlps = _scene_mlps(100 + seed, pe, dv, act)
    model = _row_model(row, mlps)
    rays, t_rand, u, noise = _row_inputs(row, seed)
    ws = model.workspace()
    ws.fill_(fill)
    out = _call(model, rays, t_rand, u, noise)
    views = L.train_workspace_views(model.cfg, rays[0].shape[0], False, training=False, vanilla=True)
    assert views["total"] == ws.numel()
    return model, mlps, (rays, t_rand, u, noise), out, views


def _check_row(row, seed):
    from tests.support import ray_stages as RS
    model, mlps, (rays, t_rand, u, noise), out, views = _run_row(row, seed)
    ws = model.workspace()
    n = rays[0].shape[0]
    res = {}
    # 1 and 5: depths and compositing from the workspace's own inputs (ray_stages)
    if u is None and model.num_fine_samples:
        u_np, upr = model.u_table.cpu().numpy(), 0
    else:
        u_np, upr = u, 1
    st = {}
    res["rays"] = RS._check_levels(model, views, ws, rays, model.z_base.cpu().numpy(), t_rand, u_np, upr, st)
    for i, (lv, o) in enumerate(zip(views["levels"], out)):
        want = torch.cat([L.workspace_view(ws, lv, "comp"), L.workspace_view(ws, lv, "disp")[:, None],
                          L.workspace_view(ws, lv, "acc")[:, None]], 1)
        got = torch.cat([o[0], o[1][:, None], o[2][:, None]], 1)
        st[f"out{i}_vs_workspace_bit_mismatches"] = int((got.view(torch.int32) != want.view(torch.int32)).sum())
        res[f"level{i}"] = _check_level(row, model, mlps, views, ws, i, rays, noise)
    res["rays"]["stage"] = st
    res["points"] = _check_points(row, model, mlps, seed)
    res["n_rays"] = n
    return res


def _assert_row(row, res):
    from tests.support import ray_stages as RS
    act, pe, dv, dens, (R, nc, nf) = row[:5]
    RS._assert_in_call(res["rays"])
    for i in range(2 if nf else 1):
        r = res[f"level{i}"]
        for k, val in r.items():
            if k.endswith("mismatches") or k == "rgbs_nonfinite":
                assert val == 0, (i, k, r)
        assert r["table"] <= 1.0 and r["density"] <= 1.0 and r["colour"] <= 1.0, (i, r)
        guards = {k: val for k, val in r.items() if k.startswith("guard_")}
        assert all(val >= GUARD for val in guards.values()), (i, guards)
        # every guard the row can have is there
        want = {"guard_table_other_mlp", "guard_density_trunk", "guard_density_other_density",
                "guard_colour_other_mlp", "guard_colour_trunk"}
        want |= {"guard_table_legacy_flipped"} if dv >= 2 else set()
        want |= {"guard_colour_neighbour_ray_row"} if R > 1 else set()
        want |= {"guard_density_encoder"} if _alt_pe(pe) is not None else set()
        want |= {"guard_density_noise_dropped"} if row[5] == "noise" else set()
        assert set(guards) == want, (set(guards) ^ want)
    for k, r in res["points"].items():
        assert r["canary_violations"] == 0, (k, r)
        assert r["raw_sigma_bit_mismatches"] == 0 and r["density_relu_bit_mismatches"] == 0, (k, r)
        assert r["table"] <= 1.0 and r["raw_rgb"] <= 1.0 and r["colour"] <= 1.0 and r["density"] <= 1.0, (k, r)
    assert len(res["points"]) == (2 if nf else 1)


@pytest.mark.gpu
@pytest.mark.parametrize("row", MATRIX, ids=_tag)
def test_vanilla_flag_matrix_row(row):
    res = _check_row(row, MATRIX.index(row))
    _record(_tag(row), res)
    _assert_row(row, res)


@pytest.mark.gpu
def test_every_bit_is_independent_of_the_sm_split(monkeypatch):
    """the row with every flag away from its default at the device's SM count, then at 16 and 61: the whole workspace
    (every view, the untouched spare rays' rows included) and the outputs bit for bit"""
    from tests.support.model_flags import _set_sms
    seed = MATRIX.index(OFF_DEFAULT)
    runs = []
    for n in ("device", 16, 61):
        _set_sms(monkeypatch, n)
        model, _, _, out, _ = _run_row(OFF_DEFAULT, seed)
        runs.append([model.workspace().clone()] + [x.clone() for lvl in out for x in lvl])
    for other in runs[1:]:
        for k, (a, b) in enumerate(zip(runs[0], other)):
            assert torch.equal(a, b), k


_VIEWS = ("z", "rgbs", "weights", "comp", "disp", "acc", "view_t")


def _outputs_and_views(model, out, n):
    ws = model.workspace()
    views = L.train_workspace_views(model.cfg, n, False, training=False, vanilla=True)
    return [x.clone() for lvl in out for x in lvl] + [L.workspace_view(ws, lv, k).clone() for lv in views["levels"]
                                                      for k in _VIEWS]


def _bit_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.gpu
def test_outputs_do_not_depend_on_the_workspace_fill():
    """a 0xFF-filled and a zero-filled workspace give the same outputs and the same views over the call's rays"""
    seed = MATRIX.index(OFF_DEFAULT)
    runs = []
    for fill in (0xFF, 0):
        model, _, (rays, _, _, _), out, _ = _run_row(OFF_DEFAULT, seed, fill)
        runs.append(_outputs_and_views(model, out, rays[0].shape[0]))
    for k, (a, b) in enumerate(zip(*runs)):
        assert _bit_equal(a, b), k


def _first(x, k):
    """the first k rays of an input (arrays, tuples of them, None)"""
    if x is None:
        return None
    return tuple(_first(y, k) for y in x) if isinstance(x, tuple) else x[:k]


@pytest.mark.gpu
def test_a_smaller_call_after_a_larger_one_matches_a_fresh_workspace():
    """40 rays after 64 on the same workspace give the outputs and views of 40 rays on a fresh one"""
    row = ("elu", (2, 8, True), 10, "softplus", (64, 64, 128), "noise", False, "blender", False)
    mlps = _scene_mlps(7, row[1], row[2], row[0])
    inputs = _row_inputs(row, 7)
    runs = []
    for warm in (True, False):
        model = _row_model(row, mlps)
        model.workspace().fill_(0xFF)
        if warm:
            _call(model, *inputs)
        out = _call(model, *(_first(x, 40) for x in inputs))
        runs.append(_outputs_and_views(model, out, 40))
    for k, (a, b) in enumerate(zip(*runs)):
        assert _bit_equal(a, b), k

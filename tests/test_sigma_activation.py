"""The softplus density (flag sigma_activation, nerf_sh/nerf/utils.py:153; models.py:280-281): the oracle against the
reference executed with nn.softplus, the flag's scope, and on the GPU the heads epilogue, the compositing backward, the
whole gradient and the CLIs.  oracle/nerf_sh_oracle.py applies relu; NerfModel.__call__ and loss_fn are restated below
with the activation as a parameter, from the oracle's own stages, and held bit-identical to it with relu.  The golden
ref_softplus.npz comes from tests/golden/make_golden_softplus.py.

Bounds (u = 2^-24):
- sigma = softplus(x) is formed in fp32 as max(x, 0) + log1pf(expf(-|x|)).  expf is within 2 ulp, log1pf within 1 ulp;
  for x >= 0 the log term is at most ln 2 <= sigma and the final add rounds once, for x < 0 the max is 0 and the log
  term carries expf's relative error through log1p's condition number (<= 1).  So |sigma - softplus64(x)| <=
  SP_BAR * u * softplus64(x), x the kernel's own fp32 argument (raw sigma plus noise); below x = -87 expf's output is
  denormal, which adds 2^-149 absolute (SP_FLOOR).
- G.w = dalpha * delta * exp(-sigma delta) * (-expm1f(-sigma)): test_ray_stages.py's magnitude of the relu factor's
  G.w, plus expm1f's 1 ulp (2 u relative) and the one more product (u / 2): GW_SP_EXTRA = 2.5 u |G.w|.
"""
import functools
import os

import numpy as np
import pytest
import torch

from tests.support.mlp_stages import CASES
from tests.support.model_flags import SP_BAR, SP_FLOOR, _scope_args, softplus64
from tests.support.ray_stages import GUARD, GW_BAR, GW_SP_EXTRA, RayCase, U24, _norm, composite_bwd_ref, composite_ref
from tests.support.records import record


_record = functools.partial(record, "parity_sigma_activation.json")


def _sp_excess(sigma, x):
    """max over rows of |sigma - softplus64(x)| / (u softplus64(x) + SP_FLOOR / SP_BAR), in units of u * softplus64"""
    ref = softplus64(x)
    err = (sigma.double() - ref).abs()
    return float((err / (U24 * ref + SP_FLOOR / SP_BAR)).max())


# =====================================================================================================================
# The oracle's NerfModel.__call__ and loss_fn (oracle/nerf_sh_oracle.py, which applies relu) restated with the density
# activation as a parameter, from the oracle's own stages.  Softplus is flax's nn.softplus, logaddexp(x, 0); its
# autograd derivative is sigmoid(x).
# =====================================================================================================================
def sigma_act_fn(name):
    name = str(name).lower()
    if name == "relu":
        return torch.relu
    if name == "softplus":
        return lambda x: torch.logaddexp(x, torch.zeros_like(x))
    raise ValueError(f"sigma_activation {name!r}")


def render_level_act(params, sh_deg, z_vals, samples, rays, white_bkgd, sigma_noise, act):
    """oracle.render_level with sigma = act(raw sigma + noise) (nerf_sh/nerf/models.py:280-281)"""
    from oracle import nerf_sh_oracle as O
    _, _, viewdirs = rays
    raw_rgb, raw_sigma = O.mlp(params, O.posenc(samples))
    raw_sigma = O.add_gaussian_noise(raw_sigma, sigma_noise)
    if sh_deg >= 0:
        K = (sh_deg + 1) ** 2
        raw_rgb = O.eval_sh(sh_deg, raw_rgb.reshape(*raw_rgb.shape[:-1], -1, K), viewdirs[:, None])
    comp_rgb, disp, acc, weights = O.volumetric_rendering(torch.sigmoid(raw_rgb), sigma_act_fn(act)(raw_sigma),
                                                          z_vals, rays[1], white_bkgd)
    return (comp_rgb, disp, acc), weights


def nerf_forward_act(params_c, params_f, sh_deg, rays, num_coarse, num_fine, near, far, white_bkgd=True, t_rand=None,
                     u=None, z_fine=None, sigma_noise=None, act="relu"):
    """oracle.nerf_forward with the density activation `act`: -> ([(rgb, disp, acc) per level], fine depths)"""
    from oracle import nerf_sh_oracle as O
    origins, directions, _ = rays
    z_vals, samples = O.sample_along_rays(origins, directions, num_coarse, near, far, t_rand)
    noise_c, noise_f = sigma_noise if sigma_noise is not None else (None, None)
    out_c, weights = render_level_act(params_c, sh_deg, z_vals, samples, rays, white_bkgd, noise_c, act)
    ret, zf = [out_c], None
    if num_fine > 0:
        if z_fine is not None:
            z_vals, samples = z_fine, O.cast_rays(z_fine, origins, directions)
        else:
            z_mid = 0.5 * (z_vals[..., 1:] + z_vals[..., :-1])
            z_vals, samples = O.sample_pdf(z_mid, weights[..., 1:-1], origins, directions, z_vals, num_fine, u)
        out_f, _ = render_level_act(params_f, sh_deg, z_vals, samples, rays, white_bkgd, noise_f, act)
        ret.append(out_f)
        zf = z_vals
    return ret, zf


def loss_fn_act(params_c, params_f, sh_deg, rays, pixels, cfg, t_rand=None, u=None, sp_points=None, z_fine=None,
                act="relu"):
    """oracle.loss_fn with the density activation `act`; the sparsity term keeps relu of raw sigma (train.py:82)"""
    import math
    from oracle import nerf_sh_oracle as O
    ret, zf = nerf_forward_act(params_c, params_f, sh_deg, rays, cfg["num_coarse_samples"], cfg["num_fine_samples"],
                               cfg["near"], cfg["far"], cfg["white_bkgd"], t_rand, u, z_fine, act=act)
    if cfg.get("sparsity_weight", 0.0) > 0.0 and sp_points is not None:
        _, sp_sigma = O.eval_points_raw(params_f if cfg["num_fine_samples"] > 0 else params_c, sp_points)
        loss_sp = cfg["sparsity_weight"] * (1.0 - torch.exp(-cfg["sparsity_length"] * torch.relu(sp_sigma)).mean())
    else:
        loss_sp = torch.zeros((), dtype=pixels.dtype)
    loss = ((ret[-1][0] - pixels[..., :3]) ** 2).mean()
    loss_c = ((ret[0][0] - pixels[..., :3]) ** 2).mean() if len(ret) > 1 else torch.zeros((), dtype=pixels.dtype)
    psnr = lambda x: -10.0 * torch.log(x) / math.log(10.0)
    all_p = [t for ps in (params_c, params_f) for wb in ps for t in wb]
    weight_l2 = sum((t ** 2).sum() for t in all_p) / sum(t.numel() for t in all_p)
    total = loss + loss_c + loss_sp + cfg.get("weight_decay_mult", 0.0) * weight_l2
    return total, dict(loss=loss, psnr=psnr(loss), loss_c=loss_c, psnr_c=psnr(loss_c) if len(ret) > 1 else loss_c,
                       loss_sp=loss_sp, weight_l2=weight_l2, _z_fine=zf)


def loss_and_grads_act(flat_c, flat_f, sh_deg, rays, pixels, cfg, t_rand, u, sp_points, dtype, z_fine=None,
                       act="relu"):
    """oracle.loss_and_grads with the density activation: -> (stats, flat gradient [MLP_0 | MLP_1] as float64)"""
    from oracle import nerf_sh_oracle as O
    fc = torch.tensor(np.asarray(flat_c), dtype=dtype, requires_grad=True)
    ff = torch.tensor(np.asarray(flat_f), dtype=dtype, requires_grad=True)
    cast = lambda a: None if a is None else torch.as_tensor(np.asarray(a)).to(dtype)
    total, stats = loss_fn_act(O.unflatten(fc, sh_deg), O.unflatten(ff, sh_deg), sh_deg, tuple(cast(r) for r in rays),
                               cast(pixels), cfg, cast(t_rand), cast(u), cast(sp_points), cast(z_fine), act=act)
    total.backward()
    zf = stats.pop("_z_fine")
    stats = {k: float(v.detach()) for k, v in stats.items()}
    stats["_z_fine"] = None if zf is None else zf.detach().numpy()
    return stats, np.concatenate([fc.grad.numpy(), ff.grad.numpy()]).astype(np.float64)


def test_restated_oracle_with_relu_equals_the_oracle():
    """with relu the restatement above computes what oracle/nerf_sh_oracle.py computes, bit for bit"""
    from oracle import nerf_sh_oracle as O
    from tests.support.mlp_stages import _setup
    fc, ff, rays, px, t_rand, u, sp = _setup(3, 6, 16, 20, 5)
    cfg = dict(num_coarse_samples=64, num_fine_samples=16, near=2.0, far=6.0, white_bkgd=True, sparsity_weight=1e-3,
               sparsity_length=0.05, weight_decay_mult=0.1)
    st_o, gc, gf = O.loss_and_grads(fc, ff, 3, rays, px, cfg, t_rand, u, sp)
    st_a, g = loss_and_grads_act(fc, ff, 3, rays, px, cfg, t_rand, u, sp, torch.float32)
    assert np.array_equal(st_o.pop("_z_fine"), st_a.pop("_z_fine"))
    assert st_o == st_a
    assert np.array_equal(np.concatenate([gc, gf]).astype(np.float64), g)


# =====================================================================================================================
# CPU: the oracle against the executed reference, the flag's scope, the ABI
# =====================================================================================================================
def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def _golden(golden_dir):
    from oracle import nerf_sh_oracle as O
    g = np.load(os.path.join(golden_dir, "ref_softplus.npz"))
    sh = int(g["sh_deg"])
    flats = []
    for s in g["seeds"]:
        f = O.init_flat_params(sh, int(s), bias_scale=0.05)
        w8 = sum(a * b + b for a, b in O.layer_dims(sh)[:8])
        f[w8:w8 + 256] *= float(g["sigma_head_scale"])
        flats.append(f)
    return g, sh, [O.unflatten(f, sh) for f in flats]


@pytest.mark.parametrize("act", ["softplus", "relu"])
def test_oracle_forward_matches_executed_reference_softplus(golden_dir, act):
    """NerfModel.__call__ with nn.softplus, both levels, deterministic and with injected draws: the oracle with softplus
    within test_oracle.py's tolerances; with relu it must miss them by far (the golden pins the activation)."""
    from oracle import nerf_sh_oracle as O
    g, sh, (pc, pf) = _golden(golden_dir)
    rays = (_t(g["origins"]), _t(g["directions"]), _t(g["viewdirs"]))
    worst = 0.0
    for tag, t_rand, u in (("det", None, None), ("rand", _t(g["t_rand"]), _t(g["u"]))):
        with torch.no_grad():
            ret, _ = nerf_forward_act(pc, pf, sh, rays, 64, 128, 2.0, 6.0, True, t_rand=t_rand, u=u, act=act)
        for lvl, (rgb, disp, acc) in zip(("coarse", "fine"), ret):
            tol = 2e-5 if lvl == "coarse" else 5e-4
            e = max(float(np.abs(rgb.numpy() - g[f"call_{tag}_{lvl}_rgb"]).max()),
                    float(np.abs(acc.numpy() - g[f"call_{tag}_{lvl}_acc"]).max())) / tol
            worst = max(worst, e)
            if act == "softplus":
                np.testing.assert_allclose(rgb.numpy(), g[f"call_{tag}_{lvl}_rgb"], rtol=0, atol=tol)
                np.testing.assert_allclose(acc.numpy(), g[f"call_{tag}_{lvl}_acc"], rtol=0, atol=tol)
                np.testing.assert_allclose(disp.numpy(), g[f"call_{tag}_{lvl}_disp"], rtol=20 * tol)
    if act == "relu":
        assert worst > 20.0, worst


def test_oracle_loss_matches_executed_reference_softplus(golden_dir):
    """train_step.loss_fn with nn.softplus density; the sparsity term keeps nn.relu of raw sigma"""
    from oracle import nerf_sh_oracle as O
    g, sh, (pc, pf) = _golden(golden_dir)
    r = np.float32(g["sparsity_radius"])
    sp = (g["sp01"] * np.float32(r - (-r)) + np.float32(-r)).astype(np.float32)
    cfg = dict(num_coarse_samples=64, num_fine_samples=128, near=2.0, far=6.0, white_bkgd=True,
               sparsity_weight=float(g["sparsity_weight"]), sparsity_length=float(g["sparsity_length"]),
               weight_decay_mult=float(g["weight_decay_mult"]))
    rays = (_t(g["origins"]), _t(g["directions"]), _t(g["viewdirs"]))
    with torch.no_grad():
        total, st = loss_fn_act(pc, pf, sh, rays, _t(g["pixels"]), cfg, _t(g["t_rand"]), _t(g["u"]), _t(sp),
                                act="softplus")
    for k, tol in (("loss", 3e-4), ("loss_c", 2e-5), ("loss_sp", 1e-4), ("weight_l2", 1e-6), ("psnr", 3e-4),
                   ("psnr_c", 2e-5)):
        assert abs(float(st[k]) - float(g[k])) <= tol * abs(float(g[k])), (k, float(st[k]), float(g[k]))
    want = float(g["loss"]) + float(g["loss_c"]) + float(g["loss_sp"]) + float(g["weight_decay_mult"]) * float(g["weight_l2"])
    assert abs(float(total) - want) < 3e-4 * want
    # a softplus sparsity term would be far off: softplus(x) > relu(x) everywhere
    with torch.no_grad():
        _, s_raw = O.eval_points_raw(pf, _t(sp))
        alt = float(g["sparsity_weight"]) * (1.0 - torch.exp(-float(g["sparsity_length"]) * softplus64(s_raw)).mean())
    assert abs(float(alt) - float(g["loss_sp"])) > 100 * 1e-4 * abs(float(g["loss_sp"]))


def test_check_scope_sigma_activation():
    from plenoctree_b200.nerf import flags as F
    for name, code in (("relu", 0), ("ReLU", 0), ("softplus", 1), ("Softplus", 1), ("SOFTPLUS", 1)):
        F.check_scope(_scope_args(sigma_activation=name))
        F.check_scope(_scope_args(sigma_activation=name, net_activation="ReLU", rgb_activation="Sigmoid"))
        assert F.sigma_activation_code(name) == code
    for bad in ("sigmoid", "elu", "softmax", "Sigmoid", "shifted_softplus"):
        with pytest.raises(NotImplementedError):
            F.check_scope(_scope_args(sigma_activation=bad))
    for kw in (dict(net_activation="gelu"), dict(net_activation="swish", sigma_activation="softplus"),
               dict(rgb_activation="relu", sigma_activation="softplus")):
        with pytest.raises(NotImplementedError):
            F.check_scope(_scope_args(**kw))


def test_abi_sigma_activation():
    from plenoctree_b200 import _lib
    assert _lib.RenderConfig(3, 64, 128, 1, 4096, 10000).sigma_activation == 0
    assert _lib.RenderConfig().sigma_activation == 0
    assert (_lib.SIGMA_RELU, _lib.SIGMA_SOFTPLUS) == (0, 1)
    assert _lib.lib.pob_abi_version() == 8
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                            "plenoctree_b200.h")).read()
    assert "#define POB_SIGMA_RELU 0" in hdr and "#define POB_SIGMA_SOFTPLUS 1" in hdr
    assert "pob_eval_points_act" in _lib.SIGNATURES


# =====================================================================================================================
# GPU
# =====================================================================================================================
def _eval_act(blob, sh, pts, vd, act, prec):
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    m = pts.shape[0]
    out = torch.full((m + 1024, 4), float("nan"), device="cuda")
    check(lib.pob_eval_points_act(ptr(blob), sh, ptr(pts), ptr(vd), m, ptr(out), act, prec, stream_ptr()))
    torch.cuda.synchronize()
    assert bool(out[m:].isnan().all()), "write past the output"
    return out[:m]


@pytest.mark.gpu
@pytest.mark.parametrize("sh", [-1, 3, 4])
@pytest.mark.parametrize("prec", [1, 3], ids=["fp16", "fp16x3"])
def test_eval_points_act_vs_fp64(sh, prec):
    """pob_eval_points_act: sigma within SP_BAR of fp64 softplus of the same precision's OUT_RAW sigma at the same
    points (raw spans about +-60 through a scaled Dense_8); rgb bit-identical to relu mode; relu mode bit-identical
    to pob_eval_points; an unknown activation refused"""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    from plenoctree_b200._lib import PobError, check, lib, ptr, stream_ptr
    flat = O.init_flat_params(sh, 91, bias_scale=0.05)
    w8 = sum(a * b + b for a, b in O.layer_dims(sh)[:8])
    flat[w8:w8 + 256] *= 40.0
    blob = ops.pack_weights(torch.from_numpy(flat).cuda(), sh)
    m = 132 * 128 * 3 + 77
    rs = np.random.RandomState(5 + sh)
    pts = torch.from_numpy(rs.uniform(-1.5, 1.5, size=(m, 3)).astype(np.float32)).cuda()
    vd = torch.nn.functional.normalize(torch.from_numpy(rs.normal(size=(m, 3)).astype(np.float32)), dim=-1).cuda()
    _, raw = ops.eval_points_raw(blob, sh, pts, want_rgb=False, precision=prec)
    raw = raw[:, 0]
    sp = _eval_act(blob, sh, pts, vd, 1, prec)
    re = _eval_act(blob, sh, pts, vd, 0, prec)
    plain = torch.empty((m, 4), device="cuda")
    check(lib.pob_eval_points(ptr(blob), sh, ptr(pts), ptr(vd), m, ptr(plain), prec, stream_ptr()))
    torch.cuda.synchronize()
    rep = dict(sp_excess=_sp_excess(sp[:, 3], raw), raw_min=float(raw.min()), raw_max=float(raw.max()),
               raw_negative_share=float((raw < 0).double().mean()),
               rgb_bit_mismatches=int((sp[:, :3] != re[:, :3]).sum()),
               relu_vs_pob_eval_points_mismatches=int((re != plain).sum()),
               relu_sigma_vs_raw_mismatches=int((re[:, 3] != raw.clamp_min(0)).sum()))
    _record(f"eval_points_act_sh{sh}_{'x3' if prec == 3 else 'fp16'}", rep)
    assert rep["sp_excess"] <= SP_BAR, rep
    assert rep["raw_min"] < -10 and rep["raw_max"] > 10, rep           # both branches, far into the tails
    assert rep["rgb_bit_mismatches"] == 0 and rep["relu_vs_pob_eval_points_mismatches"] == 0, rep
    assert rep["relu_sigma_vs_raw_mismatches"] == 0, rep
    with pytest.raises(PobError):
        check(lib.pob_eval_points_act(ptr(blob), sh, ptr(pts), ptr(vd), m, ptr(plain), 2, prec, stream_ptr()))


class SoftplusCase(RayCase):
    """a training call of test_ray_stages.py with the softplus density"""

    def __init__(self, *a, **k):
        super().__init__(*a, sigma_act="softplus", **k)

    @property
    def name(self):
        return super().name + "_softplus"


def _level_points(ctx, lv, z, sp, dev):
    from tests.support.eval_stages import _level_rows
    return _level_rows(ctx, lv, z, sp, dev)


def _softplus_call(case):
    """one softplus training call and the render of the same rays, draws and noise: per level the bit mismatches of
    the training rows against the render's, the sigma bound of the ray rows against fp64 softplus of OUT_RAW at the
    same points (+ noise in fp32, as the epilogue adds it), the sparsity rows against relu of OUT_RAW, and G (the
    compositing backward) against fp64 with the softplus factor"""
    from plenoctree_b200 import layouts as L, ops
    from plenoctree_b200.nerf.models import Rays
    from plenoctree_b200.nerf.train import default_loss_scale
    dev = torch.device("cuda")
    model = case.model()
    n = case.R
    _, ctx = case.run(model, n=n, fill=0xFF)
    (o, d, v, px), t_rand, u, sp, noise = case.inputs(n)
    ws = model.workspace(True, case.precision)
    views = L.train_workspace_views(model.cfg, n, case.nsp > 0, precision=case.precision)
    names = ("z", "rgbs", "weights", "comp", "disp", "acc")
    saved = [{k: L.workspace_view(ws, lv, k).clone() for k in names} for lv in views["levels"]]
    ls = default_loss_scale(n, case.precision)
    gscale = ls * 2.0 / (3.0 * n)
    res = {}
    dt = torch.from_numpy(d).to(dev)
    spt = torch.from_numpy(sp).to(dev) if sp is not None else None
    for i, lv in enumerate(views["levels"]):
        N, Mr, M = lv["N"], lv["M_rays"], lv["M"]
        r = {}
        rgbs = saved[i]["rgbs"]
        x, _ = _level_points(ctx, lv, saved[i]["z"], spt if i == len(views["levels"]) - 1 else None, dev)
        _, raw = ops.eval_points_raw(model.blobs[i], case.sh, x, want_rgb=False, precision=case.precision)
        raw = raw[:, 0]
        arg = raw[:Mr].clone()
        if noise is not None and noise[i] is not None:
            arg = arg + torch.from_numpy(noise[i]).to(dev).reshape(-1)          # fp32, as the epilogue adds it
        r["sigma_excess"] = _sp_excess(rgbs[:Mr, 3], arg)
        r["sparsity_rows_vs_relu_raw_mismatches"] = int((rgbs[Mr:M, 3] != raw[Mr:M].clamp_min(0)).sum())
        # compositing backward with the softplus factor, from the kernel's own inputs
        z = saved[i]["z"]
        rr = rgbs[:Mr].view(n, N, 4)
        f = composite_ref(rr[..., :3], rr[..., 3], z, dt, model.white_bkgd)
        sig = rr[..., 3].double()
        fac = f["delta"] * f["a"] * (-torch.expm1(-sig))
        b = composite_bwd_ref(f, saved[i]["comp"], torch.from_numpy(px).to(dev), gscale, factor=fac)
        b["mag_gw"] = b["mag_gw"] + GW_SP_EXTRA * b["Gw"].abs()
        G = L.workspace_view(ws, lv, "G")[:Mr].view(n, N, 4)
        r["G_w"] = float(_norm((G[..., 3].double() - b["Gw"]).abs(), b["mag_gw"]).max())
        r["G_nonfinite"] = int((~torch.isfinite(G)).sum())
        b_relu = composite_bwd_ref(f, saved[i]["comp"], torch.from_numpy(px).to(dev), gscale)
        r["relu_factor_guard"] = float(_norm((b_relu["Gw"] - b["Gw"]).abs(), b["mag_gw"]).max())
        res[f"level{i}"] = r
    # the render call: same draws, same precision, its own workspace
    rws = model.workspace(False)
    rws.fill_(0xFF)
    model(Rays(o, d, v), randomized=True, t_rand=t_rand, u=u, sigma_noise=noise, precision=case.precision)
    torch.cuda.synchronize()
    rv = L.train_workspace_views(model.cfg, n, False, training=False)
    for i, (lt, lr) in enumerate(zip(views["levels"], rv["levels"])):
        Mr = lt["M_rays"]
        bad = 0
        for k in ("z", "weights", "comp", "disp", "acc"):
            bad += int((L.workspace_view(rws, lr, k).view(torch.int32) != saved[i][k].view(torch.int32)).sum())
        bad += int((L.workspace_view(rws, lr, "rgbs").view(torch.int32) != saved[i]["rgbs"][:Mr].view(torch.int32)).sum())
        res[f"level{i}"]["render_vs_training_bit_mismatches"] = bad
    return res


def _assert_softplus_call(res):
    for k, r in res.items():
        assert r["render_vs_training_bit_mismatches"] == 0, (k, r)
        assert r["sparsity_rows_vs_relu_raw_mismatches"] == 0, (k, r)
        assert r["sigma_excess"] <= SP_BAR, (k, r)
        assert r["G_nonfinite"] == 0 and r["G_w"] <= GW_BAR, (k, r)
        assert r["relu_factor_guard"] >= GUARD * GW_BAR, (k, r)


SOFTPLUS_CASES = ([SoftplusCase(c.sh, c.R, c.nc, c.nf, c.nsp, noise=c.noise, seed=c.seed,
                                sparsity_weight=c.sparsity_weight, sp_radius=c.sp_radius, precision=p)
                   for p in (1, 3) for c in CASES])


@pytest.mark.gpu
@pytest.mark.parametrize("case", SOFTPLUS_CASES, ids=lambda c: c.name)
def test_softplus_training_rows_match_render(case):
    res = _softplus_call(case)
    _record(case.name, res)
    _assert_softplus_call(res)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [1, 3], ids=["fp16", "fp16x3"])
def test_softplus_production_step(prec):
    """the bench.py step (4096 rays x (64 + 128) + 10 000 sparsity points)"""
    from plenoctree_b200._lib import RenderConfig, lib
    from plenoctree_b200.nerf.models import ctypes_ref
    cfg = RenderConfig(3, 64, 128, 1, 4096, 10000)
    need = int(lib.pob_train_workspace_bytes(ctypes_ref(cfg), prec)) + int(lib.pob_workspace_bytes(ctypes_ref(cfg), 0))
    free, _ = torch.cuda.mem_get_info()
    if free < need + (6 << 30):
        pytest.skip(f"the production step needs {need / 2**30:.1f} GB of workspaces + ~6 GB; {free / 2**30:.1f} GB free")
    case = SoftplusCase(3, 4096, 64, 128, 10000, precision=prec)
    res = _softplus_call(case)
    _record(case.name, res)
    _assert_softplus_call(res)


@pytest.mark.gpu
def test_softplus_gradient_vs_fp64_oracle():
    """test_train_x3.py's whole-gradient check with the softplus density: fp16x3 at the oracle's own fp32 floor and
    GRAD_GAIN times closer to the fp32 oracle than the fp16 step; the fp16 step within test_train.py's gates"""
    from plenoctree_b200.nerf import train as T
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from tests.support.mlp_stages import FLOOR_SLACK, GRAD_GAIN, LOSS_REL, X3, _setup
    R, nf, nsp = 96, 128, 300
    fc, ff, rays, px, t_rand, u, sp = _setup(3, R, nf, nsp, 77)
    cfg = dict(num_coarse_samples=64, num_fine_samples=nf, near=2.0, far=6.0, white_bkgd=True,
               sparsity_weight=1e-3, sparsity_length=0.05)
    stats_o, ref = loss_and_grads_act(fc, ff, 3, rays, px, cfg, t_rand, u, sp, torch.float64, act="softplus")
    zf = stats_o.pop("_z_fine").astype(np.float32)
    _, ref32 = loss_and_grads_act(fc, ff, 3, rays, px, cfg, t_rand, u, sp, torch.float32, z_fine=zf, act="softplus")
    _, ref_relu = loss_and_grads_act(fc, ff, 3, rays, px, cfg, t_rand, u, sp, torch.float64, z_fine=zf, act="relu")
    rel = lambda g, r: float(np.linalg.norm(g - r) / np.linalg.norm(r))
    model = NerfModel(sh_deg=3, num_coarse_samples=64, num_fine_samples=nf, max_rays=R, sparsity_npoints=nsp,
                      sigma_activation="softplus")
    model.set_params(np.concatenate([fc, ff]))
    rep = {"fp32_oracle_vs_fp64": rel(ref32, ref), "relu_oracle_vs_softplus": rel(ref_relu, ref)}
    for name, prec in (("fp16", 1), ("fp16x3", X3)):
        state = T.TrainState(model)
        n = T.loss_and_grad(model, state, {"rays": Rays(*rays), "pixels": px}, sparsity_weight=1e-3,
                            sparsity_length=0.05, randomized=True, t_rand=t_rand, u=u, sp_points=sp, z_fine=zf,
                            precision=prec)
        torch.cuda.synchronize()
        g = state.grads.double().cpu().numpy()
        st = T.stats_from_raw(state.stats_raw, n, 1e-3, nsp, True)
        rep[name] = dict(grad_rel_l2=rel(g, ref), grad_rel_l2_vs_fp32_oracle=rel(g, ref32),
                         cosine=float(np.dot(g, ref) / (np.linalg.norm(g) * np.linalg.norm(ref))),
                         loss_rel=abs(st.loss - stats_o["loss"]) / stats_o["loss"],
                         loss_c_rel=abs(st.loss_c - stats_o["loss_c"]) / stats_o["loss_c"],
                         loss_sp_abs=abs(st.loss_sp - stats_o["loss_sp"]))
    rep["gain_vs_fp32_oracle"] = rep["fp16"]["grad_rel_l2_vs_fp32_oracle"] / rep["fp16x3"]["grad_rel_l2_vs_fp32_oracle"]
    _record("gradient_vs_fp64_oracle", rep)
    x, h = rep["fp16x3"], rep["fp16"]
    assert x["loss_rel"] < LOSS_REL and x["loss_c_rel"] < LOSS_REL, rep
    assert x["loss_sp_abs"] < LOSS_REL * max(abs(stats_o["loss_sp"]), 1e-6) + 1e-8, rep
    assert x["grad_rel_l2"] <= FLOOR_SLACK * rep["fp32_oracle_vs_fp64"], rep
    assert rep["gain_vs_fp32_oracle"] >= GRAD_GAIN, rep
    assert h["loss_rel"] < 5e-3 and h["loss_c_rel"] < 5e-3, rep
    assert h["loss_sp_abs"] < 2e-3 * max(abs(stats_o["loss_sp"]), 1e-6) + 1e-7, rep
    assert h["grad_rel_l2"] < 2e-2 and h["cosine"] > 0.9995, rep
    assert rep["relu_oracle_vs_softplus"] > 100 * rep["fp16x3"]["grad_rel_l2"], rep    # the check sees the activation


@pytest.mark.gpu
def test_cli_train_eval_extract_softplus(tmp_path):
    """nerf_sh.train --sigma_activation softplus learns a synthetic scene, nerf_sh.eval renders it, and
    octree.extraction builds the same tree with --sigma_activation softplus as with relu (it reads raw sigma)."""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf import datasets as D, flags as F
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf.utils import generate_rays, pose_spherical, render_image
    from plenoctree_b200.nerf_sh import eval as EV, train as TR
    from plenoctree_b200.octree import extraction as EX
    sh_deg, W = 3, 48
    ft = np.concatenate([O.init_flat_params(sh_deg, 7001, bias_scale=0.05), O.init_flat_params(sh_deg, 7002, bias_scale=0.05)])
    P = O.param_count(sh_deg)
    for m in range(2):
        off = m * P + P - 48 - 1 - 256 * 48 - 256
        ft[off:off + 256] *= 30.0
    teacher = NerfModel(sh_deg=sh_deg, max_rays=4096)
    teacher.set_params(ft)
    cam_x = 0.6911112070083618
    focal = 0.5 * W / np.tan(0.5 * cam_x)
    rs = np.random.RandomState(3)
    splits = {"train": 8, "val": 2, "test": 2}
    poses = {k: [pose_spherical(rs.uniform(-180, 180), rs.uniform(-80, -10), 4.0) for _ in range(n)] for k, n in splits.items()}
    images = {}
    for k in splits:
        rays = generate_rays(W, W, focal, np.stack(poses[k]))
        images[k] = [render_image(teacher, Rays(rays.origins[i], rays.directions[i], rays.viewdirs[i]))[0].cpu().numpy()
                     for i in range(splits[k])]
    data_dir, train_dir = str(tmp_path / "scene"), str(tmp_path / "ckpt")
    D.write_blender_scene(data_dir, images, poses, cam_x)
    (tmp_path / "cfg.yaml").write_text("dataset: blender\nfactor: 0\nnum_coarse_samples: 64\nnum_fine_samples: 128\n"
                                       "use_viewdirs: false\nwhite_bkgd: true\nbatch_size: 1024\nsh_deg: 3\n"
                                       "randomized: true\nmax_steps: 200\nsigma_activation: softplus\n")
    EX._define_cli_flags()
    F.define_flags()
    FLAGS = F.FLAGS
    if not FLAGS.is_parsed():
        FLAGS.mark_as_parsed()
    new = dict(train_dir=train_dir, data_dir=data_dir, config=str(tmp_path / "cfg"), save_every=200, print_every=100,
               render_every=0, sparsity_npoints=1000, lr_init=2e-3, lr_final=2e-4, chunk=4096, noise_std=None,
               image_batching=True, is_jaxnerf_ckpt=True, init_grid_depth=5, samples_per_cell=8, masking_mode="sigma",
               alpha_thresh=1e-6, renderer_step_size=1e-3, radius="1.5", eval=False, output=None)
    old = {k: getattr(FLAGS, k) for k in list(new) + ["sigma_activation", "max_steps"]}
    try:
        for k, v in new.items():
            setattr(FLAGS, k, v)
        model, state = TR.main(None)
        assert model.sigma_act_code == 1 and model.cfg.sigma_activation == 1 and state.step == 200
        psnr, _ = EV.main(None)
        fresh = NerfModel(sh_deg=sh_deg, max_rays=4096, sigma_activation="softplus")
        fresh.init_params(20200823)
        rays = generate_rays(W, W, focal, np.stack(poses["test"]))
        gt = torch.from_numpy(images["test"][0]).cuda()
        p_init = -10 * np.log10(float(((render_image(fresh, Rays(rays.origins[0], rays.directions[0],
                                                                  rays.viewdirs[0]))[0] - gt) ** 2).mean()))
        FLAGS.config = None
        trees = {}
        for act in ("softplus", "relu"):
            FLAGS.sigma_activation = act
            FLAGS.output = str(tmp_path / f"tree_{act}.npz")
            EX.main(None)
            trees[act] = dict(np.load(FLAGS.output))
        _record("cli", dict(psnr_init=p_init, psnr_200_steps=psnr))
        assert psnr > p_init + 2.0, (p_init, psnr)
        assert sorted(trees["softplus"]) == sorted(trees["relu"])
        for k in trees["relu"]:
            assert np.array_equal(trees["softplus"][k], trees["relu"][k]), k
    finally:
        for k, v in old.items():
            setattr(FLAGS, k, v)

"""Up to 1024 samples per ray (flags num_coarse_samples / num_fine_samples; nerf_sh/nerf/model_utils.py:104-142,
289-314): the bound and its refusals, the oracle against the reference executed at (128, 384) and (256, 768)
(ref_long_rays.npz, from tests/golden/make_golden_long_rays.py), a numpy model of the four-warp kernels' fp32 order
against test_ray_stages.py's fp64 bars, and on the GPU the wide per-ray kernels (one 128-thread block per ray for
256 < N <= 1024), the training and render calls, graph replay and the CLI.

The fp64 references, the order-independent bars and the GPU wrappers are test_ray_stages.py's, used unchanged.
"""
import os

import numpy as np
import pytest
import torch

import tests.test_ray_stages as RS
from tests.test_ray_stages import (ACC_BAR, GUARD, GW_BAR, RayCase, _norm, _t, assert_composite, assert_pdf,
                                   check_composite, check_composite_bwd, check_pdf, composite_bwd_ref, composite_ref,
                                   emu_delta, pdf_families, ray_families)

ACCEPT = [(3, 0), (1024, 0), (128, 384), (256, 768), (64, 960)]
REFUSE = [(2, 0), (512, 513), (1025, 0)]
LONG_N = [257, 288, 289, 384, 640, 1000, 1024]
LONG_PDF = [(3, 1021), (128, 384), (256, 768), (1000, 24), (1023, 1)]


# =====================================================================================================================
# CPU: the bound
# =====================================================================================================================
def _scope(nc, nf):
    from tests.test_posenc import _scope_args
    a = _scope_args()
    a.num_coarse_samples, a.num_fine_samples = nc, nf
    return a


@pytest.mark.parametrize("nc,nf", ACCEPT)
def test_sample_counts_accepted(nc, nf):
    from plenoctree_b200.nerf import flags as F
    F.check_samples(nc, nf)
    F.check_model_scope(_scope(nc, nf))


@pytest.mark.parametrize("nc,nf", REFUSE)
def test_sample_counts_refused_with_the_bound(nc, nf):
    """flags.check_samples, check_model_scope (before any data is loaded) and NerfModel (before any device memory)
    refuse the same counts and name the bound"""
    from plenoctree_b200.nerf import flags as F
    from plenoctree_b200.nerf.models import NerfModel
    for call in (lambda: F.check_samples(nc, nf), lambda: F.check_model_scope(_scope(nc, nf)),
                 lambda: NerfModel(num_coarse_samples=nc, num_fine_samples=nf, max_rays=8)):
        with pytest.raises((ValueError, NotImplementedError)) as e:
            call()
        assert "num_coarse_samples + num_fine_samples <= 1024" in str(e.value)


# =====================================================================================================================
# CPU: the oracle against the executed reference at (128, 384) and (256, 768)
# =====================================================================================================================
def _golden(golden_dir):
    from oracle import nerf_sh_oracle as O
    g = np.load(os.path.join(golden_dir, "ref_long_rays.npz"))
    sh = int(g["sh_deg"])
    flats = []
    for s in g["seeds"]:
        f = O.init_flat_params(sh, int(s), bias_scale=0.05)
        w8 = sum(a * b + b for a, b in O.layer_dims(sh)[:8])
        f[w8:w8 + 256] *= float(g["sigma_head_scale"])
        flats.append(f)
    return g, sh, flats


@pytest.mark.parametrize("nc,nf", [(128, 384), (256, 768)])
def test_oracle_forward_matches_executed_reference_long_rays(golden_dir, nc, nf):
    """NerfModel.__call__, both levels, deterministic and with injected draws, within test_oracle.py's tolerances for
    ref_render.npz"""
    from oracle import nerf_sh_oracle as O
    g, sh, (fc, ff) = _golden(golden_dir)
    rays = (_t(g["origins"]), _t(g["directions"]), _t(g["viewdirs"]))
    tag_n = f"{nc}_{nf}"
    for tag, t_rand, u in (("det", None, None), ("rand", _t(g[f"t_rand_{tag_n}"]), _t(g[f"u_{tag_n}"]))):
        with torch.no_grad():
            ret = O.nerf_forward(O.unflatten(fc, sh), O.unflatten(ff, sh), sh, rays, nc, nf, 2.0, 6.0, True,
                                 t_rand=t_rand, u=u)
        for lvl, (rgb, disp, acc) in zip(("coarse", "fine"), ret):
            tol = 2e-5 if lvl == "coarse" else 5e-4
            key = f"call_{tag_n}_{tag}_{lvl}"
            np.testing.assert_allclose(rgb.numpy(), g[f"{key}_rgb"], rtol=0, atol=tol)
            np.testing.assert_allclose(acc.numpy(), g[f"{key}_acc"], rtol=0, atol=tol)
            np.testing.assert_allclose(disp.numpy(), g[f"{key}_disp"], rtol=20 * tol)


def test_oracle_loss_matches_executed_reference_long_rays(golden_dir):
    """train_step.loss_fn at (128, 384), within test_oracle.py's tolerances for ref_loss.npz"""
    from oracle import nerf_sh_oracle as O
    g, sh, (fc, ff) = _golden(golden_dir)
    nc, nf = (int(x) for x in g["loss_size"])
    r = np.float32(g["sparsity_radius"])
    sp = (g["sp01"] * np.float32(r - (-r)) + np.float32(-r)).astype(np.float32)
    cfg = dict(num_coarse_samples=nc, num_fine_samples=nf, near=2.0, far=6.0, white_bkgd=True,
               sparsity_weight=float(g["sparsity_weight"]), sparsity_length=float(g["sparsity_length"]),
               weight_decay_mult=float(g["weight_decay_mult"]))
    rays = (_t(g["origins"]), _t(g["directions"]), _t(g["viewdirs"]))
    with torch.no_grad():
        total, st = O.loss_fn(O.unflatten(fc, sh), O.unflatten(ff, sh), sh, rays, _t(g["pixels"]), cfg,
                              _t(g[f"t_rand_{nc}_{nf}"]), _t(g[f"u_{nc}_{nf}"]), _t(sp))
    for k, tol in (("loss", 3e-4), ("loss_c", 2e-5), ("loss_sp", 1e-4), ("weight_l2", 1e-6), ("psnr", 3e-4),
                   ("psnr_c", 2e-5)):
        assert abs(float(st[k]) - float(g[k])) <= tol * abs(float(g[k])), (k, float(st[k]), float(g[k]))
    want = float(g["loss"]) + float(g["loss_c"]) + float(g["loss_sp"]) + float(g["weight_decay_mult"]) * float(g["weight_l2"])
    assert abs(float(total) - want) < 3e-4 * want


# =====================================================================================================================
# CPU: numpy fp32 model of the four-warp kernels (W = 4: 128 threads per ray, S = ceil(N / 128) samples per thread)
# =====================================================================================================================
W4 = 4
f32 = np.float32


def _threads(x, S, fill):
    """[R, N] -> [R, 128, S]: thread t holds samples t*S .. t*S + S - 1 (padding `fill`)"""
    R, N = x.shape
    out = np.full((R, 32 * W4 * S), fill, f32)
    out[:, :N] = x
    return out.reshape(R, 32 * W4, S)


def _seq(x, op, init):
    """sequential fp32 reduce over the last axis"""
    acc = np.full(x.shape[:-1], init, f32)
    for i in range(x.shape[-1]):
        acc = op(acc, x[..., i]).astype(f32)
    return acc


def _block_excl(v, op, init, reverse=False):
    """exclusive scan over the 128 threads of a ray [R, 128] in the kernels' order: within each warp over its lanes,
    then the warps' totals (a warp's last lane's exclusive value combined with its own; for the suffix, its first
    lane's) in warp order from the front (reverse: from the last warp back)"""
    R = v.shape[0]
    v = v.reshape(R, W4, 32)
    ex = np.empty_like(v)
    acc = np.full((R, W4), init, f32)
    lanes = range(31, -1, -1) if reverse else range(32)
    for ln in lanes:
        ex[:, :, ln] = acc
        acc = op(acc, v[:, :, ln]).astype(f32)
    end = 0 if reverse else 31
    tot = op(ex[:, :, end], v[:, :, end]).astype(f32)
    other = np.empty((R, W4), f32)
    for w in range(W4):
        a = np.full(R, init, f32)
        for k in (range(W4 - 1, w, -1) if reverse else range(w)):
            a = op(a, tot[:, k]).astype(f32)
        other[:, w] = a
    return op(ex, other[:, :, None]).astype(f32).reshape(R, 32 * W4)


def emu_composite_wide(rgb, sigma, z, dirs, white, px=None, gscale=None, one_minus_alpha=False):
    """composite_fwd_kernel / composite_bwd_kernel at W = 4 in fp32: per-thread loops, the lane scans, the cross-warp
    steps of T0, of the five sums and of the suffix of g * w"""
    with np.errstate(all="ignore"):
        R, N = sigma.shape
        S = -(-N // (32 * W4))
        dn = np.sqrt(((dirs[:, 0] * dirs[:, 0] + dirs[:, 1] * dirs[:, 1]).astype(f32) + dirs[:, 2] * dirs[:, 2]).astype(f32))
        gap = np.concatenate([(z[:, 1:] - z[:, :-1]).astype(f32), np.full((R, 1), 1e10, f32)], 1)
        dist = (gap * dn[:, None]).astype(f32)
        ex = np.exp(-(sigma * dist).astype(f32).astype(np.float64)).astype(f32)
        alpha = (f32(1) - ex).astype(f32)
        om = ((f32(1) - alpha).astype(f32) + f32(1e-10)).astype(f32)
        omt, alt = _threads(om, S, 1.0), _threads(alpha, S, 0.0)
        T0 = _block_excl(_seq(omt, np.multiply, 1.0), np.multiply, 1.0)
        w = np.empty_like(alt)
        Tpre = np.empty_like(alt)
        T = T0.copy()
        for i in range(S):
            Tpre[..., i] = T
            w[..., i] = (alt[..., i] * T).astype(f32)
            T = (T * omt[..., i]).astype(f32)

        def tsum(x):      # [R, 128, S] -> per ray: thread, lane, then warp order
            return _seq(_seq(_seq(x, np.add, 0.0).reshape(R, W4, 32), np.add, 0.0), np.add, 0.0)
        zt = _threads(z, S, 0.0)
        acc = tsum(w)
        depth = tsum((w * zt).astype(f32))
        comp = np.stack([tsum((w * _threads(rgb[..., c], S, 0.0)).astype(f32)) for c in range(3)], -1)
        if white:
            comp = (comp + (f32(1) - acc)[:, None]).astype(f32)
        disp = (acc / depth).astype(f32)
        disp = np.where((disp > 0) & (disp < f32(1e10)) & (acc > f32(1e-10)), disp, f32(1e10)).astype(f32)
        wf = w.reshape(R, -1)[:, :N]
        if px is None:
            return comp, disp, acc, wf
        bg = f32(1) if white else f32(0)
        dc = (f32(gscale) * (comp - px).astype(f32)).astype(f32)
        gi = ((dc[:, None, :] * (rgb - bg).astype(f32)).astype(f32)).sum(-1, dtype=f32)
        git = _threads(gi, S, 0.0)
        local = _seq((git * w).astype(f32), np.add, 0.0)
        suffix = _block_excl(local, np.add, 0.0, reverse=True)
        fac = (dist * ((f32(1) - alpha).astype(f32) if one_minus_alpha else ex)).astype(f32)
        fact, sgt = _threads(fac, S, 0.0), _threads(sigma, S, 0.0)
        G = np.zeros((R, 32 * W4, S, 4), f32)
        for i in range(S - 1, -1, -1):
            dalpha = ((git[..., i] * Tpre[..., i]).astype(f32) - (suffix / omt[..., i]).astype(f32)).astype(f32)
            G[..., i, 3] = np.where(sgt[..., i] > 0, (dalpha * fact[..., i]).astype(f32), f32(0))
            suffix = (suffix + (git[..., i] * w[..., i]).astype(f32)).astype(f32)
        G = G.reshape(R, -1, 4)[:, :N]
        G[..., :3] = (wf[..., None] * dc[:, None] * rgb * (f32(1) - rgb)).astype(f32)
        sq = float((((comp - px).astype(f32)) ** 2).astype(f32).sum(dtype=f32))
        return comp, disp, acc, wf, G, sq


def emu_pdf_wide(zc, w, u):
    """sample_pdf_kernel at W = 4 in fp32: the weight sum and the cdf in the block's thread, lane and warp order"""
    R, Nc = zc.shape
    nb, nw = Nc - 1, Nc - 2
    S = -(-nw // (32 * W4))
    out = np.empty((R, Nc + u.shape[1]), f32)
    with np.errstate(all="ignore"):
        wl = _threads(w[:, 1:-1].astype(f32), S, 0.0)
        ws = _seq(_seq(_seq(wl, np.add, 0.0).reshape(R, W4, 32), np.add, 0.0), np.add, 0.0)
        pad = np.maximum(f32(0), (f32(1e-5) - ws).astype(f32))
        padw = (pad / f32(nw)).astype(f32)
        ws = (ws + pad).astype(f32)
        pdf = ((wl + padw[:, None, None]) / ws[:, None, None]).astype(f32)
        pdf.reshape(R, -1)[:, nw:] = 0
        pre = _block_excl(_seq(pdf, np.add, 0.0), np.add, 0.0)
        run = np.empty_like(pdf)
        for i in range(S):
            pre = (pre + pdf[..., i]).astype(f32)
            run[..., i] = pre
        run = run.reshape(R, -1)[:, :nw]
        for r in range(R):
            bins = (f32(0.5) * (zc[r, 1:] + zc[r, :-1])).astype(f32)
            cdf = np.empty(nb, f32)
            cdf[0], cdf[-1] = 0, 1
            cdf[1:nw] = np.minimum(f32(1), run[r, :nw - 1])
            lo = np.searchsorted(cdf, u[r], side="right")
            i0, i1 = np.maximum(lo - 1, 0), np.minimum(lo, nb - 1)
            t = ((u[r] - cdf[i0]).astype(f32) / (cdf[i1] - cdf[i0]).astype(f32)).astype(f32)
            t = np.clip(np.nan_to_num(t, nan=0.0), 0, 1).astype(f32)
            new = (bins[i0] + (t * (bins[i1] - bins[i0]).astype(f32)).astype(f32)).astype(f32)
            out[r] = np.sort(np.concatenate([zc[r], new]))
    return out


@pytest.mark.parametrize("N", [257, 384, 1024])
def test_emulated_wide_composite_within_bars(N):
    """the four-warp order passes every compositing bar of test_ray_stages.py; the (1 - alpha) factor still fails G.w
    on the opaque-first-sample rays, by >= GUARD x the bar from sigma delta = 10 on"""
    rgb, s, z, d, px, fam = ray_families(N, 1)
    gscale = 0.37
    for white in (True, False):
        f = composite_ref(_t(rgb), _t(s), _t(z), _t(d), white)
        comp, disp, acc, w, G, sq = emu_composite_wide(rgb, s, z, d, white, px, gscale)
        r = check_composite(f, _t(comp), _t(disp), _t(acc), _t(w))
        b = composite_bwd_ref(f, _t(comp), _t(px), gscale)
        r.update(check_composite_bwd(b, _t(G), sq))
        assert_composite(r)
        assert r["disp_kernel_acc_in_0_1e-10"] > 0, r
        bad = emu_composite_wide(rgb, s, z, d, white, px, gscale, one_minus_alpha=True)[4]
        gw = _norm((_t(bad)[..., 3].double() - b["Gw"]).abs(), b["mag_gw"])[torch.from_numpy(fam == 3), 0]
        assert float(gw.min()) > GW_BAR and float(gw[1:].min()) > GUARD * GW_BAR, gw


@pytest.mark.parametrize("Nc,Nf", [(3, 1021), (128, 384), (256, 768), (1000, 24)])
def test_emulated_wide_pdf_within_bars(Nc, Nf):
    zc, w, us = pdf_families(Nc, Nf, 1)
    for u in us:
        assert_pdf(check_pdf(emu_pdf_wide(zc, w, u), zc, w, u))


# =====================================================================================================================
# GPU: the wide kernels standalone (test_ray_stages.py's checks at N > 256)
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("N", LONG_N)
def test_wide_composite_kernels_vs_fp64(N):
    """pob_composite / pob_composite_bwd at W = 4 (S = 3..8 per thread, and both ends of S = 3 at 257 and 384) per
    element against fp64: both backgrounds, every ray family, R = 1 and R not a multiple of the block"""
    RS.test_composite_kernels_vs_fp64(N)


@pytest.mark.gpu
@pytest.mark.parametrize("Nc,Nf", LONG_PDF)
def test_wide_sample_pdf_kernel_vs_fp64(Nc, Nf):
    """pob_sample_pdf with the 1024-key sort: the u table, per-ray u and k/64 ties; sorted, coarse depths bit for
    bit, the fp64 bracket and bars"""
    RS.test_sample_pdf_kernel_vs_fp64(Nc, Nf)


@pytest.mark.gpu
@pytest.mark.parametrize("lindisp", [False, True])
def test_sample_coarse_bit_exact_1024(lindisp):
    RS.test_sample_coarse_bit_exact(1024, lindisp)


@pytest.mark.gpu
def test_c_abi_refuses_past_1024():
    from plenoctree_b200._lib import lib, ptr
    x = torch.zeros(4 * 1025 * 4, device="cuda")
    assert lib.pob_composite(ptr(x), ptr(x), ptr(x), 1, 1025, 1, ptr(x), None, None, None, None) != 0
    assert lib.pob_composite_bwd(ptr(x), ptr(x), ptr(x), ptr(x), ptr(x), 1, 1025, 1, 1.0, ptr(x), None, None) != 0
    assert lib.pob_sample_pdf(ptr(x), ptr(x), ptr(x), 1, 1, 512, 513, ptr(x), None) != 0
    assert lib.pob_sample_pdf(ptr(x), ptr(x), ptr(x), 1, 1, 512, 512, ptr(x), None) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("nc,nf", [(1024, 0), (3, 1021), (128, 384)])
def test_nerf_model_accepts_the_bound(nc, nf):
    """NerfModel builds and renders at the ends of the bound"""
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf.rays import random_rays_np
    m = NerfModel(num_coarse_samples=nc, num_fine_samples=nf, max_rays=16)
    m.init_params(3)
    o, d, v, _ = random_rays_np(16, 5)
    out = m(Rays(o, d, v))
    torch.cuda.synchronize()
    assert all(torch.isfinite(t).all() for lvl in out for t in lvl)


# =====================================================================================================================
# GPU: inside the training and render calls at (128, 384)
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("precision", [1, 3])
def test_ray_stages_in_training_call_long(precision):
    """test_ray_stages.py's ray-stage checks inside pob_loss_and_grad at (128, 384), fp16 and fp16x3"""
    case = RayCase(3, 40, 128, 384, 200, precision=precision)
    res = RS._in_call(case)
    RS._record(f"long_{case.name}", res)
    RS._assert_in_call(res)


@pytest.mark.gpu
def test_mlp_stages_in_training_call_long():
    """test_train_stages.py's stage checks of the saving forward, data and weight gradients at (128, 384)"""
    from tests.test_train_stages import Case, _stage_case
    _stage_case(Case(3, 40, 128, 384, 200))


@pytest.mark.gpu
def test_mlp_stages_in_training_call_long_x3():
    from tests.test_train_stages import Case
    from tests.test_train_x3 import _stage_case_x3
    _stage_case_x3(Case(3, 40, 128, 384, 200))


@pytest.mark.gpu
@pytest.mark.parametrize("randomized", [False, True])
def test_ray_stages_render_call_long(randomized):
    """pob_render_rays at (128, 384): the render workspace's stages against fp64, outputs equal to the workspace's"""
    from plenoctree_b200 import layouts as L
    from plenoctree_b200.nerf.models import Rays
    case = RayCase(3, 64, 128, 384, 0, dir_scale=True)
    model = case.model()
    n = 53
    (o, d, v, px), t_rand, u, _, _ = case.inputs(n)
    model.workspace(False).fill_(0xFF)
    out = model(Rays(o, d, v), randomized=randomized, t_rand=t_rand if randomized else None,
                u=u if randomized else None)
    torch.cuda.synchronize()
    ws = model.workspace(False)
    views = L.train_workspace_views(model.cfg, n, False, training=False)
    uu = u if randomized else model.u_table.cpu().numpy()[None]
    st = {}
    res = RS._check_levels(model, views, ws, (o, d, v), model.z_base.cpu().numpy(), t_rand if randomized else None,
                           uu, int(randomized), st)
    for i, lv in enumerate(views["levels"]):
        got = torch.cat([out[i][0], out[i][1][:, None], out[i][2][:, None]], 1)
        want = torch.cat([L.workspace_view(ws, lv, "comp"), L.workspace_view(ws, lv, "disp")[:, None],
                          L.workspace_view(ws, lv, "acc")[:, None]], 1)
        st[f"out_bit_mismatches_{i}"] = int((got.view(torch.int32) != want.view(torch.int32)).sum())
    res["stage"] = st
    RS._record(f"long_render_rand{int(randomized)}", res)
    RS._assert_in_call(res)


@pytest.mark.gpu
@pytest.mark.parametrize("nc,nf", [(128, 384), (256, 768)])
def test_render_matches_executed_reference_long_rays(golden_dir, nc, nf):
    """NerfModel.__call__ against ref_long_rays.npz, deterministic and with the injected draws, within
    test_render.py's bars: fp16x3 1e-4 max-abs on rgb and acc; fp16 1e-3 on the coarse level; a free-running fine
    level (its samples follow the coarse weights) 1e-3 relative RMS, 60 dB and 2e-2 max-abs"""
    from plenoctree_b200 import ops
    from plenoctree_b200.nerf.models import NerfModel, Rays
    g, sh, (fc, ff) = _golden(golden_dir)
    n = g["origins"].shape[0]
    model = NerfModel(sh_deg=sh, num_coarse_samples=nc, num_fine_samples=nf, max_rays=n)
    model.set_params(np.concatenate([fc, ff]))
    rays = Rays(g["origins"], g["directions"], g["viewdirs"])
    tag_n = f"{nc}_{nf}"
    rec = {}
    for tag in ("det", "rand"):
        kw = dict(randomized=False) if tag == "det" else dict(randomized=True, t_rand=g[f"t_rand_{tag_n}"],
                                                               u=g[f"u_{tag_n}"])
        for prec, pname in ((ops.PREC_FP16X3, "fp16x3"), (ops.PREC_FP16, "fp16")):
            got = model(rays, precision=prec, **kw)
            torch.cuda.synchronize()
            for lvl, (o, name) in enumerate(zip(got, ("coarse", "fine"))):
                key = f"call_{tag_n}_{tag}_{name}"
                rgb, disp, acc = (x.cpu().numpy() for x in o)
                diff = rgb - g[f"{key}_rgb"]
                e = dict(rgb=float(np.abs(diff).max()), acc=float(np.abs(acc - g[f"{key}_acc"]).max()),
                         rel_rms=float(np.linalg.norm(diff) / np.linalg.norm(g[f"{key}_rgb"])),
                         psnr=float(-10 * np.log10(max(float((diff.astype(np.float64) ** 2).mean()), 1e-20))))
                ok = np.abs(g[f"{key}_acc"]) > 1e-3
                e["disp_rel"] = float((np.abs(disp - g[f"{key}_disp"]) / np.abs(g[f"{key}_disp"]))[ok].max())
                rec[f"{tag}_{pname}_{name}"] = e
                if prec == ops.PREC_FP16X3:
                    assert e["rgb"] < 1e-4 and e["acc"] < 1e-4, (tag, pname, name, e)
                elif lvl == 0:
                    assert e["rgb"] < 1e-3 and e["acc"] < 1e-3, (tag, pname, name, e)
                else:
                    assert e["rel_rms"] < 1e-3 and e["psnr"] > 60 and e["rgb"] < 2e-2, (tag, pname, name, e)
    RS._record(f"long_render_vs_reference_{tag_n}", rec)


# =====================================================================================================================
# GPU: graph replay and the CLI at (128, 384)
# =====================================================================================================================
@pytest.mark.gpu
def test_graphed_train_step_matches_eager_long():
    """GraphedTrainStep reproduces eager train_step at (128, 384): parameters and Adam moments bit for bit"""
    from plenoctree_b200.nerf import train as T
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf.rays import random_rays_np
    from tests.test_train_stages import _params
    R = 256
    fc, ff = _params(3, 33)
    o, d, v, px = random_rays_np(R, 33)
    b12 = torch.from_numpy(np.concatenate([o, d, v, px], axis=1)).cuda()
    lrs = [5e-4, 4e-4, 3e-4]
    outs = []
    for graphed in (False, True):
        model = NerfModel(sh_deg=3, num_coarse_samples=128, num_fine_samples=384, max_rays=R, sparsity_npoints=1000)
        model.set_params(np.concatenate([fc, ff]))
        state = T.TrainState(model)
        if graphed:
            g = T.GraphedTrainStep(model, state, R)
            for lr in lrs:
                g.step(b12, lr)
        else:
            batch = {"rays": Rays(b12[:, 0:3], b12[:, 3:6], b12[:, 6:9]), "pixels": b12[:, 9:12]}
            for lr in lrs:
                T.train_step(model, state, batch, lr)
        torch.cuda.synchronize()
        outs.append((model.params.clone(), state.m.clone(), state.v.clone()))
    for name, a, b in zip(("params", "m", "v"), *outs):
        assert torch.equal(a, b), name
    assert not torch.equal(outs[0][0], torch.from_numpy(np.concatenate([fc, ff])).cuda())


@pytest.mark.gpu
def test_cli_train_eval_long_rays(tmp_path):
    """nerf_sh.train at --num_coarse_samples 128 --num_fine_samples 384, batch 1024, learns a synthetic Blender scene;
    nerf_sh.eval runs on its checkpoint at (128, 384) and at (256, 768)"""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf import datasets as D, flags as F
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf.utils import generate_rays, pose_spherical, render_image
    from plenoctree_b200.nerf_sh import eval as EV, train as TR
    sh_deg, W = 3, 48
    ft = np.concatenate([O.init_flat_params(sh_deg, 7001, bias_scale=0.05), O.init_flat_params(sh_deg, 7002, bias_scale=0.05)])
    P = O.param_count(sh_deg)
    for m in range(2):
        off = m * P + P - 48 - 1 - 256 * 48 - 256
        ft[off:off + 256] *= 30.0
    teacher = NerfModel(sh_deg=sh_deg, num_coarse_samples=128, num_fine_samples=384, max_rays=4096)
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
    common = ("dataset: blender\nfactor: 0\nuse_viewdirs: false\nwhite_bkgd: true\nbatch_size: 1024\nsh_deg: 3\n"
              "randomized: true\nmax_steps: 200\n")
    (tmp_path / "cfg.yaml").write_text(common + "num_coarse_samples: 128\nnum_fine_samples: 384\n")
    (tmp_path / "cfg_eval.yaml").write_text(common + "num_coarse_samples: 256\nnum_fine_samples: 768\n")
    F.define_flags()
    FLAGS = F.FLAGS
    if not FLAGS.is_parsed():
        FLAGS.mark_as_parsed()
    new = dict(train_dir=train_dir, data_dir=data_dir, config=str(tmp_path / "cfg"), save_every=200, print_every=100,
               render_every=0, sparsity_npoints=1000, lr_init=2e-3, lr_final=2e-4, chunk=4096, noise_std=None,
               image_batching=True)
    keep = list(new) + ["dataset", "factor", "use_viewdirs", "white_bkgd", "batch_size", "sh_deg", "randomized",
                        "max_steps", "num_coarse_samples", "num_fine_samples"]
    old = {k: getattr(FLAGS, k) for k in keep}
    try:
        for k, v in new.items():
            setattr(FLAGS, k, v)
        fresh = NerfModel(sh_deg=sh_deg, num_coarse_samples=128, num_fine_samples=384, max_rays=4096)
        fresh.init_params(20200823)
        rays = generate_rays(W, W, focal, np.stack(poses["test"]))
        gt = torch.from_numpy(images["test"][0]).cuda()
        p_init = -10 * np.log10(float(((render_image(fresh, Rays(rays.origins[0], rays.directions[0],
                                                                  rays.viewdirs[0]))[0] - gt) ** 2).mean()))
        model, state = TR.main(None)
        assert (model.num_coarse_samples, model.num_fine_samples) == (128, 384) and state.step == 200
        psnr, _ = EV.main(None)
        FLAGS.config = str(tmp_path / "cfg_eval")
        psnr_long, _ = EV.main(None)
    finally:
        for k, v in old.items():
            setattr(FLAGS, k, v)
    RS._record("long_cli", dict(psnr_init=p_init, psnr_128_384=float(psnr), psnr_eval_256_768=float(psnr_long)))
    assert np.isfinite(psnr_long) and psnr > p_init + 5.0, (p_init, psnr, psnr_long)

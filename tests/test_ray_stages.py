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
import functools

import numpy as np
import pytest
import torch

from tests.support.mlp_stages import CASES
from tests.support.ray_stages import (ACC_BAR, GUARD, GW_BAR, PDF_Z_BAR, RayCase, U24, _assert_in_call, _check_levels,
                                      _in_call, _norm, _t, assert_composite, assert_pdf, check_composite,
                                      check_composite_bwd, check_pdf, composite_bwd_ref, composite_kernels_vs_fp64,
                                      composite_ref, emu_delta, pdf_families, pdf_ref, ray_families,
                                      sample_coarse_bit_exact, sample_pdf_kernel_vs_fp64)
from tests.support.records import record


_record = functools.partial(record, "parity_ray_stages.json")


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


_STANDALONE_N = [1, 2, 31, 32, 33, 64, 65, 96, 97, 128, 129, 160, 161, 192, 193, 224, 225, 255, 256]


@pytest.mark.gpu
@pytest.mark.parametrize("N", _STANDALONE_N)
def test_composite_kernels_vs_fp64(N):
    composite_kernels_vs_fp64(N)


_PDF_SIZES = [(3, 1), (3, 253), (4, 4), (33, 31), (34, 94), (64, 128), (64, 192), (65, 64), (66, 64), (128, 128),
              (200, 56), (255, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("Nc,Nf", _PDF_SIZES)
def test_sample_pdf_kernel_vs_fp64(Nc, Nf):
    sample_pdf_kernel_vs_fp64(Nc, Nf)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 2, 33, 256])
@pytest.mark.parametrize("lindisp", [False, True])
def test_sample_coarse_bit_exact(N, lindisp):
    sample_coarse_bit_exact(N, lindisp)


# =====================================================================================================================
# GPU: inside the training and render calls
# =====================================================================================================================


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

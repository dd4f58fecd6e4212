"""GPU parity of the per-ray stages and of NerfModel.__call__ against the CPU oracle
(BASELINE config 1: 1024 rays x 64 samples, SH16, plus the full 64+128 hierarchical path)."""
import functools

import numpy as np
import pytest
import torch

from tests.support.mlp_stages import _rays
from tests.support.records import record

pytestmark = pytest.mark.gpu


_record = functools.partial(record, "parity_render.json")


def _lib():
    from plenoctree_b200._lib import check, lib, ptr
    return check, lib, ptr


@pytest.mark.parametrize("N", [64, 192, 33, 256])
def test_composite_forward_and_backward(N):
    from oracle import nerf_sh_oracle as O
    check, lib, ptr = _lib()
    rs = np.random.RandomState(N)
    R = 257
    rgb = rs.uniform(0, 1, size=(R, N, 3)).astype(np.float32)
    sigma = (rs.uniform(-1, 3, size=(R, N, 1)).clip(0) * rs.choice([0.2, 5.0, 50.0], size=(R, 1, 1))).astype(np.float32)
    sigma[:7] = 0.0
    z = np.sort(rs.uniform(2, 6, size=(R, N)).astype(np.float32), axis=-1)
    dirs = rs.normal(size=(R, 3)).astype(np.float32)
    px = rs.uniform(0, 1, size=(R, 3)).astype(np.float32)
    for white in (1, 0):
        rgbs = torch.from_numpy(np.concatenate([rgb, sigma], -1)).cuda().contiguous()
        zt, dt = torch.from_numpy(z).cuda(), torch.from_numpy(dirs).cuda()
        out_rgb = torch.empty((R, 3), device="cuda")
        out_disp, out_acc = torch.empty(R, device="cuda"), torch.empty(R, device="cuda")
        out_w = torch.empty((R, N), device="cuda")
        check(lib.pob_composite(ptr(rgbs), ptr(zt), ptr(dt), R, N, white, ptr(out_rgb), ptr(out_disp), ptr(out_acc),
                                ptr(out_w), None))
        rgb_t = torch.from_numpy(rgb).requires_grad_(True)
        sig_t = torch.from_numpy(sigma).requires_grad_(True)
        c_o, d_o, a_o, w_o = O.volumetric_rendering(rgb_t, sig_t, torch.from_numpy(z), torch.from_numpy(dirs), bool(white))
        torch.cuda.synchronize()
        np.testing.assert_allclose(out_rgb.cpu().numpy(), c_o.detach().numpy(), rtol=1e-4, atol=2e-6)
        np.testing.assert_allclose(out_acc.cpu().numpy(), a_o.detach().numpy(), rtol=1e-4, atol=2e-6)
        np.testing.assert_allclose(out_w.cpu().numpy(), w_o.detach().numpy(), rtol=1e-4, atol=2e-6)
        np.testing.assert_allclose(out_disp.cpu().numpy(), d_o.detach().numpy(), rtol=2e-4)
        # backward: d/d(pre-activation) of gscale/2 * sum (C - px)^2, pre-activation == logit / raw sigma
        gscale = 0.37
        loss = 0.5 * gscale * ((c_o - torch.from_numpy(px)) ** 2).sum()
        g_rgb, g_sig = torch.autograd.grad(loss, [rgb_t, sig_t])
        g_pre = (g_rgb * rgb_t * (1 - rgb_t)).detach().numpy()
        g_sraw = (g_sig * (sig_t > 0)).detach().numpy()
        G = torch.empty((R, N, 4), device="cuda")
        sq = torch.zeros(1, device="cuda")
        px_t = torch.from_numpy(px).cuda()
        check(lib.pob_composite_bwd(ptr(rgbs), ptr(zt), ptr(dt), ptr(out_rgb), ptr(px_t), R, N,
                                    white, gscale, ptr(G), ptr(sq), None))
        torch.cuda.synchronize()
        Gn = G.cpu().numpy()
        scale = max(np.abs(g_pre).max(), 1e-12)
        assert np.abs(Gn[..., :3] - g_pre).max() / scale < 2e-4
        scale = max(np.abs(g_sraw).max(), 1e-12)
        assert np.abs(Gn[..., 3:] - g_sraw).max() / scale < 2e-4
        want_sq = float(((c_o.detach() - torch.from_numpy(px)) ** 2).sum())
        assert abs(float(sq) - want_sq) / want_sq < 1e-4


def test_sample_coarse_and_pdf():
    from oracle import nerf_sh_oracle as O
    check, lib, ptr = _lib()
    rs = np.random.RandomState(5)
    R, Nc, Nf = 301, 64, 128
    o, d, _ = _rays(R, 1)
    t_rand = rs.uniform(0, 1, size=(R, Nc)).astype(np.float32)
    zb = (2.0 * (1.0 - torch.linspace(0, 1, Nc)) + 6.0 * torch.linspace(0, 1, Nc)).cuda()
    for tr in (None, t_rand):
        z_o, _ = O.sample_along_rays(torch.from_numpy(o), torch.from_numpy(d), Nc, 2.0, 6.0,
                                     None if tr is None else torch.from_numpy(tr))
        z_g = torch.empty((R, Nc), device="cuda")
        tr_t = None if tr is None else torch.from_numpy(tr).cuda()   # keep alive across the async launch
        check(lib.pob_sample_coarse(ptr(zb), ptr(tr_t), R, Nc, ptr(z_g), None))
        torch.cuda.synchronize()
        np.testing.assert_array_equal(z_g.cpu().numpy(), z_o.numpy())   # bit exact
    # hierarchical resampling: peaky, flat, zero and single-bin weights
    w = rs.uniform(0, 1, size=(R, Nc)).astype(np.float32) ** 8
    w[:10] = 0.0
    w[10:20] = 1.0 / Nc
    w[20:30] = 0.0
    w[20:30, 17] = 0.9
    z_c = z_o.contiguous()
    mids = 0.5 * (z_c[..., 1:] + z_c[..., :-1])
    u_rand = rs.uniform(0, 1, size=(R, Nf)).astype(np.float32)
    for u in (None, u_rand):
        z_g = torch.empty((R, Nc + Nf), device="cuda")
        if u is None:
            ut = torch.linspace(0.0, 1.0 - float(np.finfo(np.float32).eps), Nf).cuda()
        else:
            ut = torch.from_numpy(u).cuda()
        zc_t, w_t = z_c.cuda(), torch.from_numpy(w).cuda()
        check(lib.pob_sample_pdf(ptr(zc_t), ptr(w_t), ptr(ut), 0 if u is None else 1, R, Nc, Nf,
                                 ptr(z_g), None))
        torch.cuda.synchronize()
        zg = z_g.cpu().numpy()
        assert np.all(zg[:, 1:] >= zg[:, :-1])
        # well-conditioned rays: direct comparison with the oracle's samples
        z_ref, _ = O.sample_pdf(mids, torch.from_numpy(w)[..., 1:-1], torch.from_numpy(o), torch.from_numpy(d), z_c, Nf,
                                None if u is None else torch.from_numpy(u))
        err = np.abs(zg - z_ref.numpy())
        np.testing.assert_allclose(zg[10:20], z_ref.numpy()[10:20], atol=2e-5)   # flat pdf rows
        assert np.median(err) < 1e-5
        # every ray, conditioning-independent: the union must contain the coarse depths bit-exactly, and
        # the new samples pushed forward through the (float64) reference CDF must reproduce u
        u_used = ut.cpu().numpy().astype(np.float64)
        zc_np, mids_np = z_c.numpy(), mids.numpy().astype(np.float64)
        for r in range(R):
            rest = list(zg[r])
            for zc in zc_np[r]:
                rest.remove(zc)
            ws = w[r, 1:-1].astype(np.float64)
            pad = max(0.0, 1e-5 - ws.sum())
            ws = ws + pad / ws.size
            cdf = np.concatenate([[0.0], np.minimum(1.0, np.cumsum(ws / ws.sum())[:-1]), [1.0]])
            # flat (zero-pdf) stretches make the inverse ambiguous; the forward map is still exact
            u_back = np.sort(np.interp(np.asarray(rest, np.float64), mids_np[r], cdf))
            u_want = np.sort(u_used if u is None else u_used[r])
            assert np.abs(u_back - u_want).max() < 2e-5, (r, np.abs(u_back - u_want).max())


@pytest.mark.parametrize("sh_deg,nf", [(3, 0), (3, 128), (4, 128)])
def test_nerf_forward_vs_oracle(sh_deg, nf):
    """config 1 (1024 x 64, single level) and the reference-faithful 64 + 128 hierarchy."""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    from plenoctree_b200.nerf.models import NerfModel, Rays
    R = 1024
    fc = O.init_flat_params(sh_deg, 20200823, bias_scale=0.05)
    ff = O.init_flat_params(sh_deg, 20200824, bias_scale=0.05)
    # a density scale that produces partially opaque rays (random-init sigma is ~0.1)
    for f in (fc, ff):
        off = O.param_count(sh_deg) - (3 * (sh_deg + 1) ** 2) - 1 - 256 * 3 * (sh_deg + 1) ** 2 - 256
        f[off:off + 256] *= 30.0
    o, d, v = _rays(R, 3)
    rs = np.random.RandomState(9)
    t_rand = rs.uniform(0, 1, size=(R, 64)).astype(np.float32)
    u = rs.uniform(0, 1, size=(R, nf)).astype(np.float32) if nf else None
    model = NerfModel(sh_deg=sh_deg, num_coarse_samples=64, num_fine_samples=nf, near=2.0, far=6.0, max_rays=R)
    model.set_params(np.concatenate([fc, ff]) if nf else fc)
    rays = Rays(o, d, v)
    rays_t = tuple(torch.from_numpy(a) for a in (o, d, v))
    for randomized in (False, True):
        tr = torch.from_numpy(t_rand) if randomized else None
        ur = torch.from_numpy(u) if (randomized and nf) else None
        with torch.no_grad():
            ref, aux = O.nerf_forward(O.unflatten(fc, sh_deg), O.unflatten(ff, sh_deg), sh_deg, rays_t, 64, nf, 2.0,
                                      6.0, True, tr, ur, return_aux=True)
        for prec, pname in ((ops.PREC_FP16X3, "fp16x3"), (ops.PREC_FP16, "fp16")):
            for pinned in ((False, True) if nf else (False,)):
                got = model(rays, randomized=randomized, t_rand=t_rand if randomized else None,
                            u=u if (randomized and nf) else None, precision=prec,
                            z_fine=aux["z_fine"].numpy() if pinned else None)
                torch.cuda.synchronize()
                for lvl, (g, r) in enumerate(zip(got, ref)):
                    diff = g[0].cpu() - r[0]
                    e_rgb = float(diff.abs().max())
                    e_acc = float((g[2].cpu() - r[2]).abs().max())
                    rel_rms = float(diff.norm() / r[0].norm())
                    psnr = -10 * np.log10(max(float((diff ** 2).mean()), 1e-20))
                    _record(f"sh{sh_deg}_nf{nf}_rand{int(randomized)}_{pname}_pinned{int(pinned)}_lvl{lvl}",
                            dict(rgb_max_abs=e_rgb, acc_max_abs=e_acc, rel_rms=rel_rms, psnr_vs_oracle=psnr,
                                 acc_mean=float(r[2].mean())))
                    # Tolerances (rendered RGB lives in [0,1]: absolute == relative to full scale)
                    #  fp16x3               : 1e-4 max-abs, always.
                    #  fp16, same sample positions (coarse level, or fine level with z pinned): 1e-3 max-abs.
                    #  fp16, free-running fine level: the coarse weights differ by ~1e-3, which moves the
                    #    importance samples; on a random-init field with 2^9 posenc octaves that perturbs
                    #    single rays by up to ~1e-2.  Bar: 1e-3 relative RMS, 60 dB PSNR vs oracle, 2e-2 max.
                    if prec == ops.PREC_FP16X3:
                        assert e_rgb < 1e-4 and e_acc < 1e-4, (lvl, pname, randomized, pinned, e_rgb, e_acc)
                    elif lvl == 0 or pinned:
                        assert e_rgb < 1e-3 and e_acc < 1e-3, (lvl, pname, randomized, pinned, e_rgb, e_acc)
                    else:
                        assert rel_rms < 1e-3 and psnr > 60 and e_rgb < 2e-2, (lvl, randomized, rel_rms, psnr, e_rgb)


def test_full_frame_psnr_parity():
    """north-star bar: PSNR of a rendered full frame within 0.05 dB of the reference path (oracle), measured
    against the same target image (a teacher field rendered by the oracle).  64x64 frame, SH16, 64+128."""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf import utils as U
    sh_deg, H, W = 3, 64, 64
    focal = 0.5 * W / np.tan(0.5 * 0.6911112070083618)
    pose = O.pose_spherical(40.0, -35.0, 4.0)[None]
    rays = U.generate_rays(W, H, focal, pose)
    o, d, v = (r[0].reshape(-1, 3) for r in rays)

    def field(seed):
        fc = O.init_flat_params(sh_deg, seed, bias_scale=0.05)
        ff = O.init_flat_params(sh_deg, seed + 1, bias_scale=0.05)
        off = O.param_count(sh_deg) - 48 - 1 - 256 * 48 - 256
        for f in (fc, ff):
            f[off:off + 256] *= 30.0
        return fc, ff

    def oracle_render(fc, ff):
        outs = []
        with torch.no_grad():
            for i in range(0, H * W, 1024):
                sl = tuple(torch.from_numpy(a[i:i + 1024]) for a in (o, d, v))
                outs.append(O.nerf_forward(O.unflatten(fc, sh_deg), O.unflatten(ff, sh_deg), sh_deg, sl, 64, 128, 2.0,
                                           6.0, True)[-1][0])
        return torch.cat(outs).numpy()

    target = oracle_render(*field(500))
    fc, ff = field(600)
    ref = oracle_render(fc, ff)
    model = NerfModel(sh_deg=sh_deg, max_rays=2048)
    model.set_params(np.concatenate([fc, ff]))
    img = Rays(*[r[0] for r in rays])
    psnr_ref = U.compute_psnr(float(((ref - target) ** 2).mean()))
    for prec, pname in ((ops.PREC_FP16, "fp16"), (ops.PREC_FP16X3, "fp16x3")):
        rgb, disp, acc = U.render_image(model, img, chunk=2048, precision=prec)
        torch.cuda.synchronize()
        got = rgb.reshape(-1, 3).cpu().numpy()
        psnr_gpu = U.compute_psnr(float(((got - target) ** 2).mean()))
        psnr_vs_ref = U.compute_psnr(float(((got - ref) ** 2).mean()))
        _record(f"full_frame_{pname}", dict(psnr_gpu=float(psnr_gpu), psnr_ref=float(psnr_ref),
                                             psnr_gpu_vs_ref=float(psnr_vs_ref)))
        assert abs(psnr_gpu - psnr_ref) < 0.05, (pname, psnr_gpu, psnr_ref)
        assert psnr_vs_ref > 55.0


def test_sigma_noise_forward_vs_oracle():
    """SURVEY §8 row a4: add_gaussian_noise on raw sigma (model_utils.py:317-332) at both levels, explicit draws."""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    from plenoctree_b200.nerf.models import NerfModel, Rays
    sh_deg, R, nf = 3, 256, 128
    fc = O.init_flat_params(sh_deg, 31, bias_scale=0.05)
    ff = O.init_flat_params(sh_deg, 32, bias_scale=0.05)
    for f in (fc, ff):
        off = O.param_count(sh_deg) - 48 - 1 - 256 * 48 - 256
        f[off:off + 256] *= 30.0
    o, d, v = _rays(R, 5)
    rs = np.random.RandomState(10)
    t_rand = rs.uniform(0, 1, size=(R, 64)).astype(np.float32)
    u = rs.uniform(0, 1, size=(R, nf)).astype(np.float32)
    noise = (rs.normal(size=(R, 64)).astype(np.float32) * 2.0, rs.normal(size=(R, 64 + nf)).astype(np.float32) * 2.0)
    rays_t = tuple(torch.from_numpy(a) for a in (o, d, v))
    with torch.no_grad():
        ref, aux = O.nerf_forward(O.unflatten(fc, sh_deg), O.unflatten(ff, sh_deg), sh_deg, rays_t, 64, nf, 2.0, 6.0,
                                  True, torch.from_numpy(t_rand), torch.from_numpy(u), return_aux=True,
                                  sigma_noise=tuple(torch.from_numpy(a) for a in noise))
        plain = O.nerf_forward(O.unflatten(fc, sh_deg), O.unflatten(ff, sh_deg), sh_deg, rays_t, 64, nf, 2.0, 6.0,
                               True, torch.from_numpy(t_rand), torch.from_numpy(u))
    assert float((ref[1][0] - plain[1][0]).abs().max()) > 1e-2   # the noise matters at this scale
    model = NerfModel(sh_deg=sh_deg, num_coarse_samples=64, num_fine_samples=nf, max_rays=R)
    model.set_params(np.concatenate([fc, ff]))
    got = model(Rays(o, d, v), randomized=True, t_rand=t_rand, u=u, precision=ops.PREC_FP16X3,
                z_fine=aux["z_fine"].numpy(), sigma_noise=noise)
    torch.cuda.synchronize()
    for lvl in range(2):
        e = float((got[lvl][0].cpu() - ref[lvl][0]).abs().max())
        _record(f"sigma_noise_lvl{lvl}", dict(rgb_max_abs=e))
        assert e < 1e-4, (lvl, e)
    # noise_std flag: drawn on the device when randomized, identity otherwise
    model.noise_std = 1.0
    a = model(Rays(o, d, v), randomized=False)[1][0].cpu()
    model.noise_std = None
    b = model(Rays(o, d, v), randomized=False)[1][0].cpu()
    assert float((a - b).abs().max()) == 0.0
    model.noise_std = 1.0
    c = model(Rays(o, d, v), randomized=True, t_rand=t_rand, u=u)[1][0].cpu()
    model.noise_std = None
    e = model(Rays(o, d, v), randomized=True, t_rand=t_rand, u=u)[1][0].cpu()
    assert float((c - e).abs().max()) > 1e-3

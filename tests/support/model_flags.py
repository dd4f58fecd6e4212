"""Models with every NeRF-SH flag (encoder, activations, SM count, L2 discard), their fp64 checks and budgets."""
import functools
import types

import numpy as np
import pytest
import torch

from oracle import net_activation_oracle as NA, posenc_oracle as PO
from plenoctree_b200 import _lib, layouts as L
from tests.support.mlp_stages import Stats
from tests.support.records import record

_record = functools.partial(record, "parity_net_activation.json")


SP_BAR = 4.0            # softplus in the heads epilogue, in units of u * softplus64(x)
SP_FLOOR = 2.0 ** -148  # absolute: expf's denormal outputs below x = -87


def softplus64(x):
    x = torch.as_tensor(x).double()
    return x.clamp_min(0) + torch.log1p(torch.exp(-x.abs()))


def _scope_args(**kw):
    base = dict(use_viewdirs=False, sg_dim=-1, dataset="blender", net_depth=8, net_width=256, skip_layer=4,
                min_deg_point=0, max_deg_point=10, net_activation="relu", rgb_activation="sigmoid",
                sigma_activation="relu", legacy_posenc_order=False, render_path=False, spherify=False)
    base.update(kw)
    return types.SimpleNamespace(**base)


def _gpu_params(pe, sh, seed):
    """two MLPs of the oracle's initialisation for encoder pe, Dense_8 scaled by 30 (as test_train_stages._params)"""
    out = []
    w_off = L.flat_offsets(L.K_of(sh), PO.width(pe))[0]
    for s in (seed, seed + 1):
        f = PO.init_flat_params(sh, s, bias_scale=0.05, pe=pe)
        f[w_off[8]:w_off[8] + 256] *= 30.0
        out.append(f)
    return out


def _ref_features(x, pe):
    """fp64 sines of the kernel's fp32 arguments: [M, W - 3] in the encoder's column order"""
    cols = []
    half_pi = torch.tensor(np.float32(np.pi / 2), device=x.device)
    for kind, j, c in PO.feature_index(pe)[3:]:
        xb = x[:, c] * float(2 ** j)                                 # exact fp32 product
        cols.append(torch.sin((xb if kind == "sin" else xb + half_pi).double()))
    return torch.stack(cols, 1) if cols else torch.zeros(x.shape[0], 0, dtype=torch.float64, device=x.device)


U24 = 2.0 ** -24


ACT_BOUND = 4.0            # f's fp32 error, in units of 2^-24 * |f(z)| (kernels.h: net_act_f32)
X3 = 3


# fp16x3 posenc tile: sines (hi + lo) against fp64 of the kernel's fp32 arguments, beyond lo's representation error, in
# units of 2^-24; dO's rgb columns (the fp32 product G.rgb * Y_k with the fp32 SH basis, stored in fp16 or hi + lo)
# beyond the rounding of the stored value, in units of 2^-24 * |G.rgb|.  Measured on an H100 80 GB HBM3 at a 700 W
# power limit over test_net_activation.py's cases and test_flag_matrix.py's rows, the largest value in brackets.
SIN_X3_ALLOW = 3.0          # [1.41]
DO_ALLOW = 6.0              # [2.84 fp16x3, 1.74 fp16]


def _grad_of_output(act, h):
    """fp64 f'(z) from h = f(z) (kernels.h: net_act_grad_of_output)"""
    if act == "elu":
        return torch.where(h > 0, torch.ones_like(h), h + 1.0)
    if act == "softplus":
        return -torch.expm1(-h)
    if act == "tanh":
        return (1.0 - h) * (1.0 + h)
    return (h > 0).double()


def _act64(act, z):
    return NA.activation(act)(z)


def _make_model(case, act, precision=1, pe=PO.DEFAULT, sigma_act="relu"):
    from plenoctree_b200.nerf.models import NerfModel
    m = NerfModel(sh_deg=case.sh, num_coarse_samples=case.nc, num_fine_samples=case.nf, max_rays=case.R,
                  sparsity_npoints=case.nsp, net_activation=act, sigma_activation=sigma_act,
                  white_bkgd=getattr(case, "white", True), min_deg_point=pe[0], max_deg_point=pe[1],
                  legacy_posenc_order=pe[2])
    fc, ff = _gpu_params(pe, case.sh, case.seed)
    for f in (fc, ff):
        _centre_sigma(f, case.sh, act, pe)
    m.set_params(np.concatenate([fc, ff]) if case.nf else fc)
    return m


def _centre_sigma(flat, sh, act, pe=PO.DEFAULT):
    """centre every trunk layer's pre-activations and raw sigma over the scene box (each bias minus the mean, raw
    sigma's minus the median), the state a trained network sits in.  With the relu trunk's initial parameters a
    softplus trunk's pre-activations drift up layer by layer (softplus >= 0 adds a common positive part) until raw
    sigma is negative everywhere: an empty scene, a zero gradient."""
    _, b_off, _ = L.flat_offsets(L.K_of(sh), PO.width(pe))
    box = torch.from_numpy(np.random.RandomState(5).uniform(-1.5, 1.5, (4000, 3)).astype(np.float32))
    f = NA.activation(act)
    with torch.no_grad():
        params = PO.unflatten(flat, sh, pe)
        enc = PO.encode(box, pe)
        h = enc
        for i in range(8):
            z = h @ params[i][0] + params[i][1]
            shift = z.mean(0).numpy().astype(np.float32)
            flat[b_off[i]:b_off[i] + 256] -= shift
            h = f(z - torch.from_numpy(shift))
            if i == 4:
                h = torch.cat([h, enc], -1)
        _, sig = NA.mlp(PO.unflatten(flat, sh, pe), enc, act)
    flat[b_off[8]] -= np.float32(np.median(sig.numpy()))


def _sin_excess(e_hi, e_lo, ref, x3):
    """sine columns against fp64 of the kernel's fp32 arguments.  fp16: beyond one fp16 ulp, in units of SIN_ABS
    (test_train_stages.py); fp16x3: hi + lo beyond lo's representation error, in units of 2^-24 (|sin| <= 1)"""
    from tests.support.mlp_stages import SIN_ABS, _ulp16_log2
    from tests.support.mlp_x3 import _repr_err
    if x3:
        err = (e_hi.double() + e_lo.double() - ref).abs() - _repr_err(e_lo)
        return float((err.clamp_min(0) / U24).max())
    err = (e_hi.double() - ref.half().double()).abs()
    return float(((err - _ulp16_log2(ref)).clamp_min(0) / SIN_ABS).max())


def _sigma_want(sig, onray, sigma_act):
    """the rgbs epilogue's density from fp64 raw sigma (+ noise): the model's activation on ray rows, relu on the
    free sparsity rows; and the extra allowance of softplus (test_sigma_activation.py: SP_BAR, SP_FLOOR)"""
    if sigma_act == "softplus":
        sp = softplus64(sig)
        return (torch.where(onray, sp, sig.clamp_min(0)),
                torch.where(onray, SP_BAR * U24 * sp + SP_FLOOR, torch.zeros_like(sig)))
    return sig.clamp_min(0), torch.zeros_like(sig)


def _check_level(ws, lv, flat, grad, sh, scale, st, act, x3, pe=PO.DEFAULT, sigma_act="relu", call=None, alt=None):
    """saving forward (posenc tile, trunk, rgbs epilogue), data gradient (dO, dZ) and weight gradient of one level,
    fp16 (x3 False) or fp16x3, for any encoder pe, trunk activation act and density sigma_act.  call: the rays, free
    points, noise and ray count of the training call (the posenc tile, rgbs and dO checks need them).  alt: a flag
    replaced ({"pe", "act", "sigma_act"}): the same stages against the reference of the wrong flag, under guard_*."""
    from tests.support.mlp_stages import FWD_ALLOW as FWD16, _sh_basis, _ulp16_log2
    from tests.support.mlp_x3 import FWD_ALLOW as FWD3, _repr_err, _split_ok, _weights_hilo
    alt = alt or {}
    dev = ws.device
    K = L.K_of(sh)
    NH = L.heads_width(K)
    C3 = 3 * K
    EW = PO.width(pe)
    relu = act == "relu"
    fwd_allow = FWD3 if x3 else FWD16
    w_off, b_off, P = L.flat_offsets(K, EW)
    dims = L.layer_dims(K, EW)
    if x3:
        W, B, Wh, bh = _weights_hilo(flat, K, dev, EW)
    else:
        fl = torch.from_numpy(flat).to(dev)
        W = [fl[w_off[l]:w_off[l] + dims[l][0] * 256].view(dims[l][0], 256).half().double() for l in range(8)]
        B = [fl[b_off[l]:b_off[l] + 256].half().double() for l in range(8)]
        Wh_np, bh_np = L.heads_matrix(flat, K, EW)
        Wh, bh = (torch.from_numpy(a).to(dev).half().double() for a in (Wh_np, bh_np))
    cols9 = torch.tensor([L.heads_column(K, o) for o in range(C3)], device=dev)
    N, M, Mr, tiles = lv["N"], lv["M"], lv["M_rays"], lv["tiles"]
    view = lambda k: L.workspace_view(ws, lv, k)
    H, E, DZ, DO, MASK = (view(k) for k in ("H", "E", "DZ", "DO", "mask"))
    if x3:
        Hl, El, DZl, DOl = (view(k) for k in ("H_lo", "E_lo", "DZ_lo", "DO_lo"))
    if call is not None:
        o, d, v = (torch.from_numpy(a).to(dev) for a in call["rays"])
        z = view("z").reshape(-1)
        rgbs, G = view("rgbs"), view("G")
        sp = torch.from_numpy(call["sp"]).to(dev) if call["sp"] is not None and M > Mr else None
        noise = torch.from_numpy(call["noise"]).to(dev).reshape(-1) if call["noise"] is not None else None
    shapes = {**{f"w{l}": (dims[l][0], 256) for l in range(8)}, **{f"b{l}": (256,) for l in range(8)},
              "wh": (256, NH), "bh": (NH,)}
    acc = {k: torch.zeros(s, dtype=torch.float64, device=dev) for k, s in shapes.items()}
    mag = {k: torch.zeros(s, dtype=torch.float64, device=dev) for k, s in shapes.items()}

    def wsum(key, a, b):
        if b is None:
            acc[key] += a.sum(0)
            mag[key] += a.abs().sum(0)
        else:
            acc[key] += a.T @ b
            mag[key] += a.abs().T @ b.abs()

    def excess(l, hi, lo, ref, amag, extra):
        """error beyond the stored value's rounding and `extra`, in units of 2^-24 * amag"""
        if x3:
            got = hi.double() + lo.double()
            rnd = _repr_err(lo)
        else:
            got = hi.double()
            big = torch.maximum(ref.abs(), got.abs())
            rnd = torch.where(big < 2.0 ** -14, U24, 0.5 * _ulp16_log2(big))
        err = (got - ref).abs() - rnd - extra
        return float((err.clamp_min(0) / (U24 * amag).clamp_min(1e-300)).max())

    def bits(t):
        return t.view(torch.int16)

    CH = 128
    for t0 in range(0, tiles, CH):
        t1 = min(tiles, t0 + CH)
        r0, r1 = t0 * L.TILE_M, t1 * L.TILE_M
        s = torch.arange(r0, r1, device=dev)
        real = s < M
        h_hi = [L.decode_h(H[t0:t1], l) for l in range(8)]
        dz_hi = [L.decode_dz(DZ[t0:t1], l) for l in range(8)]
        nd = 64 * ((NH + 63) // 64)
        do_hi = L.decode_do(DO[t0:t1])[:, :nd]
        e_hi = L.decode_e(E[t0:t1])
        if x3:
            h_lo = [L.decode_h(Hl[t0:t1], l) for l in range(8)]
            dz_lo = [L.decode_dz(DZl[t0:t1], l) for l in range(8)]
            do_lo = L.decode_do(DOl[t0:t1])[:, :nd]
            e_lo = L.decode_e(El[t0:t1])
            st.add("split_violations_e", _split_ok(e_hi, e_lo))
        else:
            h_lo = [torch.zeros_like(x) for x in h_hi]
            dz_lo = [torch.zeros_like(x) for x in dz_hi]
            do_lo, e_lo = torch.zeros_like(do_hi), torch.zeros_like(e_hi)
        eW = (e_hi.double() + e_lo.double())[:, :EW]
        hd = [a.double() + b.double() for a, b in zip(h_hi, h_lo)]
        # ---- posenc tile: xyz bit-exact, sines against fp64 of the fp32 arguments, pad columns [W, 63) zero, col 63
        # the constant one (lo 0)
        st.add("posenc_pad_nonzero_bits", int(((bits(e_hi[:, EW:63]) != 0) | (bits(e_lo[:, EW:63]) != 0)).sum()))
        st.add("posenc_col63_not_one", int(((e_hi[:, 63] != 1) | (e_lo[:, 63] != 0)).sum()))
        if call is not None:
            sc = s.clamp_max(M - 1)                  # load_point clamps the row: padded rows repeat row M-1
            ray = (sc // N).clamp_max(call["n"] - 1)
            x = o[ray] + z[sc.clamp_max(Mr - 1)][:, None] * d[ray]
            if sp is not None:
                x = torch.where((sc >= Mr)[:, None], sp[(sc - Mr).clamp_min(0)], x)
            xh = x.half()
            st.add("posenc_xyz_bit_mismatches", int((bits(e_hi[:, :3]) != bits(xh)).sum()))
            if x3:
                st.add("posenc_xyz_bit_mismatches", int((bits(e_lo[:, :3]) != bits((x - xh.float()).half())).sum()))
            if EW > 3:
                st.max("posenc_sin_excess", _sin_excess(e_hi[:, 3:EW], e_lo[:, 3:EW], _ref_features(x, pe), x3))
                if "pe" in alt:
                    st.max("guard_posenc_sin", _sin_excess(e_hi[:, 3:EW], e_lo[:, 3:EW],
                                                           _ref_features(x, alt["pe"]), x3))
        # ---- forward: h_l = f(pre) within the rounding of the stored value + f's fp32 bound + the GEMM allowance
        mask = [L.decode_mask(MASK[l, r0:r1]) for l in range(8)] if relu else None
        for l in range(8):
            a = eW if l == 0 else (torch.cat([hd[4], eW], 1) if l == 5 else hd[l - 1])
            pre = a @ W[l] + B[l]
            amag = a.abs() @ W[l].abs() + B[l].abs()
            ref = _act64(act, pre)
            st.max("fwd_excess", excess(l, h_hi[l], h_lo[l], ref, amag, 0.0 if relu else ACT_BOUND * U24 * ref.abs()))
            if "act" in alt:
                alt_ref = _act64(alt["act"], pre)
                st.max(f"guard_fwd_l{l}", excess(l, h_hi[l], h_lo[l], alt_ref, amag,
                                                 0.0 if alt["act"] == "relu" else ACT_BOUND * U24 * alt_ref.abs()))
            st.add("h_nonfinite", int((~torch.isfinite(hd[l])).sum()))
            st.max("pre_min", float(pre[real].min()))
            st.max("pre_max_neg", -float(pre[real].max()))
            if relu and x3:
                pos = hd[l] > 0
                st.add("mask_clear_but_positive", int((pos & ~mask[l]).sum()))
                st.add("mask_set_value_zero_not_tiny", int((mask[l] & ~pos & (pre > 2.0 ** -20)).sum()))
            elif relu:
                st.add("mask_mismatches", int((mask[l] != (h_hi[l] != 0)).sum()))
        # ---- rgbs epilogue: density activation (+ noise) on ray rows, relu on sparsity rows, sigmoid of the SH sum
        if call is not None:
            heads = hd[7] @ Wh + bh
            hmag = hd[7].abs() @ Wh.abs() + bh.abs()
            rr = s[real]
            onray = rr < Mr
            got = rgbs[r0:r0 + rr.numel()].double()
            sig = heads[real, 0]
            sig_tol = fwd_allow * U24 * hmag[real, 0]
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
                tol = 0.25 * ((Y.abs()[:, :, None] * (fwd_allow * U24 * hm + 4 * U24 * hr.abs())).sum(1)) + 2 ** -21
                st.max("rgbs_rgb_excess", ((got[onray, :3] - torch.sigmoid(prer)).abs() / tol).max())
            # ---- dO: G.w in column 0, G.rgb x SH basis in the heads columns, zero on free / padded rows and pads
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
            got_do = do_hi[:, 1:1 + C3].double() + do_lo[:, 1:1 + C3].double()
            # beyond the rounding of the stored value, in units of 2^-24 * |G.rgb|: the fp32 SH basis cancels (e.g.
            # 2zz - xx - yy), so its error is absolute, on the scale of |G.rgb|, not relative to G.rgb * Y_k
            if x3:
                rnd = _repr_err(do_lo[:, 1:1 + C3])
            else:
                big = torch.maximum(ref_do.abs(), got_do.abs())
                rnd = torch.where(big < 2.0 ** -14, U24, 0.5 * _ulp16_log2(big))
            gmag = g[:, None, :3].double().abs().expand(-1, K, 3).reshape(-1, C3)
            err = (got_do - ref_do).abs() - rnd
            st.max("dO_rgb_excess", (err.clamp_min(0) / (U24 * gmag).clamp_min(1e-300)).max())
            nzr = (do_hi != 0) | (do_lo != 0)
            st.add("dO_free_or_padded_rgb_nonzero", int(nzr[~ray_rows, 1:1 + C3].sum()))
            st.add("dO_padded_sigma_nonzero", int(nzr[~real, 0].sum()))
            st.add("dO_pad_columns_nonzero", int(nzr[:, 1 + C3:nd].sum()))
        # ---- data gradient: dZ_l = dH_l * f'(h_l) with f' from the kernel's own saved h_l (relu: its mask words)
        dod = (do_hi.double() + do_lo.double())[:, :NH]
        dzd = [a.double() + b.double() for a, b in zip(dz_hi, dz_lo)]
        for l in range(7, -1, -1):
            a, Wt = (dod, Wh.T) if l == 7 else (dzd[l + 1], W[l + 1][:256].T)
            dh = a @ Wt
            gp = mask[l].double() if relu else _grad_of_output(act, hd[l])
            ref = dh * gp
            amag = (a.abs() @ Wt.abs()) * gp.abs()
            if x3:
                sub_row = ((a != 0) & (a.abs() < 2.0 ** -14)).any(1, keepdim=True)
                normal = ~sub_row.expand_as(ref)
                ref_n = torch.where(normal, ref, dzd[l])
            else:
                normal, ref_n = None, ref
            st.max("bwd_excess", excess(l, dz_hi[l], dz_lo[l], ref_n, amag, 0.0))
            if "act" in alt:
                gpa = _grad_of_output(alt["act"], hd[l])
                mut = dh * gpa
                st.max(f"guard_bwd_l{l}", excess(l, dz_hi[l], dz_lo[l], mut, (a.abs() @ Wt.abs()) * gpa.abs(), 0.0))
            if not relu:
                # mutation: the relu mask of h_l in place of f'(h_l)
                mut = dh * (hd[l] > 0).double()
                st.min("bwd_excess_relu_mask_mutation", excess(l, dz_hi[l], dz_lo[l], mut, amag, 0.0))
            st.add("dz_nonfinite", int((~torch.isfinite(dzd[l])).sum()))
            st.add("dz_padded_nonzero", int(((dz_hi[l][~real] != 0) | (dz_lo[l][~real] != 0)).sum()))
            st.max("dz_headroom", float(dz_hi[l].abs().max()) / 65504.0)
        # ---- weight-gradient sums
        for l in range(1, 8):
            wsum(f"w{l}", hd[l - 1] if l != 5 else torch.cat([hd[4], eW], 1), dzd[l])
        wsum("w0", eW, dzd[0])
        for l in range(8):
            wsum(f"b{l}", dzd[l], None)
        wsum("wh", hd[7], dod)
        wsum("bh", dod, None)

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
    gg = grad.double()
    for l in range(10):
        for nm, a, n in (("w", w_off[l], dims[l][0] * dims[l][1]), ("b", b_off[l], dims[l][1])):
            sl = slice(a, a + n)
            err = (gg[sl] - ref[sl]).abs()
            e = float((err / rmag[sl].clamp_min(1e-300)).max())
            if e > st.d.get(f"wgrad_{nm}_max_err_over_abs_sum", float("-inf")):
                st.d[f"wgrad_{nm}_worst_tensor"] = f"Dense_{l}.{nm}"
            st.max(f"wgrad_{nm}_max_err_over_abs_sum", e)
            st.max(f"wgrad_{nm}_rel_l2", float(err.norm() / max(float(ref[sl].norm()), 1e-300)))


def _check_call(model, state, ctx, precision, act, pe=PO.DEFAULT, sigma_act="relu", alt=None):
    """_check_level on every level of the training call in the model's workspace -> {MLP_i: stages}"""
    from plenoctree_b200.nerf.train import default_loss_scale
    ws = model.workspace(True, precision)
    views = L.train_workspace_views(model.cfg, ctx["n"], ctx["sp"] is not None, precision=precision)
    assert views["total"] == ws.numel()
    scale = default_loss_scale(ctx["n"], precision)
    params = model.params.cpu().numpy()
    P = model.P
    noise = ctx.get("noise")
    res = {}
    for i, lv in enumerate(views["levels"]):
        s = Stats()
        last = i == len(views["levels"]) - 1
        call = dict(rays=ctx["rays"], n=ctx["n"], sp=ctx["sp"] if last else None,
                    noise=noise[i] if noise is not None else None)
        _check_level(ws, lv, params[i * P:(i + 1) * P], state.grads[i * P:(i + 1) * P], model.sh_deg, scale, s, act,
                     precision == X3, pe, sigma_act, call, alt)
        res[f"MLP_{i}"] = dict(stages=s.d, M=lv["M"], tiles=lv["tiles"])
    return res


def _assert_call(res, precision, act, wg_w_bar=None):
    from tests.support import mlp_stages as TS
    from tests.support import mlp_x3 as TX
    x3 = precision == X3
    fwd_allow, bwd_allow = (TX.FWD_ALLOW, TX.BWD_ALLOW) if x3 else (TS.FWD_ALLOW, TS.BWD_ALLOW)
    wg_w, wg_b = (TX.WG_EPS_W, TX.WG_EPS_B) if x3 else (TS.WG_EPS_W, TS.WG_EPS_B)
    wg_w = wg_w_bar or wg_w
    zero = ["h_nonfinite", "dz_nonfinite", "dz_padded_nonzero", "posenc_xyz_bit_mismatches", "posenc_pad_nonzero_bits",
            "posenc_col63_not_one", "dO_sigma_bit_mismatches", "dO_free_or_padded_rgb_nonzero",
            "dO_padded_sigma_nonzero", "dO_pad_columns_nonzero"]
    if x3:
        zero.append("split_violations_e")
    if act == "relu":
        zero += ["mask_clear_but_positive", "mask_set_value_zero_not_tiny"] if x3 else ["mask_mismatches"]
    for mlp, r in res.items():
        s = r["stages"]
        for k in zero:
            assert s[k] == 0, (act, mlp, k, s[k])
        assert s.get("posenc_sin_excess", 0.0) <= (SIN_X3_ALLOW if x3 else 1.0), (act, mlp, s)
        assert s["fwd_excess"] <= fwd_allow, (act, mlp, s)
        assert s["rgbs_sigma_excess"] <= 1.0 and s.get("rgbs_rgb_excess", 0.0) <= 1.0, (act, mlp, s)
        assert s["dO_rgb_excess"] <= DO_ALLOW, (act, mlp, s)
        assert s["bwd_excess"] <= bwd_allow, (act, mlp, s)
        assert s["dz_headroom"] < 1.0, (mlp, s)
        assert s["wgrad_w_max_err_over_abs_sum"] <= wg_w, (act, mlp, s)
        assert s["wgrad_b_max_err_over_abs_sum"] <= wg_b, (act, mlp, s)
        if not x3:
            assert s["wgrad_w_rel_l2"] <= TS.WG_EPS2_W and s["wgrad_b_rel_l2"] <= TS.WG_EPS2_B, (act, mlp, s)


def _stage_case(case, act, precision, wg_w_bar=None):
    from tests.support import mlp_x3 as TX
    model = _make_model(case, act)
    state, ctx = TX._run(case, model, precision, fill=0xFF)
    res = _check_call(model, state, ctx, precision, act)
    _record(f"stages_{act}_{'fp16x3' if precision == X3 else 'fp16'}_{case.name}", res)
    _assert_call(res, precision, act, wg_w_bar)
    return res


def _set_flags(**kw):
    from plenoctree_b200.nerf import flags as F
    F.define_flags()
    if not F.FLAGS.is_parsed():
        F.FLAGS.mark_as_parsed()
    for k, v in kw.items():
        setattr(F.FLAGS, k, v)
    return F.FLAGS


def _device_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _set_sms(monkeypatch, n):
    """make the library split its work for n SMs ("device": POB_SM_COUNT unset) until the test ends"""
    from plenoctree_b200._lib import lib
    dev = _device_sms()
    if n == "device":
        monkeypatch.delenv("POB_SM_COUNT", raising=False)
        n = dev
    else:
        if n > dev:
            pytest.skip(f"{n} SMs: the device has {dev}")
        monkeypatch.setenv("POB_SM_COUNT", str(n))
    assert lib.pob_sm_count() == n
    return n


def _alt_pe(pe):
    """an encoder of the same width that differs from pe: the other feature order, or (one degree) shifted degrees
    where both orders coincide; None for W = 3 (no sines)"""
    mn, mx, legacy = pe
    if mn == mx:
        return None
    if mx - mn == 1:
        return (mn - 1, mx - 1, legacy) if mn > 0 else (mn + 1, mx + 1, legacy)
    return (mn, mx, not legacy)


RAYS, NC, NF, NSP = 4096, 64, 128, 10000     # the production SH16 step (bench.py)
FILL = 0x5A


def _model(sh_deg, nf, nsp, near=2.0, far=6.0, R=RAYS):
    from plenoctree_b200.nerf.models import NerfModel
    model = NerfModel(sh_deg=sh_deg, num_coarse_samples=NC, num_fine_samples=nf, near=near, far=far,
                      white_bkgd=True, max_rays=R, sparsity_npoints=nsp)
    model.init_params(20200823)
    return model


def _batch(R, seed):
    from plenoctree_b200.nerf.models import Rays
    from plenoctree_b200.nerf.utils import random_rays_np
    o, d, v, px = random_rays_np(R, seed)
    b = torch.from_numpy(np.concatenate([o, d, v, px], axis=1)).cuda()
    return {"rays": Rays(b[:, 0:3], b[:, 3:6], b[:, 6:9]), "pixels": b[:, 9:12]}, b


def _call(model, state, batch, keep, precision=_lib.PREC_FP16, **kw):
    """loss_and_grad from a workspace filled with FILL; returns (grads, stats_raw, workspace bytes)"""
    from plenoctree_b200.nerf import train as T
    ws = model.workspace(True, precision)
    ws.fill_(FILL)
    T.loss_and_grad(model, state, batch, precision=precision, keep_saved_tiles=keep, **kw)
    torch.cuda.synchronize()
    return state.grads.clone(), state.stats_raw.clone(), ws.clone()


def _saved_grad_ranges(model, R, sparsity_on):
    """[start, end) byte ranges of the DZ and DO images the call writes"""
    views = L.train_workspace_views(model.cfg, R, sparsity_on)
    out = []
    for v in views["levels"]:
        for name in ("DZ", "DO"):
            off, shape = v[name]
            out.append((off, off + int(np.prod(shape))))
    return out


def _equal_outside(w0, w1, ranges):
    start = 0
    for a, b in sorted(ranges) + [(w0.numel(), w0.numel())]:
        if not torch.equal(w0[start:a], w1[start:a]):
            return False
        start = b
    return True


CANARY = 0x7FBADBAD         # a NaN bit pattern behind every output


def _canary(shape, tail=1024):
    """(int32 buffer of the canary, float32 view of its first prod(shape) words)"""
    n = int(np.prod(shape))
    buf = torch.full((n + tail,), CANARY, dtype=torch.int32, device="cuda")
    return buf, buf[:n].view(torch.float32).view(shape)


def _points(n, seed):
    rs = np.random.RandomState(seed)
    return torch.from_numpy(rs.uniform(-1.2, 1.2, size=(n, 3)).astype(np.float32)).cuda()


def _run_points(nerf, pts):
    """pob_sh_proj_points on a 0xFF workspace and canary outputs -> (ws, a, sigma, a_buf, sigma_buf)"""
    from plenoctree_b200._lib import check, lib, posenc_ref, ptr, stream_ptr
    m = pts.shape[0]
    ws = torch.full((int(lib.pob_sh_proj_points_workspace_bytes(m)),), 0xFF, dtype=torch.uint8, device="cuda")
    ab, a = _canary((m, 128))
    sb, s = _canary((m,))
    check(lib.pob_sh_proj_points(ptr(nerf.sigma_blob), posenc_ref(nerf._pe), ptr(pts), m, ptr(nerf.head_w),
                                 ptr(nerf.head_b), ptr(ws), ptr(a), ptr(s), stream_ptr()))
    torch.cuda.synchronize()
    return ws, a, s, ab, sb

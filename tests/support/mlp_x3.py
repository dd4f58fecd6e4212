"""The fp16x3 training MLP against fp64, stage by stage: hi + lo operands, the stage checker and its own budgets."""
import functools

import torch

from plenoctree_b200 import layouts as L
from tests.support.records import record

_record = functools.partial(record, "parity_train_x3.json")


U24 = 2.0 ** -24
X3 = 3

# ---- bars, measured on an H100 80 GB HBM3 at a 400 W power limit (largest value over the cases of test_train_x3.py in
# brackets), in units of 2^-24 * sum |a*w| beyond the representation error of the stored hi + lo.  An x3 bar must stay
# at least 2^7 below fp16's operand rounding (2^-11 = 2^13 units), or the mode is not what it claims.
FWD_ALLOW = 32.0            # [16.2]
BWD_ALLOW = 32.0            # [22.1]


# The one exception: dZ entries whose contraction reads an fp16-subnormal operand (|a| < 2^-14 in the loss-scaled chain,
# hi then carries fewer than 11 bits and lo is 0).  There the tensor cores' fp32 sum is measured up to ~390 units from
# fp64 (coarse MLP of the production step); those entries are bounded separately and recorded.
BWD_SUBNORMAL_ALLOW = 512.0  # [391]
# weight gradient + reduce, per element over sum |a*b|: the fp32 accumulation over the samples is what remains
WG_EPS_W = 1e-4             # [1.9e-5]
WG_EPS_B = 2e-6             # [2.5e-7]
# End to end.  The loss statistics within LOSS_REL of the fp64 oracle.  The gradient (and a six-step Adam update)
# against two oracles on the same inputs: fp64, and the oracle evaluated in fp32 (the reference's own precision).
# The fp32 oracle is itself some 5e-4 (relative L2) from fp64 on these inputs: fp32 sample positions o + t d, amplified
# up to 2^9 by the positional encoding.  No fp32-class step can come closer to fp64 than that, so the x3 step must sit
# at that floor (within FLOOR_SLACK of the fp32 oracle's distance to fp64) and be GRAD_GAIN times closer to the fp32
# oracle than the fp16 step is.
LOSS_REL = 1e-5             # [1.5e-6]
GRAD_GAIN = 10.0            # [780x gradient, 21x six-step update]
FLOOR_SLACK = 1.1           # [1.000 gradient, 0.995 update]


def _ulp16_frexp(x):
    """fp16 ulp at |x| (fp64 tensor), 2^-24 in the subnormal range.  The exponent comes from frexp: log2 on the GPU is
    not exact at every power of two (log2(8) < 3 there), which would halve the ulp of 8, 64, ..."""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -14))
    return torch.ldexp(torch.ones_like(x), (e - 11).to(torch.int64))


def _run(case, model, precision, n=None, fill=None, z_fine=None, inputs=None):
    from plenoctree_b200.nerf import train as T
    from plenoctree_b200.nerf.models import Rays
    n = n or case.R
    (o, d, v, px), t_rand, u, sp, noise = inputs or case.inputs(n)
    state = T.TrainState(model)
    if fill is not None:
        model.workspace(True, precision).fill_(fill)
    T.loss_and_grad(model, state, {"rays": Rays(o, d, v), "pixels": px},
                    sparsity_weight=case.sparsity_weight if case.nsp else 0.0, sparsity_length=0.05,
                    randomized=True, t_rand=t_rand, u=u, sp_points=sp, sigma_noise=noise, z_fine=z_fine,
                    precision=precision)
    torch.cuda.synchronize()
    return state, dict(rays=(o, d, v), sp=sp, noise=noise, n=n, t_rand=t_rand, u=u)


def _hilo(hi, lo):
    return hi.double() + lo.double()


def _repr_err(lo):
    """bound of |v - (hi + lo)| for the fp32 value v the kernel split: half an ulp of lo (2^-25 once lo is subnormal)"""
    return 0.5 * _ulp16_frexp(lo.double())


def _excess(hi, lo, ref, mag):
    err = (_hilo(hi, lo) - ref).abs() - _repr_err(lo)
    return float((err.clamp_min(0) / (U24 * mag).clamp_min(1e-300)).max())


def _split_ok(hi, lo):
    """|lo| <= half an ulp of hi for every pair (lo = 0 where hi = 0)"""
    return int(((lo.double().abs() > 0.5 * _ulp16_frexp(hi.double()) * (hi != 0)) | ((hi == 0) & (lo != 0))).sum())


def _weights_hilo(flat, K, dev, enc_width=L.ENC_DIM):
    """fp64 hi + lo of every operand pack_weights / pack_wt_lo make: W[l] [in, 256], B[l], Wh [256, NH], bh [NH]"""
    w_off, b_off, _ = L.flat_offsets(K, enc_width)
    dims = L.layer_dims(K, enc_width)
    fl = torch.from_numpy(flat).to(dev)
    hl = lambda x: x.half().double() + (x - x.half().float()).half().double()
    W = [hl(fl[w_off[l]:w_off[l] + dims[l][0] * 256].view(dims[l][0], 256)) for l in range(8)]
    B = [hl(fl[b_off[l]:b_off[l] + 256]) for l in range(8)]
    Wh_np, bh_np = L.heads_matrix(flat, K, enc_width)
    return W, B, hl(torch.from_numpy(Wh_np).to(dev)), hl(torch.from_numpy(bh_np).to(dev))


def _check_level_x3(ws, lv, flat, grad, case, scale, st):
    dev = ws.device
    K = L.K_of(case.sh)
    NH = L.heads_width(K)
    C3 = 3 * K
    w_off, b_off, P = L.flat_offsets(K)
    dims = L.layer_dims(K)
    W, B, Wh, bh = _weights_hilo(flat, K, dev)
    cols9 = torch.tensor([L.heads_column(K, o) for o in range(C3)], device=dev)
    M, tiles = lv["M"], lv["tiles"]
    view = lambda k: L.workspace_view(ws, lv, k)
    H, E, DZ, DO, Hl, El, DZl, DOl = (view(k) for k in ("H", "E", "DZ", "DO", "H_lo", "E_lo", "DZ_lo", "DO_lo"))
    MASK = view("mask")
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

    CH = 128
    for t0 in range(0, tiles, CH):
        t1 = min(tiles, t0 + CH)
        r0, r1 = t0 * L.TILE_M, t1 * L.TILE_M
        real = torch.arange(r0, r1, device=dev) < M
        e_hi, e_lo = L.decode_e(E[t0:t1]), L.decode_e(El[t0:t1])
        h_hi = [L.decode_h(H[t0:t1], l) for l in range(8)]
        h_lo = [L.decode_h(Hl[t0:t1], l) for l in range(8)]
        dz_hi = [L.decode_dz(DZ[t0:t1], l) for l in range(8)]
        dz_lo = [L.decode_dz(DZl[t0:t1], l) for l in range(8)]
        do_hi, do_lo = L.decode_do(DO[t0:t1]), L.decode_do(DOl[t0:t1])
        mask = [L.decode_mask(MASK[l, r0:r1]) for l in range(8)]
        nd = 64 * ((NH + 63) // 64)
        st.add("split_violations_e", _split_ok(e_hi, e_lo))
        st.add("split_violations_do", _split_ok(do_hi[:, :nd], do_lo[:, :nd]))
        st.add("split_violations_h", sum(_split_ok(a, b) for a, b in zip(h_hi, h_lo)))
        st.add("split_violations_dz", sum(_split_ok(a, b) for a, b in zip(dz_hi, dz_lo)))
        st.add("posenc_col63_not_one", int(((e_hi[:, 63] != 1) | (e_lo[:, 63] != 0)).sum()))
        e63 = _hilo(e_hi, e_lo)[:, :63]
        hd = [_hilo(a, b) for a, b in zip(h_hi, h_lo)]
        # ---- forward ----
        for l in range(8):
            a = e63 if l == 0 else (torch.cat([hd[4], e63], 1) if l == 5 else hd[l - 1])
            pre = a @ W[l] + B[l]
            amag = a.abs() @ W[l].abs() + B[l].abs()
            st.max("fwd_excess", _excess(h_hi[l], h_lo[l], pre.clamp_min(0), amag))
            pos = hd[l] > 0
            st.add("mask_clear_but_positive", int((pos & ~mask[l]).sum()))
            st.add("mask_set_value_zero", int((mask[l] & ~pos).sum()))     # relu(v) < 2^-25: hi = lo = 0
            st.add("mask_set_value_zero_not_tiny", int((mask[l] & ~pos & (pre > 2.0 ** -20)).sum()))
            st.add("h_nonfinite", int((~torch.isfinite(hd[l])).sum()))
        # ---- data gradient ----
        do_cols = 64 * ((NH + 63) // 64)            # chunks of the dO image mlp_bwd writes
        do_hi, do_lo = do_hi[:, :do_cols], do_lo[:, :do_cols]
        dod = _hilo(do_hi, do_lo)[:, :NH]
        dzd = [_hilo(a, b) for a, b in zip(dz_hi, dz_lo)]
        for x_hi, x_lo in [(do_hi, do_lo)] + list(zip(dz_hi, dz_lo)):
            st.add("padded_rows_nonzero", int(((x_hi[~real] != 0) | (x_lo[~real] != 0)).sum()))
        for l in range(7, -1, -1):
            a, Wt = (dod, Wh.T) if l == 7 else (dzd[l + 1], W[l + 1][:256].T)
            ref = (a @ Wt) * mask[l]
            amag = (a.abs() @ Wt.abs()) * mask[l]
            sub_row = ((a != 0) & (a.abs() < 2.0 ** -14)).any(1, keepdim=True)   # the row reads a subnormal operand
            normal = ~sub_row.expand_as(ref)
            ex = _excess(dz_hi[l], dz_lo[l], torch.where(normal, ref, _hilo(dz_hi[l], dz_lo[l])), amag)
            st.max("bwd_excess", ex)
            st.max(f"bwd_excess_dz{l}", ex)
            st.max("bwd_excess_subnormal_operand_rows", _excess(dz_hi[l], dz_lo[l], ref, amag))
            st.add("dz_masked_nonzero_bits", int(((dz_hi[l].view(torch.int16) != 0) | (dz_lo[l].view(torch.int16) != 0))[~mask[l]].sum()))
            st.add("dz_nonfinite", int((~torch.isfinite(dzd[l])).sum()))
            st.max("dz_headroom", float(dz_hi[l].abs().max()) / 65504.0)
            nz = dz_hi[l] != 0
            st.add("dz_nonzero", int(nz.sum()))
            st.add("dz_lo_subnormal", int((nz & (dz_lo[l].abs() < 2 ** -14)).sum()))
            st.max("dz_abs_max", float(dz_hi[l].abs().max()))
        # ---- weight-gradient sums ----
        for l in range(1, 8):
            wsum(f"w{l}", hd[l - 1] if l != 5 else torch.cat([hd[4], e63], 1), dzd[l])
        wsum("w0", e63, dzd[0])
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
            st.max(f"wgrad_{nm}_max_err_over_abs_sum", float((err / rmag[sl].clamp_min(1e-300)).max()))
            st.max(f"wgrad_{nm}_rel_l2", float(err.norm() / max(float(ref[sl].norm()), 1e-300)))


def _stage_case_x3(case):
    from plenoctree_b200.nerf.train import default_loss_scale
    from tests.support.mlp_stages import Stats
    model = case.model()
    state, ctx = _run(case, model, X3, fill=0xFF)
    ws = model.workspace(True, X3)
    views = L.train_workspace_views(model.cfg, ctx["n"], case.nsp > 0, precision=X3)
    assert views["total"] == ws.numel()
    # 1. the training forward's rgbs / comp / disp / acc are the x3 render's, bit for bit (same draws, same noise)
    from plenoctree_b200.nerf.models import Rays
    o, d, v = ctx["rays"]
    out = model(Rays(o, d, v), randomized=True, t_rand=ctx["t_rand"], u=ctx["u"], precision=X3,
                sigma_noise=ctx["noise"])
    torch.cuda.synchronize()
    rws = model.workspace(False)
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
    scale = default_loss_scale(ctx["n"], X3)
    params = model.params.cpu().numpy()
    res = {"render_bit_mismatches": mism}
    for i, lv in enumerate(views["levels"]):
        s = Stats()
        P = model.P
        _check_level_x3(ws, lv, params[i * P:(i + 1) * P], state.grads[i * P:(i + 1) * P], case, scale, s)
        res[f"MLP_{i}"] = dict(stages=s.d, M=lv["M"], tiles=lv["tiles"])
    _record(case.name, res)
    assert all(x == 0 for x in mism.values()), mism
    for mlp, r in res.items():
        if not mlp.startswith("MLP"):
            continue
        s = r["stages"]
        for k in ("split_violations_e", "split_violations_h", "split_violations_do", "split_violations_dz",
                  "posenc_col63_not_one", "mask_clear_but_positive", "mask_set_value_zero_not_tiny",
                  "h_nonfinite", "padded_rows_nonzero", "dz_masked_nonzero_bits", "dz_nonfinite"):
            assert s[k] == 0, (mlp, k, s[k])
        assert s["fwd_excess"] <= FWD_ALLOW, (mlp, s["fwd_excess"])
        assert s["bwd_excess"] <= BWD_ALLOW, (mlp, s["bwd_excess"])
        assert s["bwd_excess_subnormal_operand_rows"] <= BWD_SUBNORMAL_ALLOW, (mlp, s)
        assert s["dz_headroom"] < 1.0, (mlp, s["dz_headroom"])
        assert s["wgrad_w_max_err_over_abs_sum"] <= WG_EPS_W, (mlp, s)
        assert s["wgrad_b_max_err_over_abs_sum"] <= WG_EPS_B, (mlp, s)


def _oracle_inputs(seed, sh_deg=3, R=64, nf=128, nsp=64):
    from tests.support.mlp_stages import _setup
    return _setup(sh_deg, R, nf, nsp, seed)

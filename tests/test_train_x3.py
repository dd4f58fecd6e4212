"""The fp16x3 training step (pob_loss_and_grad_prec at POB_PREC_FP16X3): error-compensated operands x = hi + lo through
the saving forward, the data gradient and the three-pass weight gradient.

Stage checks read every intermediate back from the workspace (layouts.train_workspace_views(..., precision=3)) and
compare each with an fp64 evaluation from the kernel's own previous-stage hi + lo tiles and its hi + lo weights, in the
units test_train_stages.py uses: 2^-24 * sum |a*w| beyond the hi/lo representation error of the stored value.  End to
end, the gradient is compared with the fp64 oracle, next to the fp16 step's on the same inputs.
"""
import json
import os
import re

import numpy as np
import pytest
import torch

from plenoctree_b200 import layouts as L
from tests.test_train import OUT
from tests.test_train_stages import CASES, Case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U24 = 2.0 ** -24
X3 = 3

# ---- bars, measured on an H100 80 GB HBM3 at a 400 W power limit (largest value over the cases of this file in
# brackets), in units of 2^-24 * sum |a*w| beyond the representation error of the stored hi + lo.  An x3 bar must stay
# at least 2^7 below fp16's operand rounding (2^-11 = 2^13 units), or the mode is not what it claims.
FWD_ALLOW = 32.0            # [16.2]
BWD_ALLOW = 32.0            # [22.1]
assert max(FWD_ALLOW, BWD_ALLOW) <= 2.0 ** 13 / 2 ** 7
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


def _ulp16(x):
    """fp16 ulp at |x| (fp64 tensor), 2^-24 in the subnormal range.  The exponent comes from frexp: log2 on the GPU is
    not exact at every power of two (log2(8) < 3 there), which would halve the ulp of 8, 64, ..."""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -14))
    return torch.ldexp(torch.ones_like(x), (e - 11).to(torch.int64))


def _record(name, payload):
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, "parity_train_x3.json")
    data = json.load(open(path)) if os.path.exists(path) else {}
    data[name] = payload
    json.dump(data, open(path, "w"), indent=1)


# =====================================================================================================================
# CPU
# =====================================================================================================================
def test_x3_workspace_mirror_matches_library():
    """train_workspace_views(precision=3) reproduces carve() of the x3 step: same total as
    pob_train_workspace_bytes(cfg, 3); the fp16 size is pob_workspace_bytes(cfg, 1); the x3 buffers follow the fp16
    ones without overlap; a bad precision gives -1."""
    from plenoctree_b200._lib import RenderConfig, lib
    from plenoctree_b200.nerf.models import ctypes_ref
    n = 0
    for sh in range(-1, 5):
        for nc, nf in ((3, 0), (64, 0), (3, 5), (64, 128), (100, 156)):
            for nsp in (0, 1, 10000):
                for R in (1, 40, 4096):
                    cfg = RenderConfig(sh, nc, nf, 1, R, nsp)
                    assert lib.pob_train_workspace_bytes(ctypes_ref(cfg), 1) == lib.pob_workspace_bytes(ctypes_ref(cfg), 1)
                    want = int(lib.pob_train_workspace_bytes(ctypes_ref(cfg), X3))
                    for n_rays in sorted({1, R}):
                        v = L.train_workspace_views(cfg, n_rays, True, precision=X3)
                        v16 = L.train_workspace_views(cfg, n_rays, True)
                        assert v["total"] == want, (sh, nc, nf, nsp, R)
                        ext = []
                        for lv in v["levels"]:
                            for name in ("H_lo", "E_lo", "DZ_lo", "DO_lo"):
                                off, shape = lv[name]
                                assert shape == lv[name[:-3]][1]
                                ext.append((off, off + int(np.prod(shape))))
                        ext += [(o, o + 4 * L.WG_MAX_CTAS * L.WG_PARTIAL_FLOATS) for p in v["partials_x3"] for o in p]
                        ext += [(o, o + nb) for o, nb in v["wt_lo"]]
                        ext.sort()
                        assert ext[0][0] >= v16["total"]
                        for (a0, a1), (b0, _) in zip(ext, ext[1:] + [(want, 0)]):
                            assert a0 % 1024 == 0 and a1 <= b0
                        n += 1
    assert n > 300
    assert lib.pob_train_workspace_bytes(ctypes_ref(RenderConfig(3, 64, 128, 1, 8, 0)), 2) == -1


def _wgrad_roles():
    """wgrad_role(r) of kernels.h, read from the source: [(dense, a_op, b_op, skip, bias)]"""
    src = open(os.path.join(ROOT, "plenoctree_b200", "csrc", "kernels.h")).read()
    body = src[src.index("constexpr WgradRole wgrad_role(int r)"):]
    body = body[:body.index("}\n")]
    rows = re.findall(r"WgradRole\{([^}]*)\}", body)
    assert len(rows) == 3
    out = []
    for r in range(9):
        row = rows[0] if r < 7 else rows[1] if r == 7 else rows[2]
        f = [x.strip() for x in row.split(",")]
        skip = (r + 1 == 5) if r < 7 else False
        assert (f[6] == "r + 1 == SKIP_LAYER") if r < 7 else f[6] == "0"
        out.append(dict(a=f[1], b=f[3], skip=skip, bias=f[7]))
    return out


def _x3_passes():
    """the three WgradSegment {h, dz, e, d_o} of the x3 step, read from pipeline.cu: [{op: "hi" | "lo"}]"""
    src = open(os.path.join(ROOT, "plenoctree_b200", "csrc", "pipeline.cu")).read()
    m = re.search(r"segs\[X3_WGRAD_PASSES\] = \{(.*?)\};", src, re.S)
    segs = re.findall(r"\{([^{}]*)\}", m.group(1))
    assert len(segs) == 3
    out = []
    for s in segs:
        names = [x.strip().split(".")[1] for x in s.split(",")]
        out.append({op: ("lo" if nm.endswith("_lo") else "hi") for op, nm in zip(("WG_H", "WG_DZ", "WG_E", "WG_DO"), names)})
    return out


def test_x3_wgrad_passes_cover_every_product():
    """By linearity the x3 weight gradient is three runs of the unchanged mlp_wgrad over hi / lo tile images.  For
    every role of wgrad_role (and Dense_5's skip rows, A contracted with posenc) the passes give exactly lo*hi, hi*lo
    and hi*hi once each; the bias sums (columns of A, Dense_0: of B) of the first two passes give hi and lo once each,
    the third repeats hi (X3_BIAS_PASSES = 2)."""
    passes = _x3_passes()
    src = open(os.path.join(ROOT, "plenoctree_b200", "csrc", "kernels.h")).read()
    assert "constexpr int X3_WGRAD_PASSES = 3;" in src and "constexpr int X3_BIAS_PASSES = 2;" in src
    want = sorted([("lo", "hi"), ("hi", "lo"), ("hi", "hi")])
    for role in _wgrad_roles():
        pairs = [(p[role["a"]], p[role["b"]]) for p in passes]
        assert sorted(pairs) == want, (role, pairs)
        if role["skip"]:
            assert sorted((p[role["a"]], p["WG_E"]) for p in passes) == want
        col = role["a"] if role["bias"] == "WG_BIAS_A" else role["b"]
        assert sorted(p[col] for p in passes[:2]) == ["hi", "lo"], role
        assert passes[2][col] == "hi"


# =====================================================================================================================
# GPU
# =====================================================================================================================
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
    return 0.5 * _ulp16(lo.double())


def _excess(hi, lo, ref, mag):
    err = (_hilo(hi, lo) - ref).abs() - _repr_err(lo)
    return float((err.clamp_min(0) / (U24 * mag).clamp_min(1e-300)).max())


def _split_ok(hi, lo):
    """|lo| <= half an ulp of hi for every pair (lo = 0 where hi = 0)"""
    return int(((lo.double().abs() > 0.5 * _ulp16(hi.double()) * (hi != 0)) | ((hi == 0) & (lo != 0))).sum())


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
    from tests.test_train_stages import Stats
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


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_x3_train_stages(case):
    _stage_case_x3(case)


@pytest.mark.gpu
def test_x3_train_stages_production_step():
    """bench.py's step shape (4096 rays x (64 + 128) samples + 10 000 sparsity points): the dZ range that sets the
    x3 loss scale (dz_abs_max, dz_headroom, dz_lo_subnormal of dz_nonzero) is recorded from here."""
    from plenoctree_b200._lib import RenderConfig, lib
    from plenoctree_b200.nerf.models import ctypes_ref
    need = int(lib.pob_train_workspace_bytes(ctypes_ref(RenderConfig(3, 64, 128, 1, 4096, 10000)), X3))
    free, _ = torch.cuda.mem_get_info()
    if free < need + (8 << 30):
        pytest.skip(f"needs {need / 2**30:.1f} GB of workspace + ~8 GB for the reference; {free / 2**30:.1f} GB free")
    _stage_case_x3(Case(3, 4096, 64, 128, 10000))


def _oracle_inputs(seed, sh_deg=3, R=64, nf=128, nsp=64):
    from tests.test_train import _setup
    return _setup(sh_deg, R, nf, nsp, seed)


def _fp64_mask_disagreements(model, ws, views, rays, sp):
    """ReLU masks of the call in `ws` that disagree with an fp64 evaluation of the network (exact fp32 parameters) at
    the same sample positions (the workspace's depths, fp64 points): per level, summed over the eight layers."""
    dev = ws.device
    K = L.K_of(model.sh_deg)
    w_off, b_off, _ = L.flat_offsets(K)
    dims = L.layer_dims(K)
    o, d = (torch.from_numpy(a).to(dev).double() for a in rays[:2])
    out = []
    for i, lv in enumerate(views["levels"]):
        fl = model.params[i * model.P:(i + 1) * model.P].double()
        W = [fl[w_off[l]:w_off[l] + dims[l][0] * 256].view(dims[l][0], 256) for l in range(8)]
        B = [fl[b_off[l]:b_off[l] + 256] for l in range(8)]
        N, Mr, M = lv["N"], lv["M_rays"], lv["M"]
        z = L.workspace_view(ws, lv, "z").reshape(-1)[:Mr].double()
        ray = torch.arange(Mr, device=dev) // N
        x = o[ray] + z[:, None] * d[ray]
        if M > Mr:
            x = torch.cat([x, torch.from_numpy(sp).to(dev).double()])
        xb = (x[:, None, :] * torch.exp2(torch.arange(10, device=dev, dtype=torch.float64))[None, :, None]).reshape(-1, 30)
        e = torch.cat([x, torch.sin(xb), torch.sin(xb + np.pi / 2)], 1)
        mask = L.workspace_view(ws, lv, "mask")
        n, h = 0, None
        for l in range(8):
            a = e if l == 0 else (torch.cat([h, e], 1) if l == 5 else h)
            pre = a @ W[l] + B[l]
            n += int((L.decode_mask(mask[l, :M]) != (pre > 0)).sum())
            h = pre.clamp_min(0)
        out.append(n)
    return out


def _oracle_grads(fc, ff, rays, px, cfg, t_rand, u, sp, dtype, z_fine=None):
    from oracle import nerf_sh_oracle as O
    st, gc, gf = O.loss_and_grads(fc, ff, 3, rays, px, cfg, t_rand, u, sp, dtype=dtype, z_fine=z_fine)
    return st, np.concatenate([gc, gf]).astype(np.float64)


@pytest.mark.gpu
def test_x3_gradient_vs_fp64_oracle():
    """Against the fp64 oracle with the same draws and the oracle's fine-level depths: loss statistics within
    LOSS_REL; the whole gradient at the fp32 floor (FLOOR_SLACK) and GRAD_GAIN times closer to the fp32 oracle than
    the fp16 step's.  The ReLU masks that disagree with fp64 are recorded for both steps."""
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf import train as T
    R, nf, nsp = 96, 128, 300
    fc, ff, rays, px, t_rand, u, sp = _oracle_inputs(77, 3, R, nf, nsp)
    cfg = dict(num_coarse_samples=64, num_fine_samples=nf, near=2.0, far=6.0, white_bkgd=True,
               sparsity_weight=1e-3, sparsity_length=0.05)
    stats_o, ref = _oracle_grads(fc, ff, rays, px, cfg, t_rand, u, sp, torch.float64)
    zf = stats_o.pop("_z_fine").astype(np.float32)
    _, ref32 = _oracle_grads(fc, ff, rays, px, cfg, t_rand, u, sp, torch.float32, z_fine=zf)
    rel = lambda g, r: float(np.linalg.norm(g - r) / np.linalg.norm(r))
    model = NerfModel(sh_deg=3, num_coarse_samples=64, num_fine_samples=nf, max_rays=R, sparsity_npoints=nsp)
    model.set_params(np.concatenate([fc, ff]))
    rep = {"fp32_oracle_vs_fp64": rel(ref32, ref)}
    for name, prec in (("fp16", 1), ("fp16x3", X3)):
        state = T.TrainState(model)
        n = T.loss_and_grad(model, state, {"rays": Rays(*rays), "pixels": px}, sparsity_weight=1e-3,
                            sparsity_length=0.05, randomized=True, t_rand=t_rand, u=u, sp_points=sp, z_fine=zf,
                            precision=prec)
        torch.cuda.synchronize()
        g = state.grads.double().cpu().numpy()
        st = T.stats_from_raw(state.stats_raw, n, 1e-3, nsp, True)
        views = L.train_workspace_views(model.cfg, n, True, precision=prec)
        rep[name] = dict(grad_rel_l2=rel(g, ref), grad_rel_l2_vs_fp32_oracle=rel(g, ref32),
                         loss_rel=abs(st.loss - stats_o["loss"]) / stats_o["loss"],
                         loss_c_rel=abs(st.loss_c - stats_o["loss_c"]) / stats_o["loss_c"],
                         loss_sp_abs=abs(st.loss_sp - stats_o["loss_sp"]),
                         relu_masks_disagreeing_with_fp64=_fp64_mask_disagreements(
                             model, model.workspace(True, prec), views, rays, sp))
    rep["gain_vs_fp64"] = rep["fp16"]["grad_rel_l2"] / rep["fp16x3"]["grad_rel_l2"]
    rep["gain_vs_fp32_oracle"] = rep["fp16"]["grad_rel_l2_vs_fp32_oracle"] / rep["fp16x3"]["grad_rel_l2_vs_fp32_oracle"]
    _record("vs_fp64_oracle", rep)
    x = rep["fp16x3"]
    assert x["loss_rel"] < LOSS_REL and x["loss_c_rel"] < LOSS_REL, rep
    assert x["loss_sp_abs"] < LOSS_REL * max(abs(stats_o["loss_sp"]), 1e-6) + 1e-8, rep
    assert x["grad_rel_l2"] <= FLOOR_SLACK * rep["fp32_oracle_vs_fp64"], rep
    assert rep["gain_vs_fp32_oracle"] >= GRAD_GAIN, rep


@pytest.mark.gpu
def test_x3_six_adam_steps_vs_fp64_oracle():
    """Six optimisation steps from the same parameters and draws, against an fp64 and an fp32 oracle run (fine depths
    pinned to the fp64 run's): the x3 update at the fp32 floor and GRAD_GAIN times closer to the fp32 run than the fp16
    update."""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf import train as T
    R, nf, nsp, steps, lr = 48, 128, 64, 6, 5e-4
    fc0, ff0, rays, px, _, _, _ = _oracle_inputs(91, 3, R, nf, nsp)
    cfg = dict(num_coarse_samples=64, num_fine_samples=nf, near=2.0, far=6.0, white_bkgd=True,
               sparsity_weight=1e-3, sparsity_length=0.05)
    rs = np.random.RandomState(5)
    draws = [(rs.uniform(size=(R, 64)).astype(np.float32), rs.uniform(size=(R, nf)).astype(np.float32),
              rs.uniform(-1.5, 1.5, size=(nsp, 3)).astype(np.float32)) for _ in range(steps)]
    p0 = np.concatenate([fc0, ff0])
    zfs = []
    dp_ref = {}
    for dt in (torch.float64, torch.float32):
        npdt = np.float64 if dt == torch.float64 else np.float32
        fc, ff = fc0.astype(npdt), ff0.astype(npdt)
        mo = [np.zeros_like(fc), np.zeros_like(ff)]
        vo = [np.zeros_like(fc), np.zeros_like(ff)]
        for step, (t_rand, u, sp) in enumerate(draws):
            zf = zfs[step] if dt == torch.float32 else None
            stats_o, gc, gf = O.loss_and_grads(fc, ff, 3, rays, px, cfg, t_rand, u, sp, dtype=dt, z_fine=zf)
            if dt == torch.float64:
                zfs.append(stats_o["_z_fine"].astype(np.float32))
            fc, mo[0], vo[0] = O.adam_step(fc, gc.astype(npdt), mo[0], vo[0], float(step), lr)
            ff, mo[1], vo[1] = O.adam_step(ff, gf.astype(npdt), mo[1], vo[1], float(step), lr)
        dp_ref[dt] = np.concatenate([fc, ff]).astype(np.float64) - p0
    rel = lambda a, b: float(np.linalg.norm(a - b) / np.linalg.norm(b))
    rep = {"fp32_oracle_vs_fp64": rel(dp_ref[torch.float32], dp_ref[torch.float64])}
    for name, prec in (("fp16", 1), ("fp16x3", X3)):
        model = NerfModel(sh_deg=3, num_coarse_samples=64, num_fine_samples=nf, max_rays=R, sparsity_npoints=nsp)
        model.set_params(p0)
        state = T.TrainState(model)
        for (t_rand, u, sp), zf in zip(draws, zfs):
            T.loss_and_grad(model, state, {"rays": Rays(*rays), "pixels": px}, sparsity_weight=1e-3,
                            sparsity_length=0.05, t_rand=t_rand, u=u, sp_points=sp, z_fine=zf, precision=prec)
            check(lib.pob_adam_update(model.sh_deg, model.num_mlps, ptr(model.params), ptr(state.grads),
                                      ptr(state.m), ptr(state.v), float(lr), float(state.step), None, 1.0, 0.0,
                                      ptr(model.blobs[0]), ptr(model.blobs[1]), stream_ptr()))
            state.step += 1
        dp = model.params.double().cpu().numpy() - p0
        rep[name] = dict(vs_fp64=rel(dp, dp_ref[torch.float64]), vs_fp32_oracle=rel(dp, dp_ref[torch.float32]))
    rep["gain_vs_fp64"] = rep["fp16"]["vs_fp64"] / rep["fp16x3"]["vs_fp64"]
    rep["gain_vs_fp32_oracle"] = rep["fp16"]["vs_fp32_oracle"] / rep["fp16x3"]["vs_fp32_oracle"]
    _record("six_adam_steps_vs_fp64_oracle", rep)
    assert rep["fp16x3"]["vs_fp64"] <= FLOOR_SLACK * rep["fp32_oracle_vs_fp64"], rep
    assert rep["gain_vs_fp32_oracle"] >= GRAD_GAIN, rep


@pytest.mark.gpu
def test_x3_graphed_matches_eager_and_repeats_bitwise():
    """GraphedTrainStep(precision=x3) reproduces eager x3 train_step bit for bit (parameters and Adam moments), and
    two x3 gradient calls on the same inputs are bit-identical."""
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf import train as T
    R = 256
    fc, ff, rays, px, _, _, _ = _oracle_inputs(33, 3, R, 128, 0)
    b12 = torch.from_numpy(np.concatenate([rays[0], rays[1], rays[2], px], axis=1)).cuda()
    lrs = [5e-4, 4e-4, 3e-4]
    outs = []
    for graphed in (False, True):
        model = NerfModel(sh_deg=3, max_rays=R, sparsity_npoints=1000)
        model.set_params(np.concatenate([fc, ff]))
        state = T.TrainState(model)
        if graphed:
            g = T.GraphedTrainStep(model, state, R, precision=X3)
            for lr in lrs:
                g.step(b12, lr)
        else:
            batch = {"rays": Rays(b12[:, 0:3], b12[:, 3:6], b12[:, 6:9]), "pixels": b12[:, 9:12]}
            for lr in lrs:
                T.train_step(model, state, batch, lr, precision=X3)
        torch.cuda.synchronize()
        outs.append((model.params.clone(), state.m.clone(), state.v.clone()))
    for name, a, b in zip(("params", "m", "v"), *outs):
        assert torch.equal(a, b), name
    case = Case(3, 96, 64, 128, 300)
    model = case.model()
    g1 = _run(case, model, X3)[0].grads.clone()
    g2 = _run(case, model, X3, fill=0xFF)[0].grads.clone()
    assert torch.isfinite(g1).all() and torch.equal(g1, g2)


@pytest.mark.gpu
def test_x3_call_leaves_fp16_results_alone():
    """An x3 call between two fp16 calls does not change the fp16 gradient (separate workspaces, same blobs)."""
    case = Case(3, 96, 64, 128, 300)
    model = case.model()
    g_a = _run(case, model, 1)[0].grads.clone()
    g_x3 = _run(case, model, X3)[0].grads.clone()
    g_b = _run(case, model, 1)[0].grads.clone()
    assert torch.equal(g_a, g_b)
    assert not torch.equal(g_a, g_x3)


@pytest.mark.gpu
def test_x3_argument_errors():
    """bad precision, NULL params in x3 and a workspace sized for the fp16 step fail through pob_last_error"""
    from plenoctree_b200._lib import PobError, TrainHParams, check, lib, ptr, stream_ptr
    from plenoctree_b200.nerf.models import ctypes_ref
    case = Case(3, 8, 64, 0, 0)
    model = case.model()
    (o, d, v, px), t_rand, _, _, _ = case.inputs(8)
    dev = lambda a: torch.from_numpy(a).cuda()
    o, d, v, px, t_rand = (dev(a) for a in (o, d, v, px, t_rand))
    g = torch.zeros(model.P + 8, device="cuda")
    hp = TrainHParams(0.0, 0.05, 1024.0)
    # a plain cudaMalloc of the fp16 size: the check sees the allocation's extent (a block a caching allocator cuts
    # out of a larger allocation is beyond what the library can see)
    import ctypes
    lib.cudaMalloc.argtypes, lib.cudaFree.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_size_t], [ctypes.c_void_p]
    raw = ctypes.c_void_p()
    assert lib.cudaMalloc(ctypes.byref(raw), int(lib.pob_train_workspace_bytes(ctypes_ref(model.cfg), 1))) == 0
    ws16 = type("Raw", (), dict(data_ptr=lambda self: raw.value))()
    ws3 = model.workspace(True, X3)

    def call(ws, params, prec):
        check(lib.pob_loss_and_grad_prec(ctypes_ref(model.cfg), ctypes_ref(hp), ptr(model.blobs[0]), None, ptr(o),
                                         ptr(d), ptr(v), ptr(px), 8, ptr(model.z_base), ptr(t_rand), None, 0, None,
                                         None, ptr(g), ptr(g[model.P:]), ptr(ws), None, ptr(params), prec,
                                         stream_ptr()))
    for ws, params, prec, msg in ((ws3, model.params, 2, "precision"), (ws3, None, X3, "params_dev"),
                                  (ws16, model.params, X3, "workspace too small")):
        with pytest.raises(PobError, match=msg):
            call(ws, params, prec)
    call(ws3, model.params, X3)
    call(ws16, None, 1)
    torch.cuda.synchronize()
    lib.cudaFree(raw)


@pytest.mark.gpu
def test_train_cli_fp16x3_writes_loadable_checkpoint(tmp_path):
    """a few steps of `nerf_sh.train --train_precision fp16x3` on a small synthetic Blender scene, then nerf_sh.eval
    loads the checkpoint"""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf import datasets as D
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf.utils import generate_rays, pose_spherical, render_image
    from plenoctree_b200.nerf_sh import eval as EV, train as TR
    from tests.test_pipeline import _set_flags
    sh_deg, W = 3, 32
    ft = np.concatenate([O.init_flat_params(sh_deg, 7001, bias_scale=0.05), O.init_flat_params(sh_deg, 7002, bias_scale=0.05)])
    teacher = NerfModel(sh_deg=sh_deg, max_rays=4096)
    teacher.set_params(ft)
    cam_x = 0.6911112070083618
    focal = 0.5 * W / np.tan(0.5 * cam_x)
    rs = np.random.RandomState(3)
    splits = {"train": 4, "val": 1, "test": 1}
    poses = {k: [pose_spherical(rs.uniform(-180, 180), rs.uniform(-80, -10), 4.0) for _ in range(n)] for k, n in splits.items()}
    images = {}
    for k in splits:
        rays = generate_rays(W, W, focal, np.stack(poses[k]))
        images[k] = [render_image(teacher, Rays(rays.origins[i], rays.directions[i], rays.viewdirs[i]))[0].cpu().numpy()
                     for i in range(splits[k])]
    data_dir, train_dir = str(tmp_path / "scene"), str(tmp_path / "ckpt")
    D.write_blender_scene(data_dir, images, poses, cam_x)
    (tmp_path / "cfg.yaml").write_text("dataset: blender\nfactor: 0\nnum_coarse_samples: 64\nnum_fine_samples: 128\n"
                                       "use_viewdirs: false\nwhite_bkgd: true\nbatch_size: 512\nsh_deg: 3\n"
                                       "randomized: true\nmax_steps: 5\n")
    FLAGS = _set_flags(train_dir=train_dir, data_dir=data_dir, config=str(tmp_path / "cfg"), save_every=5,
                       print_every=5, render_every=0, sparsity_npoints=1000, lr_init=2e-3, lr_final=2e-4, chunk=4096,
                       noise_std=None, image_batching=True)
    FLAGS.train_precision = "fp16x3"
    try:
        model, state = TR.main(None)
    finally:
        FLAGS.train_precision = "fp16"
    assert os.path.exists(os.path.join(train_dir, "checkpoint_5")) and state.step == 5
    assert torch.isfinite(model.params).all()
    psnr, _ = EV.main(None)
    assert np.isfinite(psnr)

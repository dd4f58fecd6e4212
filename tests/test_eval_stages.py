"""Parity of the inference forwards of csrc/mlp_fwd.cu (no saves): render, point evaluation, grid sweep, cell means.

tests/test_eval_points.py and tests/test_render.py hold these forwards to the fp32 oracle at the north-star bars, which
measure precision and leave room for a fault confined to a few columns, one K-slot or one layer.  Here:

- fp16: without saves the forward issues the instruction sequence of the saving training forward (SAVE only adds
  stores of the same registers), so for the same point and view direction every instantiation must return the training
  forward's rgbs bit for bit, and test_train_stages.py checks that forward against fp64 stage by stage.  OUT_RAW heads
  and cell means, which the training forward does not produce, are checked against fp64 from its saved h_7 tiles.
- fp16x3: against an fp64 evaluation of the whole network with the operands the kernel represents (weights hi + lo as
  pack.cu splits them, posenc from the fp32 arguments, exact ReLU), in units of the heads GEMM's 2^-24 * sum |h_7 w|.
  A rigorous propagated bound would be ~10^9 too loose (|W| grows the error ~14x per layer), so the bar is measured,
  and a sensitivity guard shows that dropping one error-compensation term moves the reference well past it.
- cell means: against the fp64 mean of the same precision's OUT_RAW rows at the standard summation bound.
- ragged sizes, several tiles per CTA, canaries behind every output and run-to-run determinism.
"""
import json
import os
import time

import numpy as np
import pytest
import torch

from plenoctree_b200 import layouts as L
from tests.test_train import OUT
from tests.test_train_stages import (CASES, FWD_ALLOW, SENSITIVITY, U24, Case, _assert_stages, _check_all,
                                     _sh_basis)

# ---- bars (measured on an H100 80 GB HBM3 at a 400 W power limit; the largest value over all cases of this file in brackets)
# fp16x3 against fp64: error of every OUT_RAW / OUT_SIGMA value in units of 2^-24 * sum_k |h_7,k w_k| of the heads GEMM
# (points 33.9, grid 28.1, render 31.1; relative to the largest magnitude: sigma 4.6e-6, rgb 3.6e-6)
X3_ALLOW = 68.0             # [33.9]
# Sensitivity classes that cannot reach SENSITIVITY x X3_ALLOW; their ratios are recorded, and only that the perturbed
# reference alone would fail the bar (ratio >= 1) is asserted.  The fp16x3 error is itself the sum of the residues of
# the error compensation over ~75 K-slots, propagated through the trunk, so leaving out one slot's compensation term
# moves the output by only a few times that error: measured over all cases, trunk K-slot hi*hi [3.8 .. 7.5] x the bar,
# one weight slot's lo part [9.7 .. 13.7], one posenc unit's lo part [7.4 .. 13.8], the heads bias's lo part (a 2^-12
# relative change of a bias of ~0.05) [1.6 .. 4.8].  The heads in a single fp16 pass reach [32 .. 48] and are asserted.
X3_SENS_UNASSERTED = ("trunk_slot_hi_hi", "weight_slot_lo_dropped", "posenc_unit_lo_dropped", "heads_bias_hi_only")
EPI_ABS = 2.0 ** -21        # rgb epilogue: expf + division, absolute (as in test_train_stages._check_level)
CANARY = 0x7FBADBAD         # a NaN bit pattern behind every output of the direct C-ABI calls
M_RAGGED = (1, 63, 64, 65, 127, 128, 129, 255, 257, 513)
CELL_S = (1, 5, 32, 33, 96, 128, 256, 384)
CHUNK = 1 << 17             # rows per fp64 reference chunk


def _record(name, payload):
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, "parity_eval_stages.json")
    data = json.load(open(path)) if os.path.exists(path) else {}
    data[name] = payload
    json.dump(data, open(path, "w"), indent=1)


def _nbits(a, b):
    """number of 32-bit words that differ between two float32 tensors of the same shape"""
    assert a.shape == b.shape, (a.shape, b.shape)
    return int((a.contiguous().view(torch.int32) != b.contiguous().view(torch.int32)).sum())


def _sms():
    from plenoctree_b200._lib import lib
    return int(lib.pob_sm_count())


def _m_many_tiles():
    """rows that give every CTA at least nine 128-row tiles: each tile advances the fp16 ring (4 stages) or the x3 ring
    (2 stages) by 75 stages, 75 = 3 mod 8, so nine tiles take every CTA through all ring phases"""
    return 9 * _sms() * L.TILE_M + 77


# =====================================================================================================================
# direct C-ABI calls with a canary behind every output
# =====================================================================================================================
def _canary(n, tail=4096):
    return torch.full((n + tail,), CANARY, dtype=torch.int32, device="cuda")


def _tail_ok(buf, n):
    return bool((buf[n:] == CANARY).all())


def _raw(blob, sh, pts, prec, want_rgb=True, pe=None, act=0):
    """pob_eval_points_raw -> (raw_rgb [m, 3K] reference channel-major | None, raw_sigma [m]); pe (encoder) or act
    (trunk activation, _lib.NET_*) away from the default: pob_eval_points_raw_pe with that descriptor"""
    from plenoctree_b200._lib import check, lib, posenc_ref, posenc_struct, ptr, stream_ptr
    m, C3 = pts.shape[0], 3 * L.K_of(sh)
    rb = _canary(m * C3) if want_rgb else None
    sb = _canary(m)
    d = posenc_struct(pe, act)
    if d is None:
        check(lib.pob_eval_points_raw(ptr(blob), sh, ptr(pts), m, ptr(rb), ptr(sb), prec, stream_ptr()))
    else:
        check(lib.pob_eval_points_raw_pe(ptr(blob), sh, posenc_ref(d), ptr(pts), m, ptr(rb), ptr(sb), prec,
                                         stream_ptr()))
    torch.cuda.synchronize()
    assert _tail_ok(sb, m) and (rb is None or _tail_ok(rb, m * C3)), ("write past the output", m)
    return (rb[:m * C3].view(torch.float32).view(m, C3) if want_rgb else None), sb[:m].view(torch.float32)


def _rgbs(blob, sh, pts, vd, prec):
    """pob_eval_points -> rgbs [m, 4] (sigmoid rgb, relu sigma)"""
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    m = pts.shape[0]
    ob = _canary(4 * m)
    check(lib.pob_eval_points(ptr(blob), sh, ptr(pts), ptr(vd), m, ptr(ob), prec, stream_ptr()))
    torch.cuda.synchronize()
    assert _tail_ok(ob, 4 * m), ("write past the output", m)
    return ob[:4 * m].view(torch.float32).view(m, 4)


def _grid(blob, sh, reso, off, sc, x0, nx, ny, nz, prec, want_rgb):
    import ctypes
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    m, C3 = nx * ny * nz, 3 * L.K_of(sh)
    rb = _canary(m * C3) if want_rgb else None
    sb = _canary(m)
    check(lib.pob_eval_grid(ptr(blob), sh, reso, x0, nx, ny, nz, (ctypes.c_float * 3)(*off),
                            (ctypes.c_float * 3)(*sc), ptr(rb), ptr(sb), prec, stream_ptr()))
    torch.cuda.synchronize()
    assert _tail_ok(sb, m) and (rb is None or _tail_ok(rb, m * C3)), ("write past the output", m)
    return (rb[:m * C3].view(torch.float32).view(m, C3) if want_rgb else None), sb[:m].view(torch.float32)


def _cells(blob, sh, pts, n_cells, S, prec, pe=None, act=0):
    from plenoctree_b200._lib import check, lib, posenc_ref, posenc_struct, ptr, stream_ptr
    W = 3 * L.K_of(sh) + 1
    ob = _canary(n_cells * W)
    d = posenc_struct(pe, act)
    if d is None:
        check(lib.pob_eval_cells_mean(ptr(blob), sh, ptr(pts), n_cells, S, ptr(ob), prec, stream_ptr()))
    else:
        check(lib.pob_eval_cells_mean_pe(ptr(blob), sh, posenc_ref(d), ptr(pts), n_cells, S, ptr(ob), prec,
                                         stream_ptr()))
    torch.cuda.synchronize()
    assert _tail_ok(ob, n_cells * W), ("write past the output", n_cells, S)
    return ob[:n_cells * W].view(torch.float32).view(n_cells, W)


def _blob(flat, sh):
    from plenoctree_b200 import ops
    return ops.pack_weights(torch.as_tensor(flat, dtype=torch.float32).cuda().contiguous(), sh)


# =====================================================================================================================
# fp64 references
# =====================================================================================================================
def _heads_params(flat, K, dev, enc_width=L.ENC_DIM):
    """packed heads weight [256, NH] and bias [NH] (fp32) on dev, and the channel-major index of the 3K rgb columns"""
    Wh, bh = L.heads_matrix(np.asarray(flat, np.float32), K, enc_width)
    cols9 = torch.tensor([L.heads_column(K, o) for o in range(3 * K)], device=dev)
    return torch.from_numpy(Wh).to(dev), torch.from_numpy(bh).to(dev), cols9


def _raw_of_heads(heads, cols9):
    """packed heads [n, NH] -> (raw_rgb channel-major [n, 3K], raw_sigma [n])"""
    return heads[:, cols9], heads[:, 0]


def _rgb_check(rgb, raw_rgb, hm_rgb, vd, sh, allow):
    """the heads epilogue from the GPU's own OUT_RAW values: max of |rgb - sigmoid(sum_k Y_k raw_ck)| over its allowance
    (test_train_stages._check_level: sigmoid slope 1/4 times the GEMM allowance plus 4 ulps of each coefficient, plus
    EPI_ABS for expf and the division).  raw_rgb / hm_rgb channel-major [n, 3K] fp64."""
    n, K = raw_rgb.shape[0], L.K_of(sh)
    Y = _sh_basis(sh, vd.double()) if sh >= 0 else torch.ones(n, 1, dtype=torch.float64, device=vd.device)
    r = raw_rgb.view(n, 3, K)
    pre = (Y[:, None, :] * r).sum(2)
    tol = 0.25 * (Y.abs()[:, None, :] * (allow * U24 * hm_rgb.view(n, 3, K) + 4 * U24 * r.abs())).sum(2) + EPI_ABS
    return float(((rgb.double() - torch.sigmoid(pre)).abs() / tol).max())


def _hilo(w):
    """fp32 -> (hi, lo) fp64, the split layouts.pack_reference (and pack.cu) applies to every weight and bias"""
    hi = w.half()
    lo = (w - hi.float()).half()
    return hi.double(), lo.double()


class X3Ref:
    """fp64 evaluation of one MLP with the operands the fp16x3 forward represents: weights and biases hi + lo,
    posenc of encoder pe from the fp32 arguments (x * 2^j exact, + fp32(pi/2) as an fp32 add, fp64 sine), the trunk
    activation act in fp64 (relu exact)."""

    def __init__(self, flat, sh, dev, pe=None, act="relu"):
        from oracle import posenc_oracle as PO
        from oracle import net_activation_oracle as NA
        self.pe = PO.DEFAULT if pe is None else tuple(pe)
        self.act = NA.activation(act)
        W = PO.width(self.pe)
        K = self.K = L.K_of(sh)
        w_off, b_off, _ = L.flat_offsets(K, W)
        dims = L.layer_dims(K, W)
        fl = torch.as_tensor(np.asarray(flat, np.float32)).to(dev)
        self.Whi, self.W, self.B = [], [], []
        for l in range(8):
            hi, lo = _hilo(fl[w_off[l]:w_off[l] + dims[l][0] * 256].view(dims[l][0], 256))
            self.Whi.append(hi)
            self.W.append(hi + lo)
            bhi, blo = _hilo(fl[b_off[l]:b_off[l] + 256])
            self.B.append(bhi + blo)
        Wh, bh, self.cols9 = _heads_params(flat, K, dev, W)
        hi, lo = _hilo(Wh)
        self.Wh_hi, self.Wh = hi, hi + lo
        hi, lo = _hilo(bh)
        self.bh_hi, self.bh = hi, hi + lo

    def __call__(self, x, pert=None):
        """x fp32 [n, 3] -> (packed heads [n, NH], sum |h_7 w| + |b| [n, NH]) in fp64.  pert: one term of the error
        compensation left out (sensitivity guard)."""
        from tests.test_posenc import _ref_features
        e = torch.cat([x.double(), _ref_features(x, self.pe)], 1)
        if pert == "posenc_unit_lo_dropped":        # one 8-column unit of the posenc tile, hi part only
            e = e.clone()
            e[:, 16:24] = e[:, 16:24].half().double()
        h = h4 = None
        for l in range(8):
            a = e if l == 0 else (torch.cat([h4, e], 1) if l == 5 else h)
            W = self.W[l]
            if pert == "weight_slot_lo_dropped" and l == 6:   # K-slot 2 of layer 6: hi part of the weights only
                W = W.clone()
                W[64:96] = self.Whi[6][64:96]
            pre = a @ W + self.B[l]
            if pert == "trunk_slot_hi_hi" and l == 3:          # K-slot 5 of layer 3 evaluated hi * hi only
                s = slice(160, 192)
                pre = pre - a[:, s] @ W[s] + a[:, s].half().double() @ self.Whi[3][s]
            h = self.act(pre)
            if l == 4:
                h4 = h
        if pert == "heads_single_pass":
            heads = h.half().double() @ self.Wh_hi + self.bh_hi
        else:
            heads = h @ self.Wh + (self.bh_hi if pert == "heads_bias_hi_only" else self.bh)
        return heads, h.abs() @ self.Wh.abs() + self.bh.abs()


SENS_CLASSES = ("trunk_slot_hi_hi", "weight_slot_lo_dropped", "posenc_unit_lo_dropped", "heads_bias_hi_only",
                "heads_single_pass")


def _x3_errors(ref, x, raw_rgb, raw_sig, st, key):
    """fp16x3 OUT_RAW values against the fp64 reference, chunked: running maxima of the error in units of
    2^-24 * sum |h_7 w| and of |err| / max |ref| per output, under `key`."""
    for r0 in range(0, x.shape[0], CHUNK):
        r1 = min(x.shape[0], r0 + CHUNK)
        heads, mag = ref(x[r0:r1])
        rr, rs = _raw_of_heads(heads, ref.cols9)
        mr, ms = _raw_of_heads(mag, ref.cols9)
        er = (raw_rgb[r0:r1].double() - rr).abs()
        es = (raw_sig[r0:r1].double() - rs).abs()
        st.max(f"{key}_excess", max(float((er / (U24 * mr)).max()), float((es / (U24 * ms)).max())))
        st.max(f"{key}_abs_rgb", er.max())
        st.max(f"{key}_abs_sigma", es.max())
        st.max(f"{key}_refmax_rgb", rr.abs().max())
        st.max(f"{key}_refmax_sigma", rs.abs().max())


def _rel(st, key):
    d = st.d
    return dict(rgb=d[f"{key}_abs_rgb"] / d[f"{key}_refmax_rgb"], sigma=d[f"{key}_abs_sigma"] / d[f"{key}_refmax_sigma"])


class Stats:
    def __init__(self):
        self.d = {}

    def max(self, key, val):
        self.d[key] = max(self.d.get(key, float("-inf")), float(val))

    def add(self, key, val):
        self.d[key] = self.d.get(key, 0) + int(val)


# =====================================================================================================================
# A + B: fp16 render / point evaluation bit-identical to the training forward; OUT_RAW heads against fp64
# =====================================================================================================================
def _level_rows(ctx, lv, z, sp, dev):
    """fp32 point (separate multiply and add, as cast_rays) and view direction of every row of one level; free
    (sparsity) rows use their own points and ray 0's direction, as the kernel does"""
    o, d, v = (torch.from_numpy(a).to(dev) for a in ctx["rays"])
    N, Mr, M = lv["N"], lv["M_rays"], lv["M"]
    s = torch.arange(M, device=dev)
    ray = (s // N).clamp_max(ctx["n"] - 1)
    x = o[ray] + z.reshape(-1)[s.clamp_max(Mr - 1)][:, None] * d[ray]
    if M > Mr:
        x = torch.where((s >= Mr)[:, None], sp[(s - Mr).clamp_min(0)], x)
    vd = v[torch.where(s < Mr, ray, torch.zeros_like(ray))]
    return x.contiguous(), vd.contiguous()


def _fp16_vs_training(case, check_stages=False):
    from plenoctree_b200 import ops
    from plenoctree_b200.nerf.models import Rays
    t0 = time.time()
    dev = torch.device("cuda")
    model = case.model()
    state, ctx = case.run(model, fill=0xFF)
    res = {}
    if check_stages:
        res = _check_all(case, model, state, ctx, case.nsp > 0)
    n = ctx["n"]
    ws = model.workspace(True)
    tv = L.train_workspace_views(model.cfg, n, case.nsp > 0)
    names = ("z", "rgbs", "weights", "comp", "disp", "acc")
    saved = [{k: L.workspace_view(ws, lv, k).clone() for k in names} for lv in tv["levels"]]

    # render with the training call's jitter, uniforms and noise, fp16, on the render workspace
    (o, d, v, _), t_rand, u, sp, noise = case.inputs(n)
    rws = model.workspace(False)
    rws.fill_(0xFF)
    outs = model(Rays(o, d, v), randomized=True, t_rand=t_rand, u=u, sigma_noise=noise, precision=ops.PREC_FP16)
    torch.cuda.synchronize()
    rv = L.train_workspace_views(model.cfg, n, False, training=False)
    assert rv["total"] == rws.numel()
    spt = torch.from_numpy(sp).to(dev) if sp is not None else None
    K = L.K_of(case.sh)
    params = model.params
    out = {}
    for i, (lt, lr) in enumerate(zip(tv["levels"], rv["levels"])):
        st = Stats()
        ref = saved[i]
        Mr, M = lt["M_rays"], lt["M"]
        for k in ("z", "weights", "comp", "disp", "acc"):
            st.add("render_ws_bit_mismatches", _nbits(L.workspace_view(rws, lr, k), ref[k]))
        st.add("render_ws_bit_mismatches", _nbits(L.workspace_view(rws, lr, "rgbs"), ref["rgbs"][:Mr]))
        rgb_o, disp_o, acc_o = outs[i]
        st.add("render_out_bit_mismatches", _nbits(rgb_o.contiguous(), ref["comp"]) + _nbits(disp_o.contiguous(), ref["disp"])
               + _nbits(acc_o.contiguous(), ref["acc"]))

        # point evaluation of the same rows (SRC_POINTS): OUT_RGBS, OUT_SIGMA, OUT_RAW
        blob = model.blobs[i]
        x, vd = _level_rows(ctx, lt, ref["z"], spt if i == len(tv["levels"]) - 1 else None, dev)
        got = _rgbs(blob, case.sh, x, vd, ops.PREC_FP16)
        raw_rgb, raw_sig = _raw(blob, case.sh, x, ops.PREC_FP16)
        _, sig_only = _raw(blob, case.sh, x, ops.PREC_FP16, want_rgb=False)
        st.add("eval_points_rgb_bit_mismatches", _nbits(got[:, :3], ref["rgbs"][:, :3]))
        st.add("sigma_only_vs_raw_bit_mismatches", _nbits(sig_only, raw_sig))
        if not case.noise:                      # noised sigma in the training rows
            st.add("eval_points_sigma_bit_mismatches", _nbits(got[:, 3], ref["rgbs"][:, 3]))
            st.add("sigma_only_relu_mismatches", int((sig_only.clamp_min(0) != ref["rgbs"][:, 3]).sum()))
            st.add("raw_sigma_relu_mismatches", int((raw_sig.clamp_min(0) != ref["rgbs"][:, 3]).sum()))

        # B: OUT_RAW heads against fp64 from the training forward's own h_7 tiles (fp16 operands), then the rgb
        # epilogue from those OUT_RAW values
        Wh, bh, cols9 = _heads_params(params[i * model.P:(i + 1) * model.P].cpu().numpy(), K, dev)
        Wh, bh = Wh.half().double(), bh.half().double()
        H = L.workspace_view(ws, lt, "H")
        for t0_ in range(0, lt["tiles"], CHUNK // L.TILE_M):
            t1_ = min(lt["tiles"], t0_ + CHUNK // L.TILE_M)
            r0, r1 = t0_ * L.TILE_M, min(M, t1_ * L.TILE_M)
            if r0 >= M:
                break
            h7 = L.decode_h(H[t0_:t1_], 7)[:r1 - r0].double()
            heads, mag = h7 @ Wh + bh, h7.abs() @ Wh.abs() + bh.abs()
            rr, rs = _raw_of_heads(heads, cols9)
            mr, ms = _raw_of_heads(mag, cols9)
            er = (raw_rgb[r0:r1].double() - rr).abs() / (U24 * mr)
            es = (raw_sig[r0:r1].double() - rs).abs() / (U24 * ms)
            st.max("raw_heads_excess", max(float(er.max()), float(es.max())))
            st.max("rgbs_from_raw_excess", _rgb_check(got[r0:r1, :3], raw_rgb[r0:r1].double(), mr, vd[r0:r1],
                                                      case.sh, FWD_ALLOW))
        out[f"MLP_{i}"] = dict(fp16=st.d, M=M)
    res["wall_s"] = time.time() - t0
    _record(case.name, {k: v for k, v in res.items()})
    for k, r in out.items():
        _record(f"{case.name}:{k}", r)
    if check_stages:
        _assert_stages({k: v for k, v in res.items() if k.startswith("MLP")})
    for k, r in out.items():
        s = r["fp16"]
        for key, val in s.items():
            if key.endswith("mismatches"):
                assert val == 0, (case.name, k, key, val)
        assert s["raw_heads_excess"] <= FWD_ALLOW, (case.name, k, s["raw_heads_excess"])
        assert s["rgbs_from_raw_excess"] <= 1.0, (case.name, k, s["rgbs_from_raw_excess"])


WIDE = Case(4, 40, 64, 128, 1000, sp_radius=5.0)   # the tt preset's sparsity_radius: sine arguments up to ~5 * 2^9


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES + [WIDE], ids=lambda c: c.name)
def test_fp16_forwards_bit_identical_to_training(case):
    """render (SRC_RAYS / OUT_RGBS), eval_points (OUT_RGBS), eval_points_raw (OUT_RAW, OUT_SIGMA) of the rows of one
    training call: bit-identical to the saving forward; OUT_RAW heads within FWD_ALLOW of fp64 from its h_7.  The wide
    case also runs the stage checks of test_train_stages on the training forward itself."""
    _fp16_vs_training(case, check_stages=case is WIDE)


@pytest.mark.gpu
def test_fp16_forwards_bit_identical_to_training_production_step():
    """the bench.py step: ~6 200 fine-level tiles, ~47 per CTA"""
    from plenoctree_b200._lib import RenderConfig, lib
    from plenoctree_b200.nerf.models import ctypes_ref
    cfg = RenderConfig(3, 64, 128, 1, 4096, 10000)
    need = int(lib.pob_workspace_bytes(ctypes_ref(cfg), 1)) + int(lib.pob_workspace_bytes(ctypes_ref(cfg), 0))
    free, _ = torch.cuda.mem_get_info()
    if free < need + (6 << 30):
        pytest.skip(f"the production step needs {need / 2**30:.1f} GB of workspaces + ~6 GB for the reference; "
                    f"{free / 2**30:.1f} GB free on this (shared) device")
    _fp16_vs_training(Case(3, 4096, 64, 128, 10000))


# =====================================================================================================================
# C: cell means against the fp64 mean of the same precision's OUT_RAW rows
# =====================================================================================================================
def _cell_bound(S):
    """the standard summation bound of the kernel's mean, as a multiple of 2^-24 * sum |v| / S: (n_adds + 1) roundings
    on any term's path, n_adds = 32 sequential fp32 adds per 32-row half-warpgroup + S/32 atomics of the scaled partials
    (S a multiple of 32) or S atomics (otherwise), + 1 for the product with fl(1/S); the first add onto zero is exact,
    which covers the rounding of fl(1/S).  gamma_n = n u / (1 - n u) makes it rigorous."""
    n = (32 + S // 32 if S % 32 == 0 else S) + 1
    return n / (1 - n * U24)


@pytest.mark.gpu
@pytest.mark.parametrize("sh", [-1, 3, 4])
@pytest.mark.parametrize("prec", ["fp16", "fp16x3"])
def test_cell_means_vs_fp64(sh, prec):
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    pr = ops.PREC_FP16 if prec == "fp16" else ops.PREC_FP16X3
    blob = _blob(O.init_flat_params(sh, 41, bias_scale=0.05), sh)
    sms = _sms()
    rep = {}
    for S in CELL_S:
        n_cells = 3 * sms * L.TILE_M // S + 3          # three or more tiles per CTA; cells straddle tiles
        rs = np.random.RandomState(S + 7 * (sh + 2))
        centers = rs.uniform(-1.4, 1.4, size=(n_cells, 1, 3))
        pts = torch.from_numpy((centers + rs.uniform(-0.05, 0.05, size=(n_cells, S, 3))).astype(np.float32)
                               .reshape(-1, 3)).cuda()
        got = _cells(blob, sh, pts, n_cells, S, pr)
        raw_rgb, raw_sig = _raw(blob, sh, pts, pr)
        vals = torch.cat([raw_rgb, raw_sig[:, None]], 1).double().view(n_cells, S, -1)
        ref = vals.mean(1)
        bound = _cell_bound(S) * U24 * vals.abs().sum(1) / S
        frac = float(((got.double() - ref).abs() / bound.clamp_min(1e-300)).max())
        rep[f"S{S}"] = dict(n_cells=n_cells, tiles=(n_cells * S + 127) // 128, err_over_bound=frac,
                            nonfinite=int((~torch.isfinite(got)).sum()))
    _record(f"cells_mean_sh{sh}_{prec}", rep)
    for k, r in rep.items():
        assert r["nonfinite"] == 0 and r["err_over_bound"] <= 1.0, (sh, prec, k, r)


# =====================================================================================================================
# D + E + F: fp16x3 against fp64, every SRC_POINTS mode; fp16 anchored to the training forward; ragged sizes, many
# tiles per CTA, canaries, determinism
# =====================================================================================================================
def _x3_sensitivity(ref, x):
    """per class: the largest move of the reference (heads, in units of 2^-24 * sum |h_7 w|) over X3_ALLOW"""
    heads, mag = ref(x)
    out = {}
    for c in SENS_CLASSES:
        hp, _ = ref(x, pert=c)
        out[c] = float(((hp - heads).abs() / (U24 * mag))[:, :1 + 3 * ref.K].max()) / X3_ALLOW
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("radius", [1.5, 5.0])
@pytest.mark.parametrize("sh", [-1, 0, 1, 2, 3, 4])
def test_point_forwards_shapes(sh, radius):
    from plenoctree_b200 import ops
    t0 = time.time()
    dev = torch.device("cuda")
    M = _m_many_tiles()
    K = L.K_of(sh)
    # fp16: the points ride as sparsity rows of one training call (one ray of three samples in front of them), so the
    # saving forward evaluates them too
    case = Case(sh, 1, 3, 0, M, seed=101 + sh, sp_radius=radius)
    model = case.model()
    state, ctx = case.run(model)
    ws = model.workspace(True)
    lv = L.train_workspace_views(model.cfg, 1, True)["levels"][0]
    rows = L.workspace_view(ws, lv, "rgbs")[3:].clone()
    x = torch.from_numpy(ctx["sp"]).to(dev)
    v0 = torch.from_numpy(ctx["rays"][2][:1]).to(dev)
    st = Stats()
    blob = model.blobs[0]
    vd0 = v0.expand(M, 3).contiguous()
    got16 = _rgbs(blob, sh, x, vd0, ops.PREC_FP16)
    raw16, sig16 = _raw(blob, sh, x, ops.PREC_FP16)
    _, sigo16 = _raw(blob, sh, x, ops.PREC_FP16, want_rgb=False)
    st.add("fp16_bit_mismatches", _nbits(got16, rows))
    st.add("fp16_bit_mismatches", int((sigo16.clamp_min(0) != rows[:, 3]).sum()) + _nbits(sigo16, sig16))
    Wh, bh, cols9 = _heads_params(model.params.cpu().numpy(), K, dev)
    Wh, bh = Wh.half().double(), bh.half().double()
    H = L.workspace_view(ws, lv, "H")
    for t0_ in range(0, lv["tiles"], CHUNK // L.TILE_M):
        t1_ = min(lv["tiles"], t0_ + CHUNK // L.TILE_M)
        h7 = L.decode_h(H[t0_:t1_], 7).double()
        r0 = t0_ * L.TILE_M
        keep = slice(max(0, 3 - r0), min(h7.shape[0], 3 + M - r0))      # sparsity rows only
        h7 = h7[keep]
        a = r0 + keep.start - 3
        heads, mag = h7 @ Wh + bh, h7.abs() @ Wh.abs() + bh.abs()
        rr, rs_ = _raw_of_heads(heads, cols9)
        mr, ms = _raw_of_heads(mag, cols9)
        b = a + h7.shape[0]
        st.max("fp16_raw_heads_excess", max(float(((raw16[a:b].double() - rr).abs() / (U24 * mr)).max()),
                                            float(((sig16[a:b].double() - rs_).abs() / (U24 * ms)).max())))
        st.max("fp16_rgbs_from_raw_excess", _rgb_check(got16[a:b, :3], raw16[a:b].double(), mr, vd0[a:b], sh,
                                                       FWD_ALLOW))

    # fp16x3 against fp64: OUT_RAW, OUT_SIGMA, OUT_RGBS at random view directions
    ref = X3Ref(model.params.cpu().numpy(), sh, dev)
    rs = np.random.RandomState(5 + sh)
    vd = rs.normal(size=(M, 3))
    vd = torch.from_numpy((vd / np.linalg.norm(vd, axis=1, keepdims=True)).astype(np.float32)).to(dev)
    raw3, sig3 = _raw(blob, sh, x, ops.PREC_FP16X3)
    _, sigo3 = _raw(blob, sh, x, ops.PREC_FP16X3, want_rgb=False)
    got3 = _rgbs(blob, sh, x, vd, ops.PREC_FP16X3)
    st.add("x3_sigma_only_vs_raw_bit_mismatches", _nbits(sigo3, sig3))
    st.add("x3_rgbs_sigma_relu_mismatches", int((sig3.clamp_min(0) != got3[:, 3]).sum()))
    _x3_errors(ref, x, raw3, sig3, st, "x3_points")
    for r0 in range(0, M, CHUNK):
        r1 = min(M, r0 + CHUNK)
        heads, mag = ref(x[r0:r1])
        mr = mag[:, cols9]
        st.max("x3_rgbs_from_raw_excess", _rgb_check(got3[r0:r1, :3], raw3[r0:r1].double(), mr, vd[r0:r1], sh,
                                                     X3_ALLOW))
    sens = _x3_sensitivity(ref, x[:4096])

    # determinism: a second launch of every non-atomic mode on the same inputs
    for pr, first in ((ops.PREC_FP16, (got16, raw16, sig16)), (ops.PREC_FP16X3, (got3, raw3, sig3))):
        again = (_rgbs(blob, sh, x, vd0 if pr == ops.PREC_FP16 else vd, pr),) + _raw(blob, sh, x, pr)
        st.add("rerun_bit_mismatches", sum(_nbits(a, b) for a, b in zip(again, first)))

    # ragged sizes: the first m rows of the many-tile launch, bit for bit, with canaries behind every output
    for m in M_RAGGED:
        for pr, (g, r, s), v in ((ops.PREC_FP16, (got16, raw16, sig16), vd0), (ops.PREC_FP16X3, (got3, raw3, sig3), vd)):
            rr_, ss_ = _raw(blob, sh, x[:m].contiguous(), pr)
            _, so_ = _raw(blob, sh, x[:m].contiguous(), pr, want_rgb=False)
            gg = _rgbs(blob, sh, x[:m].contiguous(), v[:m].contiguous(), pr)
            st.add("ragged_bit_mismatches", _nbits(rr_, r[:m]) + _nbits(ss_, s[:m]) + _nbits(so_, s[:m])
                   + _nbits(gg, g[:m]))
    rep = dict(M=M, tiles_per_cta=(M + 127) // 128 / _sms(), stats=st.d, x3_rel_to_max=_rel(st, "x3_points"),
               sensitivity_over_bar=sens, wall_s=time.time() - t0)
    _record(f"points_sh{sh}_r{radius:g}", rep)
    s = st.d
    for key, val in s.items():
        if key.endswith("mismatches"):
            assert val == 0, (key, val)
    assert s["fp16_raw_heads_excess"] <= FWD_ALLOW, s["fp16_raw_heads_excess"]
    assert s["fp16_rgbs_from_raw_excess"] <= 1.0, s["fp16_rgbs_from_raw_excess"]
    assert s["x3_points_excess"] <= X3_ALLOW, s["x3_points_excess"]
    assert s["x3_rgbs_from_raw_excess"] <= 1.0, s["x3_rgbs_from_raw_excess"]
    for c, ratio in sens.items():
        assert ratio >= (1.0 if c in X3_SENS_UNASSERTED else SENSITIVITY), (c, ratio)


@pytest.mark.gpu
@pytest.mark.parametrize("sh", [3, 4])
def test_grid_sweep_vs_points_and_fp64(sh):
    """eval_grid (SRC_GRID) bit-identical to eval_points_raw at the same fp32 coordinates, both precisions; a full-width
    slab and one with x0 > 0 and ny, nz not multiples of 128; fp16x3 against fp64"""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    dev = torch.device("cuda")
    flat = O.init_flat_params(sh, 31, bias_scale=0.05)
    blob = _blob(flat, sh)
    ref = X3Ref(flat, sh, dev)
    reso = 256
    radius = torch.tensor([1.5, 1.3, 1.1])
    center = torch.tensor([0.1, -0.2, 0.05])
    scale = 0.5 / radius
    offset = 0.5 * (1.0 - center / radius)
    arr = (torch.arange(0, reso, dtype=torch.float32) + 0.5) / reso
    st = Stats()
    for x0, nx, ny, nz in ((0, 2, 256, 256), (37, 3, 200, 129)):
        ax = [(arr - offset[a]) / scale[a] for a in range(3)]
        g = torch.stack(torch.meshgrid(ax[0][x0:x0 + nx], ax[1][:ny], ax[2][:nz], indexing="ij"))
        pts = g.reshape(3, -1).T.contiguous().to(dev)
        for pr in (ops.PREC_FP16, ops.PREC_FP16X3):
            rp, sp_ = _raw(blob, sh, pts, pr)
            rg, sg = _grid(blob, sh, reso, offset.tolist(), scale.tolist(), x0, nx, ny, nz, pr, True)
            _, so = _grid(blob, sh, reso, offset.tolist(), scale.tolist(), x0, nx, ny, nz, pr, False)
            _, so2 = _grid(blob, sh, reso, offset.tolist(), scale.tolist(), x0, nx, ny, nz, pr, False)
            st.add("grid_bit_mismatches", _nbits(rg, rp) + _nbits(sg, sp_) + _nbits(so, sp_) + _nbits(so2, so))
            if pr == ops.PREC_FP16X3:
                _x3_errors(ref, pts, rg, sg, st, "x3_grid")
    rep = dict(stats=st.d, x3_rel_to_max=_rel(st, "x3_grid"))
    _record(f"grid_sh{sh}", rep)
    assert st.d["grid_bit_mismatches"] == 0
    assert st.d["x3_grid_excess"] <= X3_ALLOW, st.d["x3_grid_excess"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", [Case(3, 96, 64, 128, 0), Case(-1, 40, 64, 128, 0), Case(4, 40, 64, 0, 0)],
                         ids=lambda c: c.name)
def test_x3_render_vs_points_and_composite(case):
    """the fp16x3 render (SRC_RAYS / OUT_RGBS): its workspace rgbs bit-identical to fp16x3 eval_points at o + z d, its
    comp / disp / acc / weights bit-identical to pob_composite of those rows, and the rows' OUT_RAW against fp64"""
    from plenoctree_b200 import ops
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    from plenoctree_b200.nerf.models import Rays
    dev = torch.device("cuda")
    model = case.model()
    n = case.R
    (o, d, v, _), t_rand, u, _, _ = case.inputs(n)
    rws = model.workspace(False)
    rws.fill_(0xFF)
    outs = model(Rays(o, d, v), randomized=True, t_rand=t_rand, u=u, precision=ops.PREC_FP16X3)
    torch.cuda.synchronize()
    rv = L.train_workspace_views(model.cfg, n, False, training=False)
    ctx = dict(rays=(o, d, v), n=n)
    dd = torch.from_numpy(d).to(dev)
    st = Stats()
    for i, lv in enumerate(rv["levels"]):
        z = L.workspace_view(rws, lv, "z")
        rows = L.workspace_view(rws, lv, "rgbs")
        x, vd = _level_rows(ctx, lv, z, None, dev)
        blob = model.blobs[i]
        got = _rgbs(blob, case.sh, x, vd, ops.PREC_FP16X3)
        st.add("x3_render_rgbs_bit_mismatches", _nbits(rows, got))
        comp = torch.empty(n, 3, device=dev)
        disp, acc = torch.empty(n, device=dev), torch.empty(n, device=dev)
        wts = torch.empty(n, lv["N"], device=dev)
        check(lib.pob_composite(ptr(got), ptr(z), ptr(dd), n, lv["N"], int(model.white_bkgd), ptr(comp), ptr(disp),
                                ptr(acc), ptr(wts), stream_ptr()))
        torch.cuda.synchronize()
        st.add("x3_render_composite_bit_mismatches",
               sum(_nbits(L.workspace_view(rws, lv, k), t) for k, t in
                   (("comp", comp), ("disp", disp), ("acc", acc), ("weights", wts)))
               + _nbits(outs[i][0].contiguous(), comp) + _nbits(outs[i][1].contiguous(), disp)
               + _nbits(outs[i][2].contiguous(), acc))
        raw3, sig3 = _raw(blob, case.sh, x, ops.PREC_FP16X3)
        st.add("x3_render_sigma_relu_mismatches", int((sig3.clamp_min(0) != rows[:, 3]).sum()))
        _x3_errors(X3Ref(model.params[i * model.P:(i + 1) * model.P].cpu().numpy(), case.sh, dev), x, raw3, sig3,
                   st, "x3_render")
    _record(f"x3_render_{case.name}", dict(stats=st.d, x3_rel_to_max=_rel(st, "x3_render")))
    for key, val in st.d.items():
        if key.endswith("mismatches"):
            assert val == 0, (key, val)
    assert st.d["x3_render_excess"] <= X3_ALLOW, st.d["x3_render_excess"]

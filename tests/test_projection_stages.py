"""The SH projection of a vanilla NeRF (projection.cu, pob_sh_proj_*) stage by stage against fp64.

tests/test_projection.py checks the chain at the reference defaults and small sizes.  Here each stage is held to an
fp64 evaluation of its own inputs, at the shapes and flags where the kernels branch:

  A  pob_sh_proj_points, from the workspace it fills (the saving relu forward at NH = 16 with SRC_POINTS): the posenc
     tile, h_0..h_7 and their relu mask words, raw sigma, and a_p = h7 head_w + head_b against an fp32 fma-chain
     bound, from one row to 9 tiles per CTA of 16 SMs, for five point encoders;
  B  pob_sh_proj_directions at fp32 arguments: Philox4x32-10 restated on the host (pinned by its published
     known-answer vectors), the directions within CUDA's ulp limits, t_d = W10_e posenc(d) from the fp32 arguments
     the reference forms (meaningful up to deg_view 32), the SH basis, and the grid / counter edges;
  C  pob_sh_proj_cells at every tile edge (a pairwise covering matrix of samples per leaf, directions, SH degree and
     leaves per block) and at production size, against fp64 rows built from the kernel's own a_p, sigma and tables;
  D  the device chain against the reference's model: the executed reference's golden (ref_projection.npz) and the
     fp64 oracle across encoders, deg_view, the view posenc order and the MLP choice.

Every workspace and output starts as 0xFF or a NaN canary.  Each check that compares against a reference also runs
against the reference of a plausible mistake (guard_*), which must miss its bar by GUARD.  The measured maxima go to
parity_projection_stages.json beside the other parity records (tests/test_train.py: OUT).
"""
import functools
import math
import os
import time

import numpy as np
import pytest
import torch

from oracle import nerf_sh_oracle as O
from oracle import posenc_oracle as PO
from oracle import projection_oracle as PJ
from plenoctree_b200 import layouts as L
from tests.support.mlp_stages import Stats
from tests.support.model_flags import CANARY, _canary, _points, _run_points
from tests.support.records import record

U = 2.0 ** -24
GUARD = 10.0
ENCODERS = ((0, 10, False), (0, 10, True), (2, 8, True), (0, 0, False), (9, 10, True))   # test_flag_matrix.ENCODERS

# ---- bars.  Measured on an H100 80 GB HBM3 at a 700 W power limit over every case of this file, the largest value in
# brackets.  a_p against fp64 h7 head_w + head_b from the saved fp16 h7 and the device's fp32 head: err / ((256 + 2) U
# sum |h w| + U |b|), the bound of a 256-term fp32 fma chain and the bias add
A_ALLOW = 1.0               # [0.021]
# directions: err / the bound composed from acosf, sinf, cosf (2 ulp each) and the fp32 products
DIR_ALLOW = 1.0             # [0.44]
# t_d: err / (2 ulp per sine feature + the (E + 1) U fma chain)
T_ALLOW = 1.0               # [0.58, deg_view 0..32]
# SH basis of the kernel's directions against fp64 of the same directions, absolute, in units of U
BASIS_ALLOW = 8.0           # [3.02]
# leaf rows: err / (the rows' fp32 rounding bound + the upstream stages' measured error carried forward)
ROWS_ALLOW = 1.0            # [0.25 on the kernel's own inputs; 0.18 against the executed reference, 0.15 the oracle]
# the executed reference's own fp32 rounding (test_projection.test_oracle_reproduces_the_executed_reference)
GOLDEN_REL = 1e-5


_record = functools.partial(record, "parity_projection_stages.json")


@pytest.fixture(scope="module", autouse=True)
def _file_wall_time():
    """the wall time of this file's tests, beside their measured maxima (GPU runs only)"""
    t0 = time.time()
    yield
    if torch.cuda.is_available():
        _record("wall_s", time.time() - t0)


def _ulp32(x):
    """fp32 ulp at |x| (numpy float64 array), the upper binade's at a power of two"""
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


# =====================================================================================================================
# Philox4x32-10 and the direction draws, restated on the host (common.cuh: philox4x32_10, u01; projection.cu:
# proj_direction)
# =====================================================================================================================
_M32 = np.uint64(0xFFFFFFFF)
PROJ_STREAM = 0x5348


def philox4x32_10(ctr, key):
    """ctr: four uint32-valued arrays (broadcast), key: two -> four uint32 arrays.  Per round: the products
    0xD2511F53 * c0 and 0xCD9E8D57 * c2 in 64 bits give (hi(p1) ^ c1 ^ k0, lo(p1), hi(p0) ^ c3 ^ k1, lo(p0)), then the
    key advances by the Weyl constants (0x9E3779B9, 0xBB67AE85)."""
    c = [np.asarray(x, np.uint64) & _M32 for x in ctr]
    k0, k1 = (np.asarray(x, np.uint64) & _M32 for x in key)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
    return [x.astype(np.uint32) for x in c]


def _uv(seed, blocks, D):
    """(u, v) float32 [n_blocks, D] of the direction draws: counter (d, block lo, block hi, 0x5348), key (seed lo,
    seed hi), 24 bits -> (x >> 8) 2^-24"""
    d = np.arange(D, dtype=np.uint64)[None, :]
    b = np.asarray(blocks, np.uint64)[:, None]
    seed = np.uint64(seed)
    r = philox4x32_10([d, b & _M32, b >> np.uint64(32), np.uint64(PROJ_STREAM)], [seed & _M32, seed >> np.uint64(32)])
    f = lambda x: (x >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)
    return f(r[0]), f(r[1])


def _dirs_ref(u, v, theta_pi=False):
    """fp64 directions at the kernel's fp32 arguments 2u - 1 and fp32(2 pi_f32 v), and the error bound of the kernel's
    fp32 evaluation: acosf, sinf, cosf within 2 ulp (CUDA's limits), each product rounded once"""
    xc = (np.float32(2.0) * u - np.float32(1.0)).astype(np.float64)             # exact
    phi = (np.float32(6.2831854820251465) * v).astype(np.float64)              # the fp32 product
    theta = np.pi * u.astype(np.float64) if theta_pi else np.arccos(xc)
    dth = 2 * _ulp32(theta)
    st, ct, sp, cp = np.sin(theta), np.cos(theta), np.sin(phi), np.cos(phi)
    ds = dth * (np.abs(ct) + dth) + 2 * _ulp32(np.abs(st) + dth)                # sinf(acosf(.))
    dz = dth * (np.abs(st) + dth) + 2 * _ulp32(np.abs(ct) + dth)                # cosf(acosf(.))
    dcp, dsp = 2 * _ulp32(cp), 2 * _ulp32(sp)
    ref = np.stack([st * cp, st * sp, ct], -1)
    bx = np.abs(cp) * ds + (np.abs(st) + ds) * dcp
    by = np.abs(sp) * ds + (np.abs(st) + ds) * dsp
    bnd = np.stack([bx + _ulp32(np.abs(st * cp) + bx), by + _ulp32(np.abs(st * sp) + by), dz], -1)
    return ref, bnd


def _view_features(d32, deg_view, legacy, swap_sc=False):
    """posenc(d, 0, deg_view, legacy) as the kernel evaluates it: fp64 sines of the fp32 arguments d_c 2^l (exact) and
    fp32(d_c 2^l + fp32(pi / 2)); and each feature's error allowance (2 ulp of a sine, 0 for d itself).  d32: float32
    [n, 3] -> ([n, E], [n, E]) fp64.  swap_sc: sine and cosine exchanged (a guard)."""
    cols, ulps = [], []
    for kind, j, c in PO.feature_index((0, deg_view, legacy)):
        if kind == "x":
            cols.append(d32[:, c].astype(np.float64))
            ulps.append(np.zeros(d32.shape[0]))
            continue
        arg = d32[:, c] * np.float32(2.0 ** j)
        if (kind == "cos") != swap_sc:
            arg = (arg + np.float32(np.pi / 2)).astype(np.float32)
        f = np.sin(arg.astype(np.float64))
        cols.append(f)
        ulps.append(2 * _ulp32(f))
    return np.stack(cols, 1), np.stack(ulps, 1)


def _t_ref(d32, w10e, deg_view, legacy, swap_sc=False):
    """fp64 t_d [128, n] of the kernel's fp32 feature arguments and its bound [128, n]"""
    f, fu = _view_features(d32, deg_view, legacy, swap_sc)
    w = np.asarray(w10e, np.float64)
    E = f.shape[1]
    return (f @ w).T, (fu @ np.abs(w) + (E + 1) * U * (np.abs(f) @ np.abs(w))).T


# =====================================================================================================================
# CPU
# =====================================================================================================================
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))], ids=["zeros", "ones", "pi"])
def test_host_philox_known_answers(ctr, key, want):
    """the host restatement of common.cuh's round structure reproduces Philox4x32-10's published known answers"""
    got = philox4x32_10([np.uint64(c) for c in ctr], [np.uint64(k) for k in key])
    assert tuple(int(x) for x in got) == want


def test_host_philox_round_structure_is_the_kernels():
    """the constants and the output permutation restated above are the ones projection.cu's draws run"""
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    common = open(os.path.join(ROOT, "plenoctree_b200", "csrc", "common.cuh")).read()
    for s in ("__umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x",
              "__umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z",
              "ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);",
              "key.x += 0x9E3779B9u;", "key.y += 0xBB67AE85u;", "for (int r = 0; r < 10; ++r)",
              "return float(x >> 8) * (1.0f / 16777216.0f);"):
        assert s in common, s
    proj = open(os.path.join(ROOT, "plenoctree_b200", "csrc", "projection.cu")).read()
    assert f"PROJ_STREAM = 0x{PROJ_STREAM:x}u" in proj
    assert ("make_uint4(uint32_t(d), uint32_t(blk), uint32_t(blk >> 32), PROJ_STREAM),\n"
            "                                make_uint2(uint32_t(seed), uint32_t(seed >> 32))") in proj


def test_host_directions_bound_is_tight_and_guards_separate():
    """the direction bound is a few fp32 ulps, and the guard references (theta = pi u, u and v swapped) sit far
    outside it on the host's own fp32 evaluation of the reference formula"""
    u, v = _uv(7, [0, 1, 2 ** 32 - 1, 2 ** 32], 4096)
    ref, bnd = _dirs_ref(u, v)
    assert float(bnd.max()) < 64 * U
    xc = np.float32(2.0) * u - np.float32(1.0)
    th = np.arccos(xc).astype(np.float32)
    ph = np.float32(6.2831854820251465) * v
    s = np.sin(th).astype(np.float32)
    got = np.stack([s * np.cos(ph).astype(np.float32), s * np.sin(ph).astype(np.float32),
                    np.cos(th).astype(np.float32)], -1).astype(np.float64)
    assert float((np.abs(got - ref) / bnd).max()) <= 1.0
    for alt in (_dirs_ref(u, v, theta_pi=True), _dirs_ref(v, u)):
        assert float((np.abs(got - alt[0]) / bnd).max()) >= GUARD * DIR_ALLOW


def test_point_workspace_mirror_matches_library():
    """the byte layout decoded below (projection.cu: point_ws): h images [tiles, 8, 64 KB], posenc images
    [tiles, 16 KB], then relu mask words [8, rows, 8]"""
    from plenoctree_b200._lib import lib
    for m in (0, 1, 127, 128, 511, 512, 513, 3000, 9 * 16 * 128 + 77):
        assert int(lib.pob_sh_proj_points_workspace_bytes(m)) == _point_ws(m)["total"], m


def _point_ws(m):
    rows = L.padded_rows(m)
    tiles = rows // L.TILE_M
    e = tiles * L.NUM_TRUNK * L.A_TILE_BYTES
    mask = e + tiles * L.E_TILE_BYTES
    return dict(rows=rows, tiles=tiles, h=0, e=e, mask=mask, total=mask + L.NUM_TRUNK * rows * 8 * 4)


# ---- C: the covering matrix of the leaf-row kernel ------------------------------------------------------------------
C_S = (1, 2, 7, 8, 9, 32, 33, 63, 64, 65, 128, 129, 256)
C_D = (1, 63, 64, 65, 100, 10000)
C_SH = (0, 1, 2, 3, 4)
C_CPB = ("1", "G-1", "G", "G+1", "1024")       # leaves per direction block, G = leaves per CTA = max(1, 64 // S)
C_DIMS = (C_S, C_D, C_SH, C_CPB)


def _cpb(S, label):
    G = max(1, 64 // S)
    return {"1": 1, "G-1": max(1, G - 1), "G": G, "G+1": G + 1, "1024": 1024}[label]


# row (i, j) of S_i x D_j takes SH degree (i + j) mod 5 and block size (i + 2 j) mod 5: (i, j) -> (i + j, i + 2 j) is
# invertible mod 5, so with >= 5 values of i and j every pair of the last two dimensions appears too
C_MATRIX = [(S, D, C_SH[(i + j) % 5], C_CPB[(i + 2 * j) % 5]) for i, S in enumerate(C_S) for j, D in enumerate(C_D)]
# named: 64 leaves in a CTA at SH25 (4800 outputs: all 19 accumulators per thread live), and 32 leaves (2400)
C_NAMED = [(1, 10000, 4, "1024"), (2, 10000, 4, "G")]


def _n_cells(S, D, sh, label):
    """two direction blocks, the second ragged (a block of one leaf cannot be)"""
    cpb = _cpb(S, label)
    if cpb == 1:
        return 3
    return cpb + 1 + (7 * S + 3 * D + sh) % min(cpb - 1, 97)


def _c_tag(row):
    S, D, sh, label = row
    return f"S{S}_D{D}_sh{sh}_cpb{label}"


def test_cells_matrix_covers_every_pair():
    """every pair of values of any two dimensions appears in some row; every row's leaf count is not a multiple of
    its block size (but for blocks of one leaf); the named rows fill a CTA with 64 and 32 leaves at SH25"""
    from itertools import combinations
    rows = C_MATRIX + C_NAMED
    for row in rows:
        for v, dim in zip(row, C_DIMS):
            assert v in dim, (row, v)
        cpb = _cpb(row[0], row[3])
        assert cpb == 1 or _n_cells(*row) % cpb != 0, row
    missing = []
    for i, j in combinations(range(len(C_DIMS)), 2):
        seen = {(r[i], r[j]) for r in rows}
        missing += [(i, a, j, b) for a in C_DIMS[i] for b in C_DIMS[j] if (a, b) not in seen]
    assert not missing, missing
    ACC_PER_THREAD = (64 * 3 * 25 + 255) // 256
    for S, D, sh, label in C_NAMED:
        G = max(1, 64 // S)
        assert sh == 4 and min(G, _cpb(S, label)) == 64 // S
    assert ACC_PER_THREAD == 19 and 64 * 75 > 18 * 256 and 32 * 75 == 2400


# =====================================================================================================================
# GPU helpers
# =====================================================================================================================


def _tail_ok(buf, shape):
    return bool((buf[int(np.prod(shape)):] == CANARY).all())


def _mlps(seed, pe, deg_view):
    return {"MLP_0": PJ.init_params(seed, pe, deg_view), "MLP_1": PJ.init_params(seed + 1, pe, deg_view)}


def _sigma_flat(layers):
    """the plain-RGB (sh_deg -1) flat parameters of VanillaNerf's sigma blob: the trunk, Dense_8, zero rgb columns"""
    return np.concatenate([np.asarray(a, np.float32).reshape(-1) for k, b in layers[:9] for a in (k, b)] +
                          [np.zeros(256 * 3 + 3, np.float32)])


def _ws_views(ws, m):
    g = _point_ws(m)
    H = ws[:g["e"]].view(g["tiles"], L.NUM_TRUNK, L.A_TILE_BYTES)
    E = ws[g["e"]:g["mask"]].view(g["tiles"], L.E_TILE_BYTES)
    MASK = ws[g["mask"]:g["total"]].view(torch.int32).view(L.NUM_TRUNK, g["rows"], 8)
    return H, E, MASK


def _alt_pe(pe):
    from tests.support.model_flags import _alt_pe as alt
    return alt(pe)


def _check_points(nerf, layers, pe, pts, ws, a, sig, st):
    """A: every stage of one pob_sh_proj_points call against fp64 of the kernel's own previous stage"""
    from tests.support.model_flags import _ref_features
    from tests.support.mlp_stages import FP16, FWD_ALLOW, _sin_excess, excess
    dev = pts.device
    m = pts.shape[0]
    EW = PO.width(pe)
    flat = _sigma_flat(layers)
    w_off, b_off, _ = L.flat_offsets(1, EW)
    dims = L.layer_dims(1, EW)
    fl = torch.from_numpy(flat).to(dev)
    W = [fl[w_off[l]:w_off[l] + dims[l][0] * 256].view(dims[l][0], 256).half().double() for l in range(8)]
    B = [fl[b_off[l]:b_off[l] + 256].half().double() for l in range(8)]
    Wh_np, bh_np = L.heads_matrix(flat, 1, EW)
    Wh, bh = (torch.from_numpy(x).to(dev).half().double() for x in (Wh_np, bh_np))
    H, E, MASK = _ws_views(ws, m)
    rows = H.shape[0] * L.TILE_M
    s = torch.arange(rows, device=dev)
    real = s < m
    x = pts[s.clamp_max(m - 1)]                 # load_point clamps the row: padded rows repeat row m - 1
    bits = lambda t: t.view(torch.int16)
    # ---- posenc tile
    e16 = L.decode_e(E)
    st.add("posenc_xyz_bit_mismatches", int((bits(e16[:, :3]) != bits(x.half())).sum()))
    st.add("posenc_pad_nonzero_bits", int((bits(e16[:, EW:63]) != 0).sum()))
    st.add("posenc_col63_not_one", int((e16[:, 63] != 1).sum()))
    if EW > 3:
        st.max("posenc_sin_excess", _sin_excess(e16[:, 3:EW], torch.zeros_like(e16[:, 3:EW]), _ref_features(x, pe),
                                                False))
    eW = e16[:, :EW].double()
    alt = _alt_pe(pe)
    eW_alt = torch.cat([x.half().double(), _ref_features(x, alt).half().double()], 1) if alt is not None else None
    # ---- h_0..h_7 and their mask words
    h16 = [L.decode_h(H, l) for l in range(8)]
    hd = [h.double() for h in h16]
    guard = 0.0
    for l in range(8):
        inp = eW if l == 0 else (torch.cat([hd[4], eW], 1) if l == 5 else hd[l - 1])
        pre = inp @ W[l] + B[l]
        st.max("fwd_excess", excess(h16[l], torch.zeros_like(h16[l]), pre.clamp_min(0),
                                     inp.abs() @ W[l].abs() + B[l].abs(), False))
        if eW_alt is not None and l in (0, 5):
            ia = eW_alt if l == 0 else torch.cat([hd[4], eW_alt], 1)
            guard = max(guard, excess(h16[l], torch.zeros_like(h16[l]), (ia @ W[l] + B[l]).clamp_min(0),
                                      ia.abs() @ W[l].abs() + B[l].abs(), False) / FWD_ALLOW[FP16])
        st.add("h_nonfinite", int((~torch.isfinite(h16[l])).sum()))
        want = torch.from_numpy(L.encode_mask_reference(h16[l].cpu().numpy()).view(np.int32)).to(dev)
        st.add("mask_word_mismatches", int((MASK[l] != want).sum()))
    if eW_alt is not None:
        st.min("guard_fwd_alt_pe", guard)
    # ---- raw sigma: the heads GEMM's column 0, at the training checks' heads bar
    heads = hd[7] @ Wh[:, 0] + bh[0]
    hmag = hd[7].abs() @ Wh[:, 0].abs() + bh[0].abs()
    st.max("sigma_excess", float(((sig.double() - heads[:m]).abs() / (FWD_ALLOW[FP16] * U * hmag[:m])).max()))
    # ---- a_p: the fp32 fma chain over h7 and the device's head
    hw, hb = nerf.head_w.double(), nerf.head_b.double()

    def a_ratio(h):
        ref = h[:m] @ hw + hb
        bnd = (256 + 2) * U * (h[:m].abs() @ hw.abs()) + U * hb.abs()
        return float(((a.double() - ref).abs() / bnd.clamp_min(1e-300)).max())

    st.max("a_excess", a_ratio(hd[7]) / A_ALLOW)
    st.min("guard_a_from_h6", a_ratio(hd[6]) / A_ALLOW)
    st.add("a_nonfinite", int((~torch.isfinite(a)).sum()))


def _head_half_ulp(nerf, layers):
    """head_w / head_b on the device are the fp64 W9 W10_b and b9 W10_b + b10 rounded once: within half an fp32 ulp"""
    k9, b9 = (np.asarray(x, np.float64) for x in layers[9])
    k10, b10 = (np.asarray(x, np.float64) for x in layers[10])
    worst = 0.0
    for got, ref in ((nerf.head_w, k9 @ k10[:256]), (nerf.head_b, b9 @ k10[:256] + b10)):
        err = np.abs(got.cpu().numpy().astype(np.float64) - ref)
        worst = max(worst, float((err / (0.5 * _ulp32(ref))).max()))
    return worst


# =====================================================================================================================
# A. the point stage from its own saved tiles
# =====================================================================================================================
A_SIZES = (1, 127, 128, 129, 511, 512, 513, 3000, 9 * 16 * 128 + 77)


@pytest.mark.gpu
@pytest.mark.parametrize("pe", ENCODERS, ids=lambda pe: f"{pe[0]}_{pe[1]}_{'legacy' if pe[2] else 'std'}")
def test_point_stage_from_saved_tiles(pe, monkeypatch):
    """posenc tile, h_0..h_7, mask words, raw sigma and a_p of pob_sh_proj_points against fp64 of the kernel's own
    previous stage, at ragged and tile-edge sizes; the last size at 16 SMs (9 tiles per CTA: every ring phase)"""
    from plenoctree_b200.octree.projection import VanillaNerf
    from tests.support.model_flags import _set_sms
    from tests.support.mlp_stages import FP16, FWD_ALLOW
    t0 = time.time()
    layers = PJ.init_params(41, pe, 4)
    nerf = VanillaNerf({"MLP_0": layers}, pe, 4, num_fine_samples=0)
    st = Stats()
    st.max("head_err_over_half_ulp", _head_half_ulp(nerf, layers))
    for i, m in enumerate(A_SIZES):
        if m == A_SIZES[-1]:
            _set_sms(monkeypatch, 16)
        pts = _points(m, 100 + i)
        ws, a, sig, ab, sb = _run_points(nerf, pts)
        st.add("rows_past_m_written", int(not _tail_ok(ab, (m, 128))) + int(not _tail_ok(sb, (m,))))
        _check_points(nerf, layers, pe, pts, ws, a, sig, st)
    d = st.d
    _record(f"A/{pe[0]}_{pe[1]}_{int(pe[2])}", dict(stages=d, wall_s=time.time() - t0))
    for k in ("posenc_xyz_bit_mismatches", "posenc_pad_nonzero_bits", "posenc_col63_not_one", "h_nonfinite",
              "mask_word_mismatches", "a_nonfinite", "rows_past_m_written"):
        assert d[k] == 0, (k, d)
    assert d["head_err_over_half_ulp"] <= 1.0, d
    assert d.get("posenc_sin_excess", 0.0) <= 1.0, d
    assert d["fwd_excess"] <= FWD_ALLOW[FP16], d
    assert d["sigma_excess"] <= 1.0, d
    assert d["a_excess"] <= 1.0, d
    assert d["guard_a_from_h6"] >= GUARD, d
    if _alt_pe(pe) is not None:
        assert d["guard_fwd_alt_pe"] >= GUARD, d


# =====================================================================================================================
# B. direction tables at fp32 arguments
# =====================================================================================================================
def _tables(nerf, sh_deg, D, block0, n_blocks, seed):
    """pob_sh_proj_directions into canary buffers -> ((dirs, t, basis), tails intact)"""
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    K = (sh_deg + 1) ** 2
    shapes = ((n_blocks, D, 3), (n_blocks, 128, D), (n_blocks, D, K))
    bufs = [_canary(s) for s in shapes]
    dirs, t, basis = (v for _, v in bufs)
    check(lib.pob_sh_proj_directions(int(seed), int(block0), int(n_blocks), int(D), nerf.deg_view,
                                     int(bool(nerf.posenc[2])), int(sh_deg), ptr(nerf.w10e), ptr(dirs), ptr(t),
                                     ptr(basis), stream_ptr()))
    torch.cuda.synchronize()
    return (dirs, t, basis), all(_tail_ok(b, s) for (b, _), s in zip(bufs, shapes))


def _check_tables(nerf, tables, seed, block0, sh_deg, st, guards=True):
    dirs, t, basis = tables
    nb, D = dirs.shape[:2]
    dv, legacy = nerf.deg_view, bool(nerf.posenc[2])
    u, v = _uv(seed, np.arange(block0, block0 + nb, dtype=np.uint64), D)
    got = dirs.cpu().numpy().astype(np.float64)
    ref, bnd = _dirs_ref(u, v)
    st.max("dirs_excess", float((np.abs(got - ref) / bnd).max()) / DIR_ALLOW)
    if guards:
        for name, alt in (("theta_pi_u", _dirs_ref(u, v, theta_pi=True)), ("u_v_swapped", _dirs_ref(v, u))):
            st.min(f"guard_dirs_{name}", float((np.abs(got - alt[0]) / bnd).max()) / DIR_ALLOW)
    d32 = dirs.cpu().numpy().reshape(-1, 3)
    w = nerf.w10e.cpu().numpy()
    tr, tb = _t_ref(d32, w, dv, legacy)
    tg = t.cpu().numpy().astype(np.float64).transpose(1, 0, 2).reshape(128, -1)
    st.max("t_excess", float((np.abs(tg - tr) / np.maximum(tb, 1e-300)).max()) / T_ALLOW)
    if guards and dv > 0:
        st.min("guard_t_sin_cos_swapped",
               float((np.abs(tg - _t_ref(d32, w, dv, legacy, swap_sc=True)[0]) / tb).max()) / T_ALLOW)
        if dv > 1:
            st.min("guard_t_other_order",
                   float((np.abs(tg - _t_ref(d32, w, dv, not legacy)[0]) / tb).max()) / T_ALLOW)
    Y = O.sh_basis(sh_deg, dirs.reshape(-1, 3).double()).reshape(basis.shape)
    st.max("basis_err_units_u", float((basis.double() - Y).abs().max()) / U)
    st.add("nonfinite", int((~torch.isfinite(dirs)).sum() + (~torch.isfinite(t)).sum() + (~torch.isfinite(basis)).sum()))


def _assert_tables(d, guards=True):
    assert d["nonfinite"] == 0 and d.get("tails_written", 0) == 0, d
    assert d["dirs_excess"] <= 1.0 and d["t_excess"] <= 1.0, d
    assert d["basis_err_units_u"] <= BASIS_ALLOW, d
    if guards:
        for k, val in d.items():
            if k.startswith("guard_"):
                assert val >= GUARD, (k, d)


def _dir_model(deg_view, legacy, seed=14):
    from plenoctree_b200.octree.projection import VanillaNerf
    return VanillaNerf(_mlps(seed, (0, 10, legacy), deg_view), (0, 10, legacy), deg_view, num_fine_samples=0)


@pytest.mark.gpu
@pytest.mark.parametrize("legacy", [False, True], ids=["std", "legacy"])
@pytest.mark.parametrize("deg_view", [0, 1, 2, 4, 9, 10, 16, 23, 24, 31, 32])
def test_direction_tables_at_fp32_arguments(deg_view, legacy):
    """directions against the host Philox and fp64 at the kernel's fp32 arguments, t_d against fp64 sines of the
    fp32 posenc arguments the reference forms, the SH basis (sh_deg 0..4) against fp64 of the kernel's directions"""
    nerf = _dir_model(deg_view, legacy)
    st = Stats()
    for sh in range(5):
        tables, ok = _tables(nerf, sh, 300, 3 + sh, 2, seed=5 + sh)
        st.add("tails_written", int(not ok))
        _check_tables(nerf, tables, 5 + sh, 3 + sh, sh, st)
    _record(f"B/deg_view{deg_view}_{'legacy' if legacy else 'std'}", st.d)
    _assert_tables(st.d)


@pytest.mark.gpu
def test_direction_table_edges():
    """n_dirs at the 32-direction CTA edges and 10 000, 65 535 blocks of one direction, block indices across the
    counter's high word; a block's directions do not depend on the call it is drawn in; uniform on the sphere"""
    nerf = _dir_model(4, False)
    st = Stats()
    for D in (1, 31, 32, 33, 10000):
        tables, ok = _tables(nerf, 4, D, 11, 2, seed=21)
        st.add("tails_written", int(not ok))
        _check_tables(nerf, tables, 21, 11, 4, st, guards=D >= 32)
    tables, ok = _tables(nerf, 2, 1, 0, 65535, seed=22)
    st.add("tails_written", int(not ok))
    _check_tables(nerf, tables, 22, 0, 2, st, guards=False)
    big = {}
    for b0 in (2 ** 32 - 1, 2 ** 32):
        big[b0], ok = _tables(nerf, 4, 300, b0, 2, seed=23)
        st.add("tails_written", int(not ok))
        _check_tables(nerf, big[b0], 23, b0, 4, st)
    for k, v in zip(big[2 ** 32 - 1], big[2 ** 32]):
        st.add("split_call_mismatches", int((k[1] != v[0]).sum()))
    assert not torch.equal(big[2 ** 32][0][0], big[2 ** 32][0][1])
    # the high word is drawn from: block 2^32 is not block 0
    low, _ = _tables(nerf, 4, 300, 0, 1, seed=23)
    assert not torch.equal(low[0][0], big[2 ** 32][0][0])
    _record("B/edges", st.d)
    _assert_tables(st.d)
    assert st.d["split_call_mismatches"] == 0, st.d
    # uniform on the sphere: the mean direction of 20 000 draws within 4 standard deviations of 0
    d = big[2 ** 32 - 1][0].reshape(-1, 3).double()
    assert float(d.mean(0).abs().max()) < 4 / math.sqrt(3 * d.shape[0])


# =====================================================================================================================
# C. leaf rows
# =====================================================================================================================
def _rows64(a, sigma, t, Y, w11, b11, S):
    """fp64 leaf rows [n, 3K + 1] from a_p [n S, 128], raw sigma [n S], the tables t [128, D] and Y [D, K] as given
    (the kernel's own), and the bound of pob_sh_proj_cells' fp32 evaluation: fl(a + t), the 128-term rgb fma chain
    and its bias add, then the sums over the leaf's points, the 64-direction tile chains and the tile accumulation"""
    dev = a.device
    D, K = Y.shape
    n = a.shape[0] // S
    td, Yd = t.double(), Y.double()
    w, b = w11.double(), b11.double()
    wa = w.abs()
    g = (128 + 4) * U
    sumf = (S + 70 + (D // 64 + 1) * (S // 64 + 2)) * U
    c = torch.zeros(n * S, 3, K, dtype=torch.float64, device=dev)
    cb = torch.zeros_like(c)
    step = max(1, (1 << 20) // D)
    for i in range(0, n * S, step):
        ai = a[i:i + step].double()
        x = ai[:, None, :] + td.T[None]                      # [p, D, 128]
        rgb = torch.relu(x) @ w + b                          # [p, D, 3]
        rb = g * (x.abs() @ wa + b.abs())
        c[i:i + step] = torch.einsum("pdc,dk->pck", rgb, Yd)
        cb[i:i + step] = torch.einsum("pdc,dk->pck", rb + sumf * (rgb.abs() + rb), Yd.abs())
    sc = 4 * math.pi / D
    c = c.reshape(n, S, 3 * K).mean(1) * sc
    cb = cb.reshape(n, S, 3 * K).mean(1) * sc
    s = sigma.double().reshape(n, S)
    return (torch.cat([c, s.mean(1)[:, None]], 1),
            torch.cat([cb, ((S + 2) * U * s.abs().mean(1))[:, None]], 1))


def _cells(nerf, a, sig, S, sh, tables, cpb, n_cells):
    """pob_sh_proj_cells into a canary output -> (rows, tail intact)"""
    from plenoctree_b200.octree import projection as P
    K = (sh + 1) ** 2
    ob, out = _canary((n_cells, 3 * K + 1))
    P.project_cells(nerf, a, sig, S, sh, tables, cells_per_block=cpb, out=out)
    torch.cuda.synchronize()
    return out, _tail_ok(ob, (n_cells, 3 * K + 1))


def _leaf_sample(n_cells, cpb, G, S, D, rs, n_rand=8):
    """leaves checked against fp64: all when small, else the first and last CTA of every block (every accumulator
    slot) and some at random"""
    if n_cells * S * D <= 4_000_000:
        return np.arange(n_cells)
    pick = set()
    for b0 in range(0, n_cells, cpb):
        b1 = min(n_cells, b0 + cpb)
        last0 = b0 + (b1 - b0 - 1) // G * G
        pick |= set(range(b0, min(b1, b0 + G))) | set(range(last0, b1))
    pick |= set(rs.randint(0, n_cells, n_rand).tolist())
    return np.array(sorted(pick))


def _check_rows(out, nerf, a, sig, S, sh, tables, cpb, leaves, st):
    dirs, t, basis = tables
    G = max(1, 64 // S)
    for b in sorted(set((leaves // cpb).tolist())):
        lv = torch.from_numpy(leaves[leaves // cpb == b]).to(a.device)
        idx = (lv[:, None] * S + torch.arange(S, device=a.device)[None]).reshape(-1)
        ref, bnd = _rows64(a[idx], sig[idx], t[b], basis[b], nerf.w11, nerf.b11, S)
        err = (out[lv].double() - ref).abs()
        st.max("rows_excess", float((err / bnd.clamp_min(1e-300)).max()) / ROWS_ALLOW)
    st.add("rows_nonfinite", int((~torch.isfinite(out)).sum()))
    st.max("leaves_per_cta", min(G, cpb))


_C_MODEL = {}


def _c_model():
    from plenoctree_b200.octree.projection import VanillaNerf
    if not _C_MODEL:
        _C_MODEL["m"] = VanillaNerf(_mlps(13, (0, 10, False), 4), (0, 10, False), 4, num_fine_samples=128)
    return _C_MODEL["m"]


@pytest.mark.gpu
@pytest.mark.parametrize("row", C_MATRIX + C_NAMED, ids=_c_tag)
def test_leaf_rows_against_fp64(row):
    S, D, sh, label = row
    cpb = _cpb(S, label)
    n_cells = _n_cells(*row)
    nerf = _c_model()
    pts = _points(n_cells * S, seed=S * 31 + D)
    n_blk = (n_cells + cpb - 1) // cpb
    tables, ok = _tables(nerf, sh, D, 9, n_blk, seed=77)
    a, sig = nerf.point_stage(pts)
    out, tail = _cells(nerf, a, sig, S, sh, tables, cpb, n_cells)
    st = Stats()
    st.add("tails_written", int(not ok) + int(not tail))
    leaves = _leaf_sample(n_cells, cpb, max(1, 64 // S), S, D, np.random.RandomState(S + D))
    _check_rows(out, nerf, a, sig, S, sh, tables, cpb, leaves, st)
    st.max("leaves_checked", len(leaves))
    _record(f"C/{_c_tag(row)}", st.d)
    assert st.d["tails_written"] == 0 and st.d["rows_nonfinite"] == 0, st.d
    assert st.d["rows_excess"] <= 1.0, st.d


@pytest.mark.gpu
def test_production_launch():
    """one project_leaves call of blocks_per_launch(8, 10000, 4) blocks of 1024 leaves (262 144 points): first, last
    and 16 random leaves of every block against fp64, every row finite, the sigma column of every leaf; the same
    leaves in two launches split at a block boundary give bit-identical rows"""
    from plenoctree_b200.octree import projection as P
    t0 = time.time()
    S, D, sh, cpb = 8, 10000, 4, P.CELLS_PER_BLOCK
    nb = P.blocks_per_launch(S, D, sh)
    assert nb == 32
    nerf = _c_model()
    n_cells = nb * cpb
    pts = _points(n_cells * S, seed=8).reshape(n_cells, S, 3)
    b0 = 5
    out = P.project_leaves(nerf, sh, D, pts, S, b0)
    torch.cuda.synchronize()
    st = Stats()
    st.add("rows_nonfinite", int((~torch.isfinite(out)).sum()))
    a, sig = nerf.point_stage(pts.reshape(-1, 3))
    tables, ok = _tables(nerf, sh, D, b0, nb, seed=P.PROJ_SEED)
    st.add("tails_written", int(not ok))
    rs = np.random.RandomState(3)
    leaves = np.concatenate([np.unique(np.concatenate([[b * cpb, b * cpb + cpb - 1], b * cpb + rs.randint(0, cpb, 16)]))
                             for b in range(nb)])
    _check_rows(out, nerf, a, sig, S, sh, tables, cpb, leaves, st)
    s64 = sig.double().reshape(n_cells, S)
    st.max("sigma_col_excess", float(((out[:, -1].double() - s64.mean(1)).abs() /
                                      ((S + 2) * U * s64.abs().mean(1)).clamp_min(1e-300)).max()))
    h = nb // 2 * cpb
    o1 = P.project_leaves(nerf, sh, D, pts[:h], S, b0)
    o2 = P.project_leaves(nerf, sh, D, pts[h:], S, b0 + nb // 2)
    torch.cuda.synchronize()
    st.add("split_launch_bit_mismatches", int((torch.cat([o1, o2]).view(torch.int32) != out.view(torch.int32)).sum()))
    st.max("wall_s", time.time() - t0)
    _record("C/production", st.d)
    d = st.d
    assert d["rows_nonfinite"] == 0 and d["tails_written"] == 0 and d["split_launch_bit_mismatches"] == 0, d
    assert d["rows_excess"] <= 1.0 and d["sigma_col_excess"] <= 1.0, d


# =====================================================================================================================
# D. the device chain against the reference's model
# =====================================================================================================================
def _carried(da, dt, dY, a, t, Y, w11, b11, S):
    """the upstream stages' measured error carried to the leaf rows: relu is 1-Lipschitz, so an error da in a_p and dt
    in t_d moves raw rgb by at most sum_j |W11_jc| (|da_j| + |dt_j|), and an error dY in the basis moves a coefficient
    by sum_d |dY_dk| |rgb_dc|.  All [.., n S] -> [n, 3K] (4 pi / D, mean over the leaf's points)"""
    wa, ba = w11.double().abs(), b11.double().abs()
    D, K = Y.shape
    Ya, dYs = Y.double().abs(), dY.double()
    pa = da.double() @ wa                                    # [P, 3]
    at = (a.double().abs() @ wa + ba)                        # [P, 3]
    td = dt.double().T @ wa                                  # [D, 3]
    tt = t.double().abs().T @ wa                             # [D, 3]
    c = pa[:, :, None] * Ya.sum(0)[None, None] + (td.T @ Ya)[None] \
        + at[:, :, None] * dYs.sum(0)[None, None] + (tt.T @ dYs)[None]
    n = da.shape[0] // S
    return c.reshape(n, S, 3 * K).mean(1) * (4 * math.pi / D)


def _perm_view(layers, deg_view, legacy):
    """the layers with W10_e's rows reordered so that the correct-order posenc meets the rows of the other order: the
    view branch of a model that encodes directions in the other feature order"""
    fi = PO.feature_index((0, deg_view, legacy))
    fo = PO.feature_index((0, deg_view, not legacy))
    pos = {f: i for i, f in enumerate(fi)}
    k10, b10 = layers[10]
    rows = k10[256:]
    new = np.empty_like(rows)
    for i, f in enumerate(fo):
        new[pos[f]] = rows[i]
    out = list(layers)
    out[10] = (np.concatenate([k10[:256], new]), b10)
    return out


@pytest.mark.gpu
def test_chain_against_the_executed_reference(golden_dir):
    """the golden's MLP pair through VanillaNerf(num_fine_samples=128).point_stage, host-built tables of its own 40
    directions, pob_sh_proj_cells at S = 1: the executed reference's coefficients and sigma for sh_deg 1..4 within
    its fp32 rounding + the point stage's measured error carried forward + the rows' rounding bound"""
    from plenoctree_b200.octree.projection import VanillaNerf
    from tests.support.eval_stages import TOL_FP16_ANY
    z = np.load(os.path.join(golden_dir, "ref_projection.npz"))
    mlps = {"MLP_0": PJ.init_params(int(z["seeds"][0])), "MLP_1": PJ.init_params(int(z["seeds"][1]))}
    nerf = VanillaNerf(mlps, (0, 10, False), 4, num_fine_samples=128)
    dev = torch.device("cuda")
    pts = torch.from_numpy(z["points"]).to(dev)
    n = pts.shape[0]
    a, sig = nerf.point_stage(pts)
    l64 = [(k.astype(np.float64), b.astype(np.float64)) for k, b in mlps["MLP_1"]]
    a64 = PJ.a_p(l64, pts.cpu().double()).to(dev)
    da = (a.double() - a64).abs()
    d32 = z["dirs"]
    D = d32.shape[0]
    enc = PO.posenc(torch.from_numpy(d32).double(), 0, 4).to(dev)
    t64 = (enc @ torch.from_numpy(mlps["MLP_1"][10][0][256:]).double().to(dev)).T.contiguous()      # [128, D]
    t32 = t64.float()
    st = Stats()
    for sh in range(1, 5):
        K = (sh + 1) ** 2
        Y64 = O.sh_basis(sh, torch.from_numpy(d32).double().to(dev))
        Y32 = Y64.float()
        out, tail = _cells(nerf, a, sig, 1, sh, (None, t32[None].contiguous(), Y32[None].contiguous()), n, n)
        st.add("tails_written", int(not tail))
        ref = torch.from_numpy(np.concatenate([z[f"coeffs_deg{sh}"], z[f"sigma_deg{sh}"]], 1)).double().to(dev)
        _, stage = _rows64(a, sig, t32, Y32, nerf.w11, nerf.b11, 1)
        carry = _carried(da, (t32.double() - t64).abs(), (Y32.double() - Y64).abs(), a, t64, Y64, nerf.w11,
                         nerf.b11, 1)
        gold = GOLDEN_REL * ref[:, :3 * K].abs().max()
        bnd = stage[:, :3 * K] + carry + gold
        st.max("golden_excess", float(((out[:, :3 * K].double() - ref[:, :3 * K]).abs() / bnd).max()) / ROWS_ALLOW)
        # raw sigma (stage-checked in A) at the fp16 point-evaluation bar
        sb = stage[:, 3 * K:] + (GOLDEN_REL + TOL_FP16_ANY) * ref[:, 3 * K:].abs().max()
        st.max("golden_sigma_excess", float(((out[:, 3 * K:].double() - ref[:, 3 * K:]).abs() / sb).max()))
        # guard: the coarse MLP's branch in place of the fine one
        other = PJ.project(mlps["MLP_0"], pts.cpu().double(), torch.from_numpy(d32).double(), sh)[0]
        other = other.reshape(n, -1).to(dev)
        st.min("guard_golden_other_mlp", float(((out[:, :3 * K].double() - other).abs() / bnd).max()))
        st.max("carried_over_gold", float((carry / gold).max()))
    _record("D/golden", st.d)
    assert st.d["tails_written"] == 0, st.d
    assert st.d["golden_excess"] <= 1.0 and st.d["golden_sigma_excess"] <= 1.0, st.d
    assert st.d["guard_golden_other_mlp"] >= GUARD, st.d


D_ROWS = [((0, 10, False), 4, 128), ((2, 8, True), 10, 0), ((0, 0, False), 0, 128), ((2, 8, True), 4, 128),
          ((0, 0, False), 10, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("pe,deg_view,nfs", D_ROWS,
                         ids=lambda v: (f"{v[0]}_{v[1]}_{int(v[2])}" if isinstance(v, tuple) else str(v)))
def test_chain_against_the_oracle_across_flags(pe, deg_view, nfs):
    """the device chain (point stage, direction tables, leaf rows) on the kernel's own directions against the fp64
    oracle PJ.leaf_rows of the MLP that eval_points_raw picks (MLP_1 with a fine level, else MLP_0), under the rows'
    bound plus the measured point-stage and table errors carried forward.  Guards: the other MLP, the other view
    posenc order, b10 left out of the composed head bias."""
    from plenoctree_b200.octree import projection as P
    from plenoctree_b200.octree.projection import VanillaNerf
    from tests.support.eval_stages import TOL_FP16_ANY
    dev = torch.device("cuda")
    mlps = _mlps(61, pe, deg_view)
    nerf = VanillaNerf(mlps, pe, deg_view, num_fine_samples=nfs)
    used, other = (mlps["MLP_1"], mlps["MLP_0"]) if nfs > 0 else (mlps["MLP_0"], mlps["MLP_1"])
    S, n, D, sh = 2, 40, 100, 4
    pts = _points(n * S, seed=deg_view + 7)
    tables, ok = _tables(nerf, sh, D, 0, 1, seed=19)
    dirs, t, basis = (x[0] for x in tables)
    a, sig = nerf.point_stage(pts)
    out, tail = _cells(nerf, a, sig, S, sh, tables, n, n)
    l64 = lambda ls: [(k.astype(np.float64), b.astype(np.float64)) for k, b in ls]
    p64, d64 = pts.cpu().double(), dirs.cpu().double()
    a64 = PJ.a_p(l64(used), p64, pe).to(dev)
    enc = PO.posenc(d64, 0, deg_view, bool(pe[2])).to(dev)
    t64 = (enc @ torch.from_numpy(used[10][0][256:]).double().to(dev)).T
    Y64 = O.sh_basis(sh, d64.to(dev))
    _, stage = _rows64(a, sig, t, basis, nerf.w11, nerf.b11, S)
    carry = _carried((a.double() - a64).abs(), (t.double() - t64).abs(), (basis.double() - Y64).abs(), a, t64, Y64,
                     nerf.w11, nerf.b11, S)
    bnd = stage[:, :-1] + carry

    def ratio(layers):
        ref = PJ.leaf_rows(l64(layers), p64.reshape(n, S, 3), d64, sh, pe, deg_view).to(dev)
        return float(((out[:, :-1].double() - ref[:, :-1]).abs() / bnd.clamp_min(1e-300)).max()), ref

    st = Stats()
    st.add("tails_written", int(not ok) + int(not tail))
    r, ref = ratio(used)
    st.max("oracle_excess", r / ROWS_ALLOW)
    # raw sigma (stage-checked in A) at the fp16 point-evaluation bar
    sb = stage[:, -1] + TOL_FP16_ANY * ref[:, -1].abs().max()
    st.max("sigma_excess", float(((out[:, -1].double() - ref[:, -1]).abs() / sb).max()))
    st.min("guard_other_mlp", ratio(other)[0])
    if deg_view > 1:
        st.min("guard_other_view_order", ratio(_perm_view(used, deg_view, bool(pe[2])))[0])
    no_b10 = list(used)
    no_b10[10] = (used[10][0], np.zeros_like(used[10][1]))
    st.min("guard_no_b10", ratio(no_b10)[0])
    _record(f"D/{pe[0]}_{pe[1]}_{int(pe[2])}_dv{deg_view}_nfs{nfs}", st.d)
    d = st.d
    assert d["tails_written"] == 0, d
    assert d["oracle_excess"] <= 1.0 and d["sigma_excess"] <= 1.0, d
    for k, v in d.items():
        if k.startswith("guard_"):
            assert v >= GUARD, (k, d)

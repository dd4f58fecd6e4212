"""The training and inference kernels at every SM count they split work for (POB_SM_COUNT).

The library divides its work by the SM count it runs on (include/plenoctree_b200.h: pob_sm_count): the persistent
grids of the forward and the data gradient, the backward's share of data-gradient CTAs (pipeline.cu:
DGRAD_SMS_OF_132), the weight gradient's CTAs per role, and with them each CTA's row half and tile stride
(wgrad_body.cuh) and the partials reduce_grads sums (optim.cu).  The rest of the suite runs at the split of the card
it runs on; here POB_SM_COUNT replays, on one card, the splits of

  16          the floor: one CTA per weight-gradient unit, every wgrad CTA sums all tiles of its level
  32, 60, 64  MIG slices
  114         the H100 PCIe
  17, 61      fp16x3 passes with an odd number of CTAs beyond the 16 units
  device      the card itself (POB_SM_COUNT unset)

and holds each to the existing stage checks against fp64 (test_train_stages.py, test_train_x3.py,
test_net_activation.py), to bit-identical per-tile results across splits, and to the refusal of counts outside
[16, device SMs].  Per-count figures, with each count's work split, go to parity_sm_splits.json beside the other
parity records (tests/test_train.py: OUT).

An odd number of wgrad CTAs beyond the 16 units leaves one that only a transposed role (Dense_0^T, heads^T) can take,
which changes that role's CTA count and tile stride: the fp16 step has one at 32, 60 and 64 SMs (SH16) and at 60, 64
and 114 (SH25), the fp16x3 passes at 17 and 61.

Weight-gradient bar: WG_EPS_W was measured with up to ~1 200 tiles summed per CTA.  At 16 SMs every wgrad CTA sums
every tile of its level (its role has one CTA per row half), so the cases below keep a level at <= 392 tiles.
"""
import functools
import json
import os
import re
import time

import numpy as np
import pytest
import torch

from plenoctree_b200 import layouts as L
from tests.support.mlp_stages import X3, Case, stage_case
from tests.support.model_flags import _device_sms, _set_sms
from tests.support.records import ROOT, record

COUNTS = (16, 17, 32, 60, 61, 64, 114, "device")
MIN_SMS = 16


_record = functools.partial(record, "parity_sm_splits.json")


# =====================================================================================================================
# the work split, restated
# =====================================================================================================================
def _dgrad_share():
    """(DGRAD_SMS_OF_132, DGRAD_SMS_OF_132_NH80), read from pipeline.cu"""
    src = open(os.path.join(ROOT, "plenoctree_b200", "csrc", "pipeline.cu")).read()
    return tuple(int(re.search(rf"constexpr int {n} = (\d+);", src).group(1))
                 for n in ("DGRAD_SMS_OF_132", "DGRAD_SMS_OF_132_NH80"))


def _assign_roles(n_in, NH):
    """optim.cu: wgrad_assign_roles -> CTAs per role (Dense_1..7 in row-half pairs, Dense_0^T, heads^T)"""
    halves = [2] * 7 + [1, 1]
    cost = [32 + 64 + (16 if r + 1 == 5 else 0) for r in range(7)] + [16 + 64, (16 if NH <= 64 else 32) + 64]
    n = max(min(n_in, L.WG_MAX_CTAS), sum(halves))
    per_unit = [1] * 9
    left = n - sum(halves)
    while True:
        best = -1
        for r in range(9):
            if halves[r] <= left and (best < 0 or cost[r] * per_unit[best] > cost[best] * per_unit[r]):
                best = r
        if best < 0:
            break
        per_unit[best] += 1
        left -= halves[best]
    return [p * h for p, h in zip(per_unit, halves)]


def split_table(sms, NH):
    """the backward's split at `sms` SMs: data-gradient CTAs and wgrad CTAs per role of the fp16 step (beside the data
    gradient) and of each fp16x3 pass (on all SMs)"""
    share = _dgrad_share()[0 if NH <= 64 else 1]
    dgrad = sms * share // 132
    return dict(dgrad_ctas=dgrad, wgrad_fp16=_assign_roles(sms - dgrad, NH), wgrad_fp16x3=_assign_roles(sms, NH))


def test_split_tables_differ_between_counts():
    """every count of the sweep (and the 132 SMs of an H100 SXM) gives its own split, so none of them re-tests
    another's; each is resident on the device: dgrad + wgrad CTAs <= the device's SMs (here the SXM's 132)"""
    seen = {}
    for sms in [c for c in COUNTS if c != "device"] + [132]:
        t16, t80 = split_table(sms, 16), split_table(sms, 80)
        key = json.dumps([t16, t80])
        assert key not in seen, (sms, seen.get(key))
        seen[key] = sms
        for t in (t16, t80):
            assert t["dgrad_ctas"] >= 1
            assert t["dgrad_ctas"] + sum(t["wgrad_fp16"]) <= 132 and sum(t["wgrad_fp16x3"]) <= 132
            assert all(c % 2 == 0 for c in t["wgrad_fp16"][:7] + t["wgrad_fp16x3"][:7])
    # the odd leftovers the sweep is meant to reach (module docstring): the fp16 step at both heads widths, fp16x3
    def odd(sms, NH, key):
        t = split_table(sms, NH)
        return (sum(t[key]) - 16) % 2 == 1
    counts = [c for c in COUNTS if c != "device"]
    assert [c for c in counts if odd(c, 16, "wgrad_fp16")] == [32, 60, 64]
    assert [c for c in counts if odd(c, 80, "wgrad_fp16")] == [60, 64, 114]
    assert [c for c in counts if odd(c, 16, "wgrad_fp16x3")] == [17, 61]
    assert split_table(60, 16)["wgrad_fp16"][7:] == [3, 2] and split_table(17, 16)["wgrad_fp16x3"][7:] == [2, 1]
    assert split_table(16, 16)["wgrad_fp16"] == split_table(16, 80)["wgrad_fp16"] == [2] * 7 + [1, 1]


# =====================================================================================================================
# GPU: the count in effect
# =====================================================================================================================


def _counts():
    dev = _device_sms()
    return [c for c in COUNTS if c == "device" or c <= dev]


@pytest.fixture(params=COUNTS, ids=str)
def sms(request, monkeypatch):
    """the SM count the library splits for during the test (monkeypatch restores POB_SM_COUNT afterwards)"""
    return _set_sms(monkeypatch, request.param)


# =====================================================================================================================
# A-C: the stage checks against fp64 at each split
# =====================================================================================================================
STAGE_CASES = [
    Case(3, 96, 64, 128, 300),      # test_train.py's shape: 148 fine-level tiles
    Case(-1, 40, 64, 128, 64),      # NH 16: the heads role is split-K
    Case(4, 40, 64, 128, 64),       # NH 80: heads from two A chunks; its own dgrad share (DGRAD_SMS_OF_132_NH80)
    Case(3, 1, 3, 5, 1),            # one tile: almost every CTA has no items
    Case(3, 8, 64, 0, 1),           # 513 rows
    Case(3, 256, 64, 128, 1000),    # 392 fine-level tiles: at 16 SMs every wgrad CTA sums all 392, at 132 >= 39
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", STAGE_CASES, ids=lambda c: c.name)
def test_fp16_stages_at_split(sms, case):
    """test_train_stages' checks unchanged (0xFF-filled workspace, sensitivity guard on) at this count: forward and
    data gradient against fp64 from their own inputs, weight gradient + reduce against fp64 sums at WG_EPS_W"""
    table = split_table(sms, L.heads_width(L.K_of(case.sh)))
    stage_case(case, lambda name, res: _record(f"fp16_stages/{sms}/{name}", {**res, "split": table}))


@pytest.mark.gpu
@pytest.mark.parametrize("case", [Case(3, 96, 64, 128, 300), Case(4, 40, 64, 128, 64)], ids=lambda c: c.name)
def test_fp16x3_stages_at_split(sms, case):
    """test_train_x3's checks unchanged: the x3 data gradient and all three wgrad passes run on all `sms` SMs"""
    table = split_table(sms, L.heads_width(L.K_of(case.sh)))
    stage_case(case.replace(precision=X3),
               lambda name, res: _record(f"fp16x3_stages/{sms}/{name}", {**res, "split": table}), guard=False)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [Case(3, 96, 64, 128, 300), Case(4, 40, 64, 128, 64)], ids=lambda c: c.name)
def test_elu_trunk_stages_at_split(sms, case):
    """test_net_activation's fp16 checks with an elu trunk: its data gradient reads h, not the masks"""
    table = split_table(sms, L.heads_width(L.K_of(case.sh)))
    stage_case(case.replace(act="elu", centre=True),
               lambda name, res: _record(f"elu_stages/{sms}/stages_elu_fp16_{name}", {**res, "split": table}),
               guard=False)


# =====================================================================================================================
# D: what is computed per tile does not depend on the split
# =====================================================================================================================
PER_TILE = ("z", "rgbs", "weights", "comp", "disp", "acc", "G", "H", "E", "DZ", "DO", "mask")


def _level_bytes(ws, views):
    """{(level, region): workspace bytes} of every per-tile / per-ray region of a training call"""
    out = {}
    for i, lv in enumerate(views["levels"]):
        for name in PER_TILE:
            off, shape = lv[name]
            n = int(np.prod(shape)) * (1 if name in ("H", "E", "DZ", "DO") else 4)
            out[(i, name)] = ws[off:off + n].clone()
    return out


def _written_partials(ws, views, mlp):
    """wgrad partial slots of one MLP that a CTA wrote: each CTA writes some of its slot's 256 bias sums, and a slot no
    CTA owns keeps the 0xFF fill"""
    off = views["partials"][mlp]
    P = ws[off:off + 4 * L.WG_MAX_CTAS * L.WG_PARTIAL_FLOATS].view(torch.int32).view(L.WG_MAX_CTAS, -1)
    written = (P[:, 65536:65536 + 256] != -1).any(1).cpu().numpy()
    return written


@pytest.mark.gpu
@pytest.mark.parametrize("case", [Case(3, 96, 64, 128, 300), Case(4, 40, 64, 128, 64)], ids=lambda c: c.name)
def test_per_tile_results_do_not_depend_on_the_split(case, monkeypatch):
    """z, rgbs, weights, comp / disp / acc, G and the saved H, E, masks, DZ, DO are bit-identical at every count to the
    device's; the flat gradient differs only in the order of its fp32 sums (test_fp16_stages_at_split holds each
    count to fp64), and two calls at one count give the same bits.  The wgrad partial slots the CTAs wrote are
    exactly the first sum(split_table(...)["wgrad_fp16"]) of each MLP: the restated split is the library's."""
    t0 = time.time()
    NH = L.heads_width(L.K_of(case.sh))
    base = None
    rep = {}
    for n in ["device"] + [c for c in _counts() if c != "device"]:
        sms = _set_sms(monkeypatch, n)
        model = case.model()
        state, ctx = case.run(model, fill=0xFF)
        ws = model.workspace(True)
        views = L.train_workspace_views(model.cfg, ctx["n"], case.nsp > 0)
        regions = _level_bytes(ws, views)
        grads = state.grads.clone()
        want = sum(split_table(sms, NH)["wgrad_fp16"])
        written = [_written_partials(ws, views, i) for i in range(len(views["levels"]))]
        again, _ = case.run(model, fill=0xFF)
        if base is None:
            base = (regions, grads)
        g0 = base[1].double()
        rep[str(sms)] = dict(
            split=split_table(sms, NH),
            region_mismatches={f"{i}.{k}": int((v != base[0][(i, k)]).sum()) for (i, k), v in regions.items()},
            grad_max_rel_diff_from_device=float((grads.double() - g0).abs().max() / g0.abs().max()),
            grad_bit_differences_from_device=int((grads.view(torch.int32) != base[1].view(torch.int32)).sum()),
            repeat_bit_differences=int((again.grads.view(torch.int32) != grads.view(torch.int32)).sum()),
            written_partial_slots=[int(w.sum()) for w in written],
            first_unwritten_slot=[int(np.argmin(w)) if not w.all() else L.WG_MAX_CTAS for w in written],
            wgrad_ctas=want)
    _record(f"invariance/{case.name}", dict(counts=rep, wall_s=time.time() - t0))
    for sms, r in rep.items():
        assert all(v == 0 for v in r["region_mismatches"].values()), (sms, r["region_mismatches"])
        assert r["repeat_bit_differences"] == 0, (sms, r)
        assert r["written_partial_slots"] == [r["wgrad_ctas"]] * len(r["written_partial_slots"]), (sms, r)
        assert r["first_unwritten_slot"] == r["written_partial_slots"], (sms, r)
        assert np.isfinite(r["grad_max_rel_diff_from_device"]), (sms, r)


# =====================================================================================================================
# E, F: L2 discard and graph replay at other splits
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("sms", [16, 61, "device"], indirect=True, ids=str)
@pytest.mark.parametrize("sh_deg", [3, 4])
def test_l2_discard_at_split(sms, sh_deg):
    """POB_TRAIN_DISCARD_SAVED_GRADS on and off (test_l2_discard's helpers, 512 rays): which CTA loads, and so
    discards, each dZ / dO tile depends on the split.  Gradient bit-identical, the loss sums (float atomics over rays)
    within test_l2_discard's bar, every workspace byte outside DZ / DO identical."""
    from plenoctree_b200.nerf import train as T
    from tests.support import model_flags as LD
    R = 512
    model = LD._model(sh_deg, LD.NF, 1000, R=R)
    state = T.TrainState(model)
    batch, _ = LD._batch(R, 11)
    kw = dict(sparsity_length=0.05, sparsity_radius=1.5)
    g0, s0, w0 = LD._call(model, state, batch, True, **kw)
    g1, s1, w1 = LD._call(model, state, batch, False, **kw)
    assert torch.isfinite(g0).all()
    assert torch.equal(g0, g1)
    assert torch.allclose(s0, s1, rtol=1e-5, atol=0)
    assert LD._equal_outside(w0, w1, LD._saved_grad_ranges(model, R, True))


@pytest.mark.gpu
@pytest.mark.parametrize("sms", [60], indirect=True, ids=str)
def test_graph_replay_at_split(sms):
    """a GraphedTrainStep captured at 60 SMs replays the eager train_step at 60 bit for bit (params, Adam moments)"""
    from plenoctree_b200.nerf import train as T
    from tests.support import model_flags as LD
    R = 512
    batch, b12 = LD._batch(R, 13)
    outs = []
    for graphed in (False, True):
        model = LD._model(3, LD.NF, 1000, R=R)
        state = T.TrainState(model)
        graph = T.GraphedTrainStep(model, state, R) if graphed else None
        for lr in (5e-4, 4e-4, 3e-4):
            if graphed:
                graph.step(b12, lr)
            else:
                T.train_step(model, state, batch, lr)
        torch.cuda.synchronize()
        outs.append((model.params.clone(), state.m.clone(), state.v.clone()))
    for name, a, b in zip(("params", "m", "v"), *outs):
        assert torch.equal(a, b), name


# =====================================================================================================================
# G: inference forwards
# =====================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("sh", [3, 4])
def test_inference_forwards_do_not_depend_on_the_split(sh, monkeypatch):
    """eval_points_raw (rgb + sigma, sigma only), eval_points, eval_grid and render_rays, fp16 and fp16x3: bit-identical
    at every count, at test_eval_stages' ragged sizes and at 9 tiles per CTA of 16 SMs (each CTA through every ring
    phase), canaries behind every output.  Cell means use float atomics: at every count against the fp64 mean of the
    same precision's OUT_RAW rows at test_eval_stages' summation bound."""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    from plenoctree_b200.nerf.models import Rays
    from tests.support import eval_stages as ES
    t0 = time.time()
    dev = torch.device("cuda")
    blob = ES._blob(O.init_flat_params(sh, 43, bias_scale=0.05), sh)
    M = 9 * MIN_SMS * L.TILE_M + 77
    rs = np.random.RandomState(3 + sh)
    x = torch.from_numpy(rs.uniform(-1.5, 1.5, size=(M, 3)).astype(np.float32)).to(dev)
    vd = rs.normal(size=(M, 3))
    vd = torch.from_numpy((vd / np.linalg.norm(vd, axis=1, keepdims=True)).astype(np.float32)).to(dev)
    reso, off, sc = 128, [0.5, 0.45, 0.55], [0.3, 0.35, 0.32]
    slab = (5, 2, 128, 77)
    case = Case(sh, 96, 64, 128, 0) if sh == 3 else Case(sh, 40, 64, 0, 0)
    model = case.model()
    (o, d, v, _), t_rand, u, _, _ = case.inputs(case.R)
    cells = {S: 3 * MIN_SMS * L.TILE_M // S + 3 for S in (5, 96)}      # three or more tiles per CTA of 16 SMs

    def outputs():
        out = {}
        for pr in (ops.PREC_FP16, ops.PREC_FP16X3):
            for m in ES.M_RAGGED + (M,):
                xm, vm = x[:m].contiguous(), vd[:m].contiguous()
                out[(pr, "raw", m)] = ES._raw(blob, sh, xm, pr)
                out[(pr, "sigma", m)] = ES._raw(blob, sh, xm, pr, want_rgb=False)[1]
                out[(pr, "rgbs", m)] = ES._rgbs(blob, sh, xm, vm, pr)
            out[(pr, "grid")] = ES._grid(blob, sh, reso, off, sc, *slab, pr, True)
            out[(pr, "grid_sigma")] = ES._grid(blob, sh, reso, off, sc, *slab, pr, False)[1]
            model.workspace(False).fill_(0xFF)
            r = model(Rays(o, d, v), randomized=True, t_rand=t_rand, u=u, precision=pr)
            torch.cuda.synchronize()
            out[(pr, "render")] = [t.clone() for lvl in r for t in lvl] + [model.workspace(False).clone()]
        return out

    def flat(v):
        return [t for t in (v if isinstance(v, (tuple, list)) else (v,)) if t is not None]

    def cell_errors():
        worst = 0.0
        for pr in (ops.PREC_FP16, ops.PREC_FP16X3):
            for S, n_cells in cells.items():
                g = np.random.RandomState(S)
                centres = g.uniform(-1.4, 1.4, size=(n_cells, 1, 3))
                pts = torch.from_numpy((centres + g.uniform(-0.05, 0.05, size=(n_cells, S, 3))).astype(np.float32)
                                       .reshape(-1, 3)).to(dev)
                got = ES._cells(blob, sh, pts, n_cells, S, pr)
                rr, ss = ES._raw(blob, sh, pts, pr)
                vals = torch.cat([rr, ss[:, None]], 1).double().view(n_cells, S, -1)
                bound = ES._cell_bound(S) * ES.U24 * vals.abs().sum(1) / S
                assert torch.isfinite(got).all()
                worst = max(worst, float(((got.double() - vals.mean(1)).abs() / bound.clamp_min(1e-300)).max()))
        return worst

    rep = {}
    base = None
    for n in ["device"] + [c for c in _counts() if c != "device"]:
        sms = _set_sms(monkeypatch, n)
        out = outputs()
        if base is None:
            base = out
        mism = {f"{k[0]}/{k[1]}" + (f"/{k[2]}" if len(k) > 2 else ""):
                sum(ES._nbits(a, b) for a, b in zip(flat(out[k]), flat(base[k]))) for k in out}
        rep[str(sms)] = dict(bit_mismatches=mism, cell_err_over_bound=cell_errors())
    _record(f"inference/sh{sh}", dict(counts=rep, M=M, wall_s=time.time() - t0))
    for sms, r in rep.items():
        assert all(v == 0 for v in r["bit_mismatches"].values()), (sms, {k: v for k, v in r["bit_mismatches"].items() if v})
        assert r["cell_err_over_bound"] <= 1.0, (sms, r["cell_err_over_bound"])


@pytest.mark.gpu
def test_projection_point_stage_does_not_depend_on_the_split(monkeypatch):
    """pob_sh_proj_points (the saving relu forward on SRC_POINTS, then a_p): a_p, raw sigma and the whole workspace
    (h_0..h_7, posenc and mask images) bit-identical at every count, at 9 tiles per CTA of 16 SMs"""
    from plenoctree_b200.octree.projection import VanillaNerf
    from oracle import projection_oracle as PJ
    from tests.support.model_flags import _points, _run_points
    nerf = VanillaNerf({"MLP_0": PJ.init_params(45)}, (0, 10, False), 4, num_fine_samples=0)
    M = 9 * MIN_SMS * L.TILE_M + 77
    pts = _points(M, 9)
    base, rep = None, {}
    for c in ["device"] + [c for c in _counts() if c != "device"]:
        sms = _set_sms(monkeypatch, c)
        ws, a, s, ab, sb = _run_points(nerf, pts)
        out = (a.contiguous().view(torch.int32), s.view(torch.int32), ws, ab, sb)
        base = base or out
        rep[str(sms)] = dict(a=int((out[0] != base[0]).sum()), sigma=int((out[1] != base[1]).sum()),
                             workspace=int((out[2] != base[2]).sum()), tails=int((out[3] != base[3]).sum()) +
                             int((out[4] != base[4]).sum()))
    _record("projection_points", dict(counts=rep, M=M))
    assert bool(torch.isfinite(base[0].view(torch.float32)).all()) and bool(torch.isfinite(base[1].view(torch.float32)).all())
    for sms, r in rep.items():
        assert all(v == 0 for v in r.values()), (sms, r)


# =====================================================================================================================
# H: octree optimiser steps
# =====================================================================================================================
@pytest.mark.gpu
def test_octree_optimiser_steps_do_not_depend_on_the_split(monkeypatch):
    """pob_octree_sgd_step, _sgd_momentum_step (plain and Nesterov) and _adam_step: grid-stride loops over
    sms * 16 blocks, four float4 per thread per pass and a scalar tail; n gives 16 SMs several passes and a
    3-element tail.  Data, gradient, momentum buffer and Adam moments bit-identical at every count."""
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    dev = torch.device("cuda")
    n = 3 * 4 * 4 * MIN_SMS * 16 * 256 + 7
    g = torch.Generator(device="cpu").manual_seed(5)
    data0 = torch.randn(n, generator=g).to(dev)
    grad0 = torch.randn(n, generator=g).to(dev) * (torch.rand(n, generator=g) < 0.6).to(dev)   # zeros are skipped
    buf0 = torch.randn(n, generator=g).to(dev) * (torch.rand(n, generator=g) < 0.5).to(dev)
    v0 = torch.rand(n, generator=g).to(dev)

    def steps():
        out = {}
        d, gr = data0.clone(), grad0.clone()
        check(lib.pob_octree_sgd_step(ptr(d), ptr(gr), n, 0.7, stream_ptr()))
        out["sgd"] = (d, gr)
        for nest in (0, 1):
            d, gr, b = data0.clone(), grad0.clone(), buf0.clone()
            check(lib.pob_octree_sgd_momentum_step(ptr(d), ptr(gr), ptr(b), n, 0.7, 0.9, nest, stream_ptr()))
            out[f"momentum_nesterov{nest}"] = (d, gr, b)
        d, gr, m, v = data0.clone(), grad0.clone(), buf0.clone(), v0.clone()
        check(lib.pob_octree_adam_step(ptr(d), ptr(gr), ptr(m), ptr(v), n, 0.1, 3.0, 1e-8, stream_ptr()))
        out["adam"] = (d, gr, m, v)
        torch.cuda.synchronize()
        return out

    base = None
    rep = {}
    for c in ["device"] + [c for c in _counts() if c != "device"]:
        sms = _set_sms(monkeypatch, c)
        out = steps()
        base = base or out
        rep[str(sms)] = {k: sum(int((a.view(torch.int32) != b.view(torch.int32)).sum()) for a, b in zip(out[k], base[k]))
                         for k in out}
    _record("octree_optimisers", rep)
    assert not torch.equal(base["sgd"][0], data0) and bool((base["sgd"][1] == 0).all())
    for sms, r in rep.items():
        assert all(v == 0 for v in r.values()), (sms, r)


# =====================================================================================================================
# I: counts outside [16, device SMs] are refused before anything is launched
# =====================================================================================================================
@pytest.mark.gpu
def test_out_of_range_counts_are_refused(monkeypatch):
    """POB_SM_COUNT = 15, device + 1, 0, -3, abc, "" and 16x: pob_sm_count() < 0, and every entry point that splits
    work by it fails with a message naming POB_SM_COUNT, launches nothing and leaves the canary behind (or in) its
    output untouched.  A valid count afterwards works again."""
    import ctypes
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200._lib import PobError, lib, ptr, stream_ptr
    from plenoctree_b200.nerf import train as T
    from plenoctree_b200.nerf.models import Rays
    from tests.support import eval_stages as ES
    dev = torch.device("cuda")
    sh = 3
    blob = ES._blob(O.init_flat_params(sh, 47, bias_scale=0.05), sh)
    m, C3 = 1000, 3 * L.K_of(sh)
    x = torch.rand(m, 3, device=dev)
    vd = torch.nn.functional.normalize(torch.randn(m, 3, device=dev), dim=1)
    case = Case(3, 40, 64, 128, 64)
    model = case.model()
    (o, d, v, px), t_rand, u, sp, _ = case.inputs(case.R)
    state = T.TrainState(model)
    nq = 4096 + 3
    from oracle import projection_oracle as PJ
    from plenoctree_b200.octree.projection import VanillaNerf
    vn = VanillaNerf({"MLP_0": PJ.init_params(46)}, (0, 10, False), 4, num_fine_samples=0)
    nd, ncell, S, psh = 40, 10, 2, 4
    K = (psh + 1) ** 2
    a_in, s_in = torch.zeros(ncell * S, 128, device=dev), torch.zeros(ncell * S, device=dev)
    t_in, y_in = torch.zeros(128 * nd, device=dev), torch.zeros(nd * K, device=dev)

    def canary(k):
        return ES._canary(k, tail=0)

    def calls():
        """name -> (call returning rc or raising PobError, buffers that must keep the canary)"""
        rb, sb, ob, gb, cb, tb = canary(m * C3), canary(m), canary(4 * m), canary(m * C3), canary(10 * (C3 + 1)), canary(64)
        q = [canary(nq) for _ in range(4)]
        pw = canary(int(lib.pob_sh_proj_points_workspace_bytes(m)) // 4)
        pa, ps = canary(m * 128), canary(m)
        pd, pt, pb = canary(2 * nd * 3), canary(2 * 128 * nd), canary(2 * nd * K)
        pc = canary(ncell * (3 * K + 1))
        f3 = ctypes.c_float * 3
        return {
            "pob_eval_points_raw": (lambda: lib.pob_eval_points_raw(ptr(blob), sh, ptr(x), m, ptr(rb), ptr(sb), 1,
                                                                    stream_ptr()), [rb, sb]),
            "pob_eval_points": (lambda: lib.pob_eval_points(ptr(blob), sh, ptr(x), ptr(vd), m, ptr(ob), 3,
                                                            stream_ptr()), [ob]),
            "pob_eval_grid": (lambda: lib.pob_eval_grid(ptr(blob), sh, 16, 0, 3, 16, 16, f3(0.5, 0.5, 0.5),
                                                        f3(0.3, 0.3, 0.3), ptr(gb), ptr(sb), 1, stream_ptr()), [gb, sb]),
            "pob_eval_cells_mean": (lambda: lib.pob_eval_cells_mean(ptr(blob), sh, ptr(x), 10, 100, ptr(cb), 1,
                                                                    stream_ptr()), [cb]),
            "pob_draw_uniforms": (lambda: lib.pob_draw_uniforms(1, 0.0, None, ptr(tb), 64, None, 0, None, 0, 1.5,
                                                                stream_ptr()), [tb]),
            "pob_octree_sgd_step": (lambda: lib.pob_octree_sgd_step(ptr(q[0]), ptr(q[1]), nq, 0.5, stream_ptr()),
                                    q[:2]),
            "pob_octree_sgd_momentum_step": (lambda: lib.pob_octree_sgd_momentum_step(
                ptr(q[0]), ptr(q[1]), ptr(q[2]), nq, 0.5, 0.9, 1, stream_ptr()), q[:3]),
            "pob_octree_adam_step": (lambda: lib.pob_octree_adam_step(ptr(q[0]), ptr(q[1]), ptr(q[2]), ptr(q[3]), nq,
                                                                      0.5, 1.0, 1e-8, stream_ptr()), q),
            "pob_sh_proj_points": (lambda: lib.pob_sh_proj_points(ptr(vn.sigma_blob), None, ptr(x), m, ptr(vn.head_w),
                                                                  ptr(vn.head_b), ptr(pw), ptr(pa), ptr(ps),
                                                                  stream_ptr()), [pw, pa, ps]),
            "pob_sh_proj_directions": (lambda: lib.pob_sh_proj_directions(5, 0, 2, nd, 4, 0, psh, ptr(vn.w10e),
                                                                          ptr(pd), ptr(pt), ptr(pb), stream_ptr()),
                                       [pd, pt, pb]),
            "pob_sh_proj_cells": (lambda: lib.pob_sh_proj_cells(ncell, S, 4, ptr(a_in), ptr(s_in), nd, psh, ptr(t_in),
                                                                ptr(y_in), ptr(vn.w11), ptr(vn.b11), ptr(pc),
                                                                stream_ptr()), [pc]),
        }

    def raises(fn):
        try:
            fn()
        except PobError as e:
            return str(e)
        return None

    bad = ["15", str(_device_sms() + 1), "0", "-3", "abc", "", "16x"]
    for val in bad:
        monkeypatch.setenv("POB_SM_COUNT", val)
        assert lib.pob_sm_count() < 0, val
        launches = lib.pob_launch_count()
        for name, (fn, bufs) in calls().items():
            assert fn() != 0, (val, name)
            msg = lib.pob_last_error().decode()
            assert "POB_SM_COUNT" in msg and name in msg, (val, name, msg)
            torch.cuda.synchronize()
            assert all(bool((b == ES.CANARY).all()) for b in bufs), (val, name)
        ws = model.workspace(False)
        ws.fill_(0xFF)
        msg = raises(lambda: model(Rays(o, d, v), randomized=True, t_rand=t_rand, u=u))
        assert msg is not None and "POB_SM_COUNT" in msg and "pob_render_rays" in msg, (val, msg)
        tws = model.workspace(True)
        tws.fill_(0xFF)
        state.grads.fill_(float("nan"))
        msg = raises(lambda: T.loss_and_grad(model, state, {"rays": Rays(o, d, v), "pixels": px}, t_rand=t_rand, u=u,
                                             sp_points=sp))
        assert msg is not None and "POB_SM_COUNT" in msg and "pob_loss_and_grad" in msg, (val, msg)
        torch.cuda.synchronize()
        assert bool((ws == 0xFF).all()) and bool((tws == 0xFF).all()) and bool(state.grads.isnan().all()), val
        assert lib.pob_launch_count() == launches, val
    _set_sms(monkeypatch, MIN_SMS)
    fn, bufs = calls()["pob_eval_points_raw"]
    assert fn() == 0
    torch.cuda.synchronize()
    assert torch.isfinite(bufs[1].view(torch.float32)).all()

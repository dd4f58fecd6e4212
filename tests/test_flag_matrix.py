"""The NeRF-SH model flags combined: precision, trunk activation (net_activation), point encoder (min_deg_point,
max_deg_point, legacy_posenc_order), density activation (sigma_activation), SH degree (heads width), ray length,
sigma noise and background, over a covering matrix of rows.

Each flag came in tested with every other flag at its default, while the CLIs accept any combination, and some
compiled paths run only when flags are combined: the fp16 forward's runtime ("generic") encoder inside the elu,
softplus and tanh instantiations, the fp16x3 posenc tile of a narrow encoder, the softplus factor of G.w in the
one-block-per-ray compositing backward (N > 256), a smooth trunk under the softplus density.

CPU: the matrix's covering properties, the forward / data-gradient instantiations each entry point reaches, and the
anchor of the fp64 inference reference to the golden-anchored oracles.
GPU, per row: one training call on a 0xFF-filled workspace, every level's stages against fp64 from the kernels' own
saved tiles (tests/support/mlp_stages.py: check_level) and the per-ray stages (test_ray_stages), each checked again against
the reference of a wrong flag (mutation guards), and the inference forwards of the fine MLP with the same flags.
Once: a CUDA-graph replay of a row with every flag away from its default.
"""
import functools
import os
import re

import numpy as np
import pytest
import torch

from oracle import net_activation_oracle as NA
from oracle import posenc_oracle as PO
from plenoctree_b200 import layouts as L
from tests.support.covering import assert_covers_every_pair
from tests.support.model_flags import _alt_pe
from tests.support.ray_stages import RayCase
from tests.support.records import ROOT, record

X3 = 3
GUARD = 10.0        # a check must miss its bar by at least this factor against the reference of a wrong flag
CELL_S = 32         # cells of 32 samples: the cell-mean epilogue's per-32-row branch (S = 1 takes the other)

DEF_PE = (0, 10, False)
PRECISIONS = ("fp16", "fp16x3")
TRUNKS = ("relu", "elu", "softplus", "tanh")
ENCODERS = (DEF_PE, (0, 10, True), (2, 8, True), (0, 0, False), (9, 10, True))
DENSITIES = ("relu", "softplus")
SH_DEGS = (-1, 2, 3, 4)                        # heads width 16 (split-K heads role), 32, 64, 80
# (rays, coarse, fine, sparsity points)
SHAPES = ((40, 64, 128, 64),                   # both levels, sparsity rows behind the fine level's samples
          (64, 64, 0, 200),                    # one level: sparsity rows on MLP_0
          (16, 128, 384, 200),                 # N = 512: the one-block-per-ray compositing paths
          (1, 3, 5, 1))                        # one real tile
NOISE = (False, True)
WHITE = (True, False)
DIMS = (PRECISIONS, TRUNKS, ENCODERS, DENSITIES, SH_DEGS, SHAPES, NOISE, WHITE)

# precision, trunk, encoder, density, sh_deg, shape, noise, white_bkgd
MATRIX = [
    ("fp16x3", "tanh", (9, 10, True), "softplus", 4, (1, 3, 5, 1), False, True),
    ("fp16x3", "softplus", (0, 10, True), "relu", 2, (64, 64, 0, 200), True, False),
    ("fp16", "relu", (2, 8, True), "relu", 3, (40, 64, 128, 64), True, True),
    ("fp16", "elu", DEF_PE, "softplus", -1, (16, 128, 384, 200), False, False),
    ("fp16x3", "relu", (0, 0, False), "softplus", 3, (1, 3, 5, 1), False, False),
    ("fp16", "softplus", (0, 0, False), "relu", 4, (16, 128, 384, 200), True, True),
    ("fp16", "tanh", (0, 10, True), "relu", -1, (1, 3, 5, 1), True, True),
    ("fp16x3", "elu", DEF_PE, "softplus", 2, (40, 64, 128, 64), True, True),
    ("fp16", "elu", (2, 8, True), "relu", 4, (64, 64, 0, 200), False, True),
    ("fp16x3", "softplus", DEF_PE, "softplus", 4, (40, 64, 128, 64), False, False),
    ("fp16x3", "elu", (2, 8, True), "softplus", 2, (1, 3, 5, 1), False, False),
    ("fp16", "tanh", DEF_PE, "relu", 3, (64, 64, 0, 200), False, False),
    ("fp16x3", "relu", DEF_PE, "relu", -1, (16, 128, 384, 200), True, False),
    ("fp16x3", "tanh", DEF_PE, "softplus", 2, (16, 128, 384, 200), True, True),
    ("fp16", "relu", DEF_PE, "softplus", 2, (64, 64, 0, 200), True, True),
    ("fp16", "softplus", (9, 10, True), "relu", 3, (16, 128, 384, 200), False, False),
    ("fp16", "softplus", DEF_PE, "relu", -1, (1, 3, 5, 1), False, True),
    ("fp16x3", "elu", (0, 10, True), "softplus", 3, (40, 64, 128, 64), False, False),
    ("fp16x3", "relu", (9, 10, True), "softplus", -1, (40, 64, 128, 64), True, True),
    ("fp16x3", "tanh", (0, 0, False), "softplus", 2, (40, 64, 128, 64), False, False),
    ("fp16x3", "elu", (0, 0, False), "softplus", -1, (64, 64, 0, 200), True, True),
    ("fp16x3", "relu", (0, 10, True), "relu", 4, (16, 128, 384, 200), False, True),
    ("fp16x3", "softplus", (2, 8, True), "relu", -1, (16, 128, 384, 200), True, True),
    ("fp16x3", "elu", (9, 10, True), "relu", 2, (64, 64, 0, 200), False, False),
    ("fp16x3", "tanh", (2, 8, True), "softplus", 4, (40, 64, 128, 64), False, True),
]

# the forward (NSPLIT, OUTM, SAVE) and data-gradient NSPLIT each entry point reaches, per trunk activation
# (capi.cu: pob_eval_points_raw_pe, pob_eval_points_act_pe, pob_eval_cells_mean_pe, pob_eval_grid_pe; pipeline.cu:
# the render and training forwards; mlp_bwd.cu: launch_mlp_bwd), and what this file calls per precision
ENTRY_FWD = {
    "train": lambda n: (n, "OUT_RGBS", True),
    "render": lambda n: (n, "OUT_RGBS", False),
    "eval_points": lambda n: (n, "OUT_RGBS", False),
    "eval_points_raw": lambda n: (n, "OUT_RAW", False),
    "eval_points_raw_sigma": lambda n: (n, "OUT_SIGMA", False),
    "eval_grid": lambda n: (n, "OUT_RAW", False),
    "eval_grid_sigma": lambda n: (n, "OUT_SIGMA", False),
    "eval_cells_mean": lambda n: (n, "OUT_CELL_MEAN", False),
}
ENTRY_DGRAD = {"train"}
ROW_ENTRIES = tuple(ENTRY_FWD)                 # every row calls every entry point at its precision
# the saving OUT_SIGMA forward is launched by pob_sh_proj_points alone (projection.cu), which refuses every trunk but
# relu: its relu instantiation runs there (checked stage by stage in test_projection_stages.py,
# test_point_stage_from_saved_tiles); the elu, softplus and tanh ones are compiled and launched by no entry point
PROJ_FWD = {(1, "OUT_SIGMA", True, "relu")}
UNREACHABLE_FWD = {(1, "OUT_SIGMA", True, a) for a in TRUNKS[1:]}


def _tag(row):
    prec, act, pe, dens, sh, (R, nc, nf, nsp), noise, white = row
    return (f"{prec}_{act}_{pe[0]}_{pe[1]}_{'legacy' if pe[2] else 'std'}_{dens}_sh{sh}_R{R}_{nc}+{nf}_sp{nsp}"
            + ("_noise" if noise else "") + ("" if white else "_black"))


_record = functools.partial(record, "parity_flag_matrix.json")


# =====================================================================================================================
# CPU
# =====================================================================================================================
def test_matrix_covers_every_pair():
    """every pair of values of any two dimensions appears in some row"""
    assert_covers_every_pair(MATRIX, DIMS)


def test_matrix_covers_both_encoder_branches_of_every_forward():
    """every (precision, trunk, default or non-default encoder) triple: each forward instantiation runs the default
    and the generic posenc code"""
    seen = {(r[0], r[1], r[2] == DEF_PE) for r in MATRIX}
    want = {(p, a, d) for p in PRECISIONS for a in TRUNKS for d in (True, False)}
    assert seen == want, want - seen


def _compiled_fwd():
    src = open(os.path.join(ROOT, "plenoctree_b200", "csrc", "mlp_fwd.cu")).read()
    body = src[src.index("cudaError_t launch_mlp_fwd("):]
    found = set(re.findall(r"mlp_fwd_kernel<(\d), (OUT_\w+), (true|false), A>", body))
    return {(int(n), o, s == "true") for n, o, s in found}


def test_every_instantiation_is_reached_by_an_entry_point():
    """the forward <NSPLIT, OUTM, SAVE, ACT> and data-gradient <NSPLIT, ACT> instantiations compiled in mlp_fwd.cu /
    mlp_bwd.cu, against the entry table above: every one but the recorded unreachable ones is launched by the rows of
    this file or by the projection's point stage; the table matches the sources' out_mode choices (the training
    forward is the one saving launch of forward_levels, the projection's the only other one and relu only)"""
    fwd = _compiled_fwd()
    assert len(fwd) == 11, sorted(fwd)
    bwd_src = open(os.path.join(ROOT, "plenoctree_b200", "csrc", "mlp_bwd.cu")).read()
    assert "nsplit == 1 ? mlp_bwd_kernel<1, A> : mlp_bwd_kernel<3, A>" in bwd_src
    for act in ("NET_RELU", "NET_ELU", "NET_SOFTPLUS", "NET_TANH"):
        assert f"case {act}:" in bwd_src and f"std::integral_constant<int, {act}>" in bwd_src
    capi = open(os.path.join(ROOT, "plenoctree_b200", "csrc", "capi.cu")).read()
    assert capi.count("p.out_mode = raw_rgb_dev ? pob::OUT_RAW : pob::OUT_SIGMA;") == 2     # points_raw, grid
    assert "p.out_mode = pob::OUT_RGBS;" in capi and "p.out_mode = pob::OUT_CELL_MEAN;" in capi
    pipe = open(os.path.join(ROOT, "plenoctree_b200", "csrc", "pipeline.cu")).read()
    fwd_levels = pipe[pipe.index("int forward_levels("):pipe.index("__global__ void pack_outputs_kernel")]
    assert "p.out_mode = OUT_RGBS;" in fwd_levels and "p.save_h = L.H;" in fwd_levels
    assert fwd_levels.count("launch_mlp_fwd(") == 1 and pipe.count("launch_mlp_fwd(") == 1
    proj = open(os.path.join(ROOT, "plenoctree_b200", "csrc", "projection.cu")).read()
    body = proj[proj.index("int pob_sh_proj_points("):proj.index("int pob_sh_proj_directions(")]
    assert "if (p.net_act != pob::NET_RELU) return pob_fail(" in body
    assert "p.out_mode = pob::OUT_SIGMA;" in body and "p.save_h = base + ws.h;" in body
    assert "pob::launch_mlp_fwd(p, POB_PREC_FP16, sms," in body
    assert "#define POB_PREC_FP16 1\n" in open(os.path.join(ROOT, "include", "plenoctree_b200.h")).read()
    assert "launch_mlp_fwd" not in proj.replace(body, "")
    acts = {(0 if r[0] == "fp16" else 1, r[1]) for r in MATRIX}
    reached_fwd, reached_bwd = set(), set()
    for prec_i, act in acts:
        n = (1, X3)[prec_i]
        for e in ROW_ENTRIES:
            reached_fwd.add(ENTRY_FWD[e](n) + (act,))
            if e in ENTRY_DGRAD:
                reached_bwd.add((n, act))
    reached_fwd |= PROJ_FWD
    want_fwd = {f + (a,) for f in fwd for a in TRUNKS} - UNREACHABLE_FWD
    assert reached_fwd == want_fwd, (want_fwd - reached_fwd, reached_fwd - want_fwd)
    assert {f[:3] for f in UNREACHABLE_FWD | PROJ_FWD} <= fwd
    assert reached_bwd == {(n, a) for n in (1, X3) for a in TRUNKS}


def _anchor_flat(sh, pe, seed):
    return PO.init_flat_params(sh, seed, bias_scale=0.05, pe=pe)


@pytest.mark.parametrize("pe", ENCODERS[1:], ids=lambda pe: f"{pe[0]}_{pe[1]}_{pe[2]}")
def test_reference_anchor_encoder(pe):
    """NA.mlp(PO.unflatten(flat, sh, pe), PO.encode(x, pe), "relu") is the posenc oracle's eval_points_raw, bit for
    bit: the fp64 reference of the inference checks, with only the encoder away from its default"""
    x = torch.from_numpy(np.random.RandomState(2).uniform(-1.5, 1.5, (300, 3)).astype(np.float32))
    for sh in (-1, 3):
        p = PO.unflatten(_anchor_flat(sh, pe, 11), sh, pe)
        with torch.no_grad():
            a = NA.mlp(p, PO.encode(x, pe), "relu")
            b = PO.eval_points_raw(p, x, pe)
        for u, w in zip(a, b):
            assert torch.equal(u, w)


@pytest.mark.parametrize("act", TRUNKS[1:])
def test_reference_anchor_trunk(act):
    """the same reference with only the trunk activation away from its default is the net-activation oracle's
    eval_points_raw, bit for bit"""
    from oracle import nerf_sh_oracle as O
    x = torch.from_numpy(np.random.RandomState(3).uniform(-1.5, 1.5, (300, 3)).astype(np.float32))
    for sh in (-1, 3):
        flat = _anchor_flat(sh, DEF_PE, 12)
        with torch.no_grad():
            a = NA.mlp(PO.unflatten(flat, sh, DEF_PE), PO.encode(x, DEF_PE), act)
            b = NA.eval_points_raw(O.unflatten(flat, sh), x, act)
        for u, w in zip(a, b):
            assert torch.equal(u, w)


# =====================================================================================================================
# GPU
# =====================================================================================================================


def _row_case(row):
    prec, act, pe, dens, sh, (R, nc, nf, nsp), noise, white = row
    return RayCase(sh, R, nc, nf, nsp, noise=noise, white=white, precision=1 if prec == "fp16" else X3, act=act, pe=pe,
                   sigma_act=dens, centre=True)


def _check_row(row):
    from plenoctree_b200 import ops
    from plenoctree_b200.nerf.models import Rays
    from tests.support import ray_stages as RS
    from tests.support.eval_stages import X3Ref, _cell_bound, _level_rows, _nbits, _x3_errors
    from tests.support.mlp_stages import check_call
    prec, act, pe, dens, sh = row[:5]
    case = _row_case(row)
    x3 = case.precision == X3
    dev = torch.device("cuda")
    model = case.model()
    n = case.R
    state, ctx = case.run(model, fill=0xFF)
    called = set()

    # ---- stage checks, and each again against the reference of a wrong flag
    alt = {"act": "softplus" if act == "relu" else "relu", "sigma_act": "softplus" if dens == "relu" else "relu"}
    if _alt_pe(pe) is not None:
        alt["pe"] = _alt_pe(pe)
    res = check_call(model, state, ctx, case.precision, alt)
    called.add("train")
    rays = RS._in_call_checks(case, model, state, n)
    out = {"stages": res, "rays": rays, "alt": dict(alt), "guard_pe_skipped": "pe" not in alt}

    # ---- inference forwards of the last level (the fine MLP, or the only one) with the same flags
    ws = model.workspace(True, case.precision)
    views = L.train_workspace_views(model.cfg, n, case.nsp > 0, precision=case.precision)
    saved = [{k: L.workspace_view(ws, lv, k).clone() for k in ("z", "rgbs")} for lv in views["levels"]]
    (o, d, v, _), t_rand, u, sp, noise = case.inputs(n)
    rws = model.workspace(False)
    rws.fill_(0xFF)
    model(Rays(o, d, v), randomized=True, t_rand=t_rand, u=u, sigma_noise=noise, precision=case.precision)
    torch.cuda.synchronize()
    called.add("render")
    rv = L.train_workspace_views(model.cfg, n, False, training=False)
    inf = {"render_rgbs_bit_mismatches": sum(
        _nbits(L.workspace_view(rws, lr, "rgbs"), saved[i]["rgbs"][:lt["M_rays"]])
        for i, (lt, lr) in enumerate(zip(views["levels"], rv["levels"])))}
    i = len(views["levels"]) - 1
    lv = views["levels"][i]
    Mr, M = lv["M_rays"], lv["M"]
    spt = torch.from_numpy(sp).to(dev) if sp is not None else None
    x, vd = _level_rows(ctx, lv, saved[i]["z"], spt, dev)
    rows = saved[i]["rgbs"][:M]
    blob = model.blobs[i]
    kw = dict(precision=case.precision, posenc=pe, net_activation=model.net_act_code)
    e_rgb, e_sig = ops.eval_points(blob, sh, x, vd, sigma_activation=model.sigma_act_code, **kw)
    called.add("eval_points")
    raw_rgb, raw_sig = ops.eval_points_raw(blob, sh, x, **kw)
    _, sig_only = ops.eval_points_raw(blob, sh, x, want_rgb=False, **kw)
    called |= {"eval_points_raw", "eval_points_raw_sigma"}
    raw_sig, sig_only = raw_sig[:, 0], sig_only[:, 0]
    torch.cuda.synchronize()
    # training rows: the model's density (+ noise) on ray samples, relu of raw sigma on the sparsity rows
    inf["eval_points_rgb_bit_mismatches"] = _nbits(e_rgb[:Mr].contiguous(), rows[:Mr, :3].contiguous())
    if noise is None or noise[i] is None:
        inf["eval_points_sigma_bit_mismatches"] = _nbits(e_sig[:Mr, 0].contiguous(), rows[:Mr, 3].contiguous())
        if dens == "relu":
            inf["raw_sigma_relu_mismatches"] = int((raw_sig[:Mr].clamp_min(0) != rows[:Mr, 3]).sum())
    inf["sparsity_rows_vs_relu_raw_mismatches"] = int((raw_sig[Mr:M].clamp_min(0) != rows[Mr:M, 3]).sum())
    inf["sigma_only_vs_raw_bit_mismatches"] = _nbits(sig_only, raw_sig)
    # cells of one sample are the raw outputs themselves; cells of CELL_S samples within the summation bound
    cells1 = ops.eval_cells_mean(blob, sh, x.reshape(-1, 1, 3).contiguous(), 1, **kw)
    inf["cells_S1_bit_mismatches"] = _nbits(cells1, torch.cat([raw_rgb, raw_sig[:, None]], 1))
    nc_ = M // CELL_S
    if nc_:
        cells = ops.eval_cells_mean(blob, sh, x[:nc_ * CELL_S].contiguous(), CELL_S, **kw)
        vals = torch.cat([raw_rgb, raw_sig[:, None]], 1)[:nc_ * CELL_S].double().view(nc_, CELL_S, -1)
        bound = _cell_bound(CELL_S) * 2.0 ** -24 * vals.abs().sum(1) / CELL_S
        inf["cells_S32_err_over_bound"] = float(((cells.double() - vals.mean(1)).abs() / bound.clamp_min(1e-300)).max())
    called.add("eval_cells_mean")
    # grid: the voxel centres, formed as the kernel forms them (power-of-two scale), through eval_points_raw
    reso, off, scl = 16, (0.5, 0.5, 0.5), (0.5, 0.5, 0.5)
    g_rgb, g_sig = ops.eval_grid(blob, sh, reso, off, scl, want_rgb=True, **kw)
    _, g_sig_only = ops.eval_grid(blob, sh, reso, off, scl, want_rgb=False, **kw)
    called |= {"eval_grid", "eval_grid_sigma"}
    ii = (torch.arange(reso, device=dev, dtype=torch.float32) + 0.5) * (1.0 / reso)
    gx, gy, gz = torch.meshgrid(ii, ii, ii, indexing="ij")
    gp = torch.stack([(g.reshape(-1) - o_) / s_ for g, o_, s_ in zip((gx, gy, gz), off, scl)], 1).contiguous()
    p_rgb, p_sig = ops.eval_points_raw(blob, sh, gp, **kw)
    torch.cuda.synchronize()
    inf["grid_vs_points_bit_mismatches"] = _nbits(g_rgb, p_rgb) + _nbits(g_sig, p_sig[:, 0])
    inf["grid_sigma_only_bit_mismatches"] = _nbits(g_sig_only, p_sig[:, 0])
    if x3:
        from tests.support.mlp_stages import Stats
        st = Stats()
        ref = X3Ref(model.params[i * model.P:(i + 1) * model.P].cpu().numpy(), sh, dev, pe, act)
        _x3_errors(ref, x, raw_rgb, raw_sig, st, "points")
        _x3_errors(ref, gp, p_rgb, p_sig[:, 0], st, "grid")
        inf["x3_points_excess"] = st.d["points_excess"]
        inf["x3_grid_excess"] = st.d["grid_excess"]
    out["inference"] = inf
    assert called == set(ROW_ENTRIES), called
    return out


def _assert_row(row, out):
    from tests.support import ray_stages as RS
    from tests.support.eval_stages import X3_ALLOW
    from tests.support.mlp_stages import BWD_ALLOW, FWD_ALLOW, SIN_ALLOW, assert_stages
    from tests.support.ray_stages import GW_BAR
    prec, act, pe, dens = row[:4]
    x3 = prec == "fp16x3"
    precision = X3 if x3 else 1
    assert_stages(out["stages"], precision, act, guard=False)
    RS._assert_in_call(out["rays"])
    fwd_allow, bwd_allow, sin_bar = FWD_ALLOW[precision], BWD_ALLOW[precision], SIN_ALLOW[precision]
    for mlp, r in out["stages"].items():
        s = r["stages"]
        g_fwd = min(s[f"guard_fwd_l{l}"] for l in range(8))
        g_bwd = min(s[f"guard_bwd_l{l}"] for l in range(8))
        assert g_fwd >= GUARD * fwd_allow and g_bwd >= GUARD * bwd_allow, (mlp, g_fwd, g_bwd)
        assert s["guard_rgbs_sigma"] >= GUARD, (mlp, s["guard_rgbs_sigma"])
        if "pe" in out["alt"]:
            assert s["guard_posenc_sin"] >= GUARD * sin_bar, (mlp, s["guard_posenc_sin"])
    if dens == "softplus":
        for k, r in out["rays"].items():
            if k.startswith("level"):
                assert r["relu_factor_guard"] >= GUARD * GW_BAR, (k, r)
    inf = out["inference"]
    for k, val in inf.items():
        if k.endswith("mismatches"):
            assert val == 0, (k, inf)
    assert inf.get("cells_S32_err_over_bound", 0.0) <= 1.0, inf
    if x3:
        assert inf["x3_points_excess"] <= X3_ALLOW and inf["x3_grid_excess"] <= X3_ALLOW, inf


@pytest.mark.gpu
@pytest.mark.parametrize("row", MATRIX, ids=_tag)
def test_flag_matrix_row(row):
    out = _check_row(row)
    _record(_tag(row), out)
    _assert_row(row, out)


@pytest.mark.gpu
def test_graph_replay_with_every_flag_non_default():
    """GraphedTrainStep at fp16x3 with an elu trunk, a (2, 8, legacy) encoder, the softplus density, SH degree 2 and
    a black background reproduces three eager train_steps bit for bit: parameters and Adam moments (the narrow
    encoder's pob_adam_update_pe and operand repack inside the graph)"""
    from plenoctree_b200.nerf import train as T
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf.rays import random_rays_np
    from tests.support.mlp_stages import _centre_sigma, params
    pe, sh, R = (2, 8, True), 2, 256
    fc, ff = params(sh, 33, pe)
    for f in (fc, ff):
        _centre_sigma(f, sh, "elu", pe)
    o, d, v, px = random_rays_np(R, 33)
    b12 = torch.from_numpy(np.concatenate([o, d, v, px], axis=1)).cuda()
    lrs = [5e-4, 4e-4, 3e-4]
    outs = []
    for graphed in (False, True):
        model = NerfModel(sh_deg=sh, max_rays=R, sparsity_npoints=1000, white_bkgd=False, net_activation="elu",
                          sigma_activation="softplus", min_deg_point=pe[0], max_deg_point=pe[1],
                          legacy_posenc_order=pe[2])
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
        assert torch.isfinite(a).all() and torch.equal(a, b), name
    assert not torch.equal(outs[0][0], torch.from_numpy(np.concatenate([fc, ff])).cuda())

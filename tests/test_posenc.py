"""NeRF-SH models with the reference's point-encoder flags min_deg_point, max_deg_point and legacy_posenc_order
(nerf_sh/nerf/utils.py:119-124,155-159): posenc(x, min_deg, max_deg, legacy) of width W = 3 + 6 (max - min) in the
kernels' posenc tile, Dense_0 [W, 256] and Dense_5 [256 + W, 256] in the flat layout, the C ABI's pob_posenc
descriptor, the host model, checkpoints and CLIs.

CPU: the oracle (oracle/posenc_oracle.py) against the executed reference (tests/golden/ref_posenc.npz, written by
tests/golden/make_golden_posenc.py), the checkpoint bridge, the flag scope, initialisation and the ABI tables.
GPU: the training stages of each encoder against fp64 built from the kernels' own saved tiles
(tests/support/mlp_stages.py: check_level), the evaluators against the training forward, legacy against standard order, the default
encoder against the parent's entry points, and the CLI chain with a non-default encoder."""
import ctypes
import functools
import os

import numpy as np
import pytest
import torch

from oracle import nerf_sh_oracle as O
from oracle import posenc_oracle as PO
from plenoctree_b200 import layouts as L
from tests.support.mlp_stages import FP16, assert_stages, check_call, params
from tests.support.model_flags import _scope_args
from tests.support.records import record

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "ref_posenc.npz")

# encoders of the golden file, and the ones the GPU tests run (the default first)
VARIANTS = [(0, 10, True), (2, 8, False), (2, 8, True), (0, 0, False), (3, 10, False)]
GPU_VARIANTS = [(0, 10, False), (0, 8, False), (0, 10, True), (2, 8, True), (0, 0, False), (3, 10, False),
                (10, 10, False), (9, 10, True)]


def _tag(pe):
    return f"{pe[0]}_{pe[1]}_{'legacy' if pe[2] else 'std'}"


def _g():
    return np.load(GOLDEN)


# =====================================================================================================================
# CPU
# =====================================================================================================================
def test_golden_covers_the_variants():
    g = _g()
    assert [tuple(int(a) for a in v[:2]) + (bool(v[2]),) for v in g["variants"]] == VARIANTS
    for pe in VARIANTS:
        assert g[f"jax_enc_{_tag(pe)}"].shape == (64, PO.width(pe))


@pytest.mark.parametrize("pe", VARIANTS, ids=_tag)
def test_oracle_posenc_matches_reference(pe):
    """the oracle's posenc against the reference's JAX posenc and its torch twin, executed with the same flags"""
    g = _g()
    x = torch.from_numpy(g["x"])
    enc = PO.encode(x, pe).numpy()
    np.testing.assert_array_equal(enc, g[f"torch_enc_{_tag(pe)}"])
    np.testing.assert_allclose(enc, g[f"jax_enc_{_tag(pe)}"], rtol=0, atol=2e-6)
    # the feature table the kernel implements (mlp_fwd.cu: posenc_row) names every column
    idx = PO.feature_index(pe)
    assert len(idx) == PO.width(pe) == L.posenc_width(pe)
    for col, (kind, j, c) in enumerate(idx):
        if kind == "x":
            np.testing.assert_array_equal(enc[:, col], g["x"][:, c])
        else:
            xb = x[:, c] * float(2 ** j)
            ref = torch.sin((xb if kind == "sin" else xb + np.float32(np.pi / 2)).double())
            assert float((torch.from_numpy(enc[:, col]).double() - ref).abs().max()) < 1e-5, (col, kind, j, c)


def test_oracle_default_is_the_fixed_oracle():
    x = torch.from_numpy(_g()["x"])
    np.testing.assert_array_equal(PO.encode(x).numpy(), O.posenc(x).numpy())
    assert PO.layer_dims(3) == O.layer_dims(3) and PO.param_count(4) == O.param_count(4)
    np.testing.assert_array_equal(PO.init_flat_params(3, 5, 0.1), O.init_flat_params(3, 5, 0.1))


def _flats(pe, g):
    k = VARIANTS.index(pe)
    return [PO.init_flat_params(int(g["sh_deg"]), 9100 + 10 * k + m, bias_scale=0.05, pe=pe) for m in range(2)]


@pytest.mark.parametrize("pe", VARIANTS, ids=_tag)
def test_oracle_forward_matches_reference(pe):
    """NerfModel.__call__ (JAX, over the numpy stand-ins) and the torch twin's eval_points_raw with the same weights"""
    g = _g()
    sh = int(g["sh_deg"])
    fc, ff = _flats(pe, g)
    pc, pf = PO.unflatten(fc, sh, pe), PO.unflatten(ff, sh, pe)
    rays = tuple(torch.from_numpy(g[k]) for k in ("origins", "directions", "viewdirs"))
    with torch.no_grad():
        ret = PO.nerf_forward(pc, pf, sh, rays, 32, 32, 2.0, 6.0, True, pe=pe)
    for lvl, (rgb, disp, acc) in zip(("coarse", "fine"), ret):
        # test_sigma_activation.py's tolerances: the fine level inherits the resampled depths' fp32 differences
        tol = 2e-5 if lvl == "coarse" else 5e-4
        np.testing.assert_allclose(rgb.numpy(), g[f"call_{_tag(pe)}_{lvl}_rgb"], rtol=0, atol=tol)
        np.testing.assert_allclose(acc.numpy(), g[f"call_{_tag(pe)}_{lvl}_acc"], rtol=0, atol=tol)
        np.testing.assert_allclose(disp.numpy(), g[f"call_{_tag(pe)}_{lvl}_disp"], rtol=20 * tol)
    if pe[0] != pe[1]:
        # the golden pins the feature order: the other order misses the coarse level by far
        other = (pe[0], pe[1], not pe[2])
        with torch.no_grad():
            wrong = PO.nerf_forward(pc, pf, sh, rays, 32, 32, 2.0, 6.0, True, pe=other)
        assert float(np.abs(wrong[0][0].numpy() - g[f"call_{_tag(pe)}_coarse_rgb"]).max()) > 20 * 2e-5
    with torch.no_grad():
        rgb, sig = PO.eval_points_raw(pf, torch.from_numpy(g["points"]), pe)
    np.testing.assert_allclose(rgb.numpy(), g[f"twin_raw_rgb_{_tag(pe)}"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(sig.numpy(), g[f"twin_raw_sigma_{_tag(pe)}"], rtol=0, atol=2e-5)


def test_reference_restores_a_checkpoint_written_here():
    """the torch twin's restore_model_state_from_jaxnerf loaded a flax checkpoint of a (2, 8, legacy) model written by
    plenoctree_b200.nerf.checkpoints: its eval_points_raw is the oracle's with the same weights"""
    g = _g()
    pe = tuple(int(a) for a in g["ckpt_variant"][:2]) + (bool(g["ckpt_variant"][2]),)
    sh = int(g["sh_deg"])
    fc, ff = _flats(pe, g)
    W = PO.width(pe)
    assert tuple(g["ckpt_dense0_shape"]) == (256, W) and tuple(g["ckpt_dense5_shape"]) == (256, 256 + W)
    pts = torch.from_numpy(g["points"])
    for flat, lvl in ((ff, "fine"), (fc, "coarse")):
        with torch.no_grad():
            rgb, sig = PO.eval_points_raw(PO.unflatten(flat, sh, pe), pts, pe)
        np.testing.assert_allclose(rgb.numpy(), g[f"ckpt_raw_rgb_{lvl}"], rtol=0, atol=2e-5)
        np.testing.assert_allclose(sig.numpy(), g[f"ckpt_raw_sigma_{lvl}"], rtol=0, atol=2e-5)


@pytest.mark.parametrize("pe", [(2, 8, True), (0, 0, False), (3, 10, False), (0, 10, False)], ids=_tag)
def test_checkpoint_round_trips_are_exact(pe, tmp_path):
    from plenoctree_b200.nerf import checkpoints as C
    sh = 3
    flat = np.concatenate([PO.init_flat_params(sh, 31, 0.1, pe), PO.init_flat_params(sh, 32, 0.1, pe)])
    assert C.param_count(sh, pe) == PO.param_count(sh, pe) == flat.size // 2
    tree = C.flat_to_flax_params(flat, sh, pe)
    assert tree["MLP_0"]["Dense_0"]["kernel"].shape == (PO.width(pe), 256)
    assert tree["MLP_1"]["Dense_5"]["kernel"].shape == (256 + PO.width(pe), 256)
    np.testing.assert_array_equal(C.flax_params_to_flat(tree, sh, pe), flat)
    np.testing.assert_array_equal(C.torch_state_dict_to_flat(C.flat_to_torch_state_dict(flat, sh, pe), sh, pe), flat)
    m = flat * 0.5
    v = np.abs(flat)
    sd = C.msgpack_restore(C.msgpack_serialize(C.train_state_dict(flat, m, v, 7, sh, pe)))
    p2, m2, v2, step = C.state_dict_to_flat(sd, sh, pe)
    assert step == 7
    for a, b in ((p2, flat), (m2, m), (v2, v)):
        np.testing.assert_array_equal(a, b)
    if pe != (0, 10, False):
        with pytest.raises(ValueError, match="min_deg_point"):
            C.flax_params_to_flat(tree, sh)            # a checkpoint of another encoder is refused, and says why


def test_check_scope_table():
    from plenoctree_b200.nerf import flags as F
    for mn in range(11):
        for mx in range(mn, 11):
            for legacy in (False, True):
                F.check_scope(_scope_args(min_deg_point=mn, max_deg_point=mx, legacy_posenc_order=legacy))
    for mn, mx in ((0, 11), (-1, 10), (5, 4), (0, 16), (11, 11)):
        with pytest.raises(NotImplementedError, match="min_deg_point"):
            F.check_scope(_scope_args(min_deg_point=mn, max_deg_point=mx))
    for kw in (dict(net_depth=6), dict(net_width=128), dict(skip_layer=3), dict(use_viewdirs=True), dict(sg_dim=4),
               dict(net_activation="gelu"), dict(rgb_activation="relu"), dict(sigma_activation="elu")):
        with pytest.raises(NotImplementedError):
            F.check_scope(_scope_args(**kw))


def test_layout_glorot_and_weight_decay_follow_width():
    import math
    from plenoctree_b200.nerf.models import NerfModel, glorot_uniform_flat
    for pe in ((0, 10, False), (2, 8, True), (0, 0, False), (3, 10, False)):
        W = PO.width(pe)
        assert L.layer_dims(16, W) == PO.layer_dims(3, pe)
        assert L.flat_offsets(16, W)[2] == PO.param_count(3, pe)
        flat = glorot_uniform_flat(3, torch.Generator().manual_seed(1), pe)
        assert flat.numel() == PO.param_count(3, pe)
        for (w, _), (cin, cout) in zip(PO.unflatten(flat, 3, pe), PO.layer_dims(3, pe)):
            a = math.sqrt(6.0 / (cin + cout))
            assert float(w.abs().max()) <= a and float(w.abs().max()) > 0.9 * a, (pe, cin, cout)
        m = NerfModel(sh_deg=3, device="cpu", min_deg_point=pe[0], max_deg_point=pe[1], legacy_posenc_order=pe[2])
        # weight_l2 = sum(theta^2) / numel over both MLPs (nerf_sh/train.py weight_l2): the denominator follows W
        assert m.P == PO.param_count(3, pe) and m.params.numel() == 2 * PO.param_count(3, pe)
    # the default encoder draws the same initial parameters as before the flags existed
    g1, g2 = torch.Generator().manual_seed(5), torch.Generator().manual_seed(5)
    assert torch.equal(glorot_uniform_flat(3, g1), glorot_uniform_flat(3, g2, (0, 10, False)))
    with pytest.raises(ValueError):
        NerfModel(sh_deg=3, device="cpu", max_deg_point=11)


def test_pack_reference_posenc_rows():
    """rows [W, 63) of the posenc slots are zero and the Dense_0 / Dense_5 biases sit at posenc column 63"""
    for pe in ((2, 8, True), (0, 0, False)):
        W = PO.width(pe)
        flat = PO.init_flat_params(3, 3, 0.5, pe)
        pk = L.pack_reference(flat, 3, pe)
        w_off, b_off, _ = L.flat_offsets(16, W)
        r, c = np.meshgrid(np.arange(256), np.arange(32), indexing="ij")
        off = L.w_slot_offset(r, c) // 2

        def slot(i):
            return pk["w_hi"].view(np.float16)[i * 8192:(i + 1) * 8192][off].astype(np.float32)  # [out, k]
        s0 = np.concatenate([slot(0), slot(1)], 1)                 # layer 0: posenc columns 0..63
        k0 = flat[w_off[0]:w_off[0] + W * 256].reshape(W, 256)
        np.testing.assert_array_equal(s0[:, :W], k0.T.astype(np.float16).astype(np.float32))
        assert (s0[:, W:63] == 0).all()
        np.testing.assert_array_equal(s0[:, 63], flat[b_off[0]:b_off[0] + 256].astype(np.float16).astype(np.float32))
        first5 = 2 + 9 * 4                                         # layer 5's slots: 8 of h4, then 2 of posenc
        s5 = np.concatenate([slot(first5 + 8), slot(first5 + 9)], 1)
        k5 = flat[w_off[5]:w_off[5] + (256 + W) * 256].reshape(256 + W, 256)
        np.testing.assert_array_equal(s5[:, :W], k5[256:].T.astype(np.float16).astype(np.float32))
        assert (s5[:, W:63] == 0).all()


def test_abi_posenc_descriptor():
    from plenoctree_b200 import _lib
    lib = _lib.lib
    hdr = open(os.path.join(os.path.dirname(HERE), "include", "plenoctree_b200.h")).read()
    assert "typedef struct pob_posenc {" in hdr and "const pob_posenc* posenc;" in hdr
    assert [f[0] for f in _lib.NetDesc._fields_] == ["min_deg", "max_deg", "legacy_order", "net_activation"]
    assert _lib.RenderConfig._fields_[-1] == ("posenc", ctypes.c_void_p)
    assert _lib.RenderConfig(3, 64, 128, 1, 4096, 10000).posenc is None        # an unset descriptor is NULL
    for sh in (-1, 3, 4):
        assert lib.pob_param_count_pe(sh, None) == lib.pob_param_count(sh)
        d = _lib.NetDesc(0, 10, 0, 0)
        assert lib.pob_param_count_pe(sh, ctypes.addressof(d)) == lib.pob_param_count(sh)
        for pe in ((2, 8, 1), (0, 0, 0), (3, 10, 0), (10, 10, 1)):
            d = _lib.NetDesc(*pe, 0)
            assert lib.pob_param_count_pe(sh, ctypes.addressof(d)) == PO.param_count(sh, pe)
    for bad in ((0, 11, 0), (-1, 5, 0), (6, 5, 0), (0, 10, 2)):
        d = _lib.NetDesc(*bad, 0)
        assert lib.pob_param_count_pe(3, ctypes.addressof(d)) == -1
    assert _lib.posenc_struct((0, 10, False)) is None and _lib.posenc_struct(None) is None


def test_no_gpu_descriptor_calls_fail_loudly():
    if torch.cuda.is_available():
        return
    from plenoctree_b200 import _lib
    d = _lib.NetDesc(2, 8, 1, 0)
    rc = _lib.lib.pob_eval_points_raw_pe(1, 3, ctypes.addressof(d), 1, 16, None, 1, 1, None)
    assert rc != 0 and len(_lib.lib.pob_last_error()) > 0


# =====================================================================================================================
# GPU
# =====================================================================================================================


def _model(pe, sh=3, R=24, nc=32, nf=64, nsp=64, seed=17):
    from plenoctree_b200.nerf.models import NerfModel
    m = NerfModel(sh_deg=sh, num_coarse_samples=nc, num_fine_samples=nf, max_rays=R, sparsity_npoints=nsp,
                  min_deg_point=pe[0], max_deg_point=pe[1], legacy_posenc_order=pe[2])
    fc, ff = params(sh, seed, pe)
    m.set_params(np.concatenate([fc, ff]) if nf else fc)
    return m


def _inputs(m, R, seed=17, sp_radius=1.5):
    from plenoctree_b200.nerf.rays import random_rays_np
    o, d, v, px = random_rays_np(R, seed)
    rs = np.random.RandomState(seed + 1)
    t_rand = rs.uniform(0, 1, size=(R, m.num_coarse_samples)).astype(np.float32)
    u = rs.uniform(0, 1, size=(R, m.num_fine_samples)).astype(np.float32) if m.num_fine_samples else None
    sp = rs.uniform(-sp_radius, sp_radius, size=(m.sparsity_npoints, 3)).astype(np.float32) \
        if m.sparsity_npoints else None
    return (o, d, v, px), t_rand, u, sp


def _train_call(m, R, fill=0xFF, precision=1, sp_radius=1.5):
    from plenoctree_b200.nerf import train as T
    from plenoctree_b200.nerf.models import Rays
    (o, d, v, px), t_rand, u, sp = _inputs(m, R, sp_radius=sp_radius)
    state = T.TrainState(m)
    if fill is not None:
        m.workspace(True, precision).fill_(fill)
    T.loss_and_grad(m, state, {"rays": Rays(o, d, v), "pixels": px}, sparsity_weight=0.1 if sp is not None else 0.0,
                    sparsity_length=0.05, randomized=True, t_rand=t_rand, u=u, sp_points=sp, precision=precision)
    torch.cuda.synchronize()
    return state, dict(rays=(o, d, v), px=px, t_rand=t_rand, u=u, sp=sp, n=R)


def _oracle_grad(m, ctx, pe, sh, precision=1):
    """fp64 oracle gradient of the call in ctx, with the fine-level depths the GPU used (sample_pdf in fp64 would place
    a few of them elsewhere)"""
    views = L.train_workspace_views(m.cfg, ctx["n"], ctx["sp"] is not None, precision=precision)
    z_fine = L.workspace_view(m.workspace(True, precision), views["levels"][1], "z").cpu().numpy()
    cfg = dict(num_coarse_samples=m.num_coarse_samples, num_fine_samples=m.num_fine_samples, near=2.0, far=6.0,
               white_bkgd=True, sparsity_weight=0.1, sparsity_length=0.05)
    P = m.P
    _, gc, gf = PO.loss_and_grads(m.params[:P].cpu().numpy(), m.params[P:].cpu().numpy(), sh, ctx["rays"], ctx["px"],
                                  cfg, ctx["t_rand"], ctx["u"], ctx["sp"], z_fine=z_fine, pe=pe)
    return np.concatenate([gc, gf])


_record = functools.partial(record, "posenc.json")


@pytest.mark.gpu
@pytest.mark.parametrize("pe", GPU_VARIANTS, ids=_tag)
def test_train_stages_posenc(pe):
    """stages of every level against fp64 built from the kernels' own saved tiles (mlp_stages.check_level with the
    encoder), then the compact flat gradient against the fp64 oracle of the encoder (test_train.py's gate)"""
    sh, R = 3, 24
    m = _model(pe, sh, R)
    state, ctx = _train_call(m, R)
    res = check_call(m, state, ctx, FP16)
    g = state.grads.double().cpu().numpy()
    ref = _oracle_grad(m, ctx, pe, sh)
    st = dict(stages=res, grad_rel_l2=float(np.linalg.norm(g - ref) / np.linalg.norm(ref)),
              grad_cosine=float(np.dot(g, ref) / (np.linalg.norm(g) * np.linalg.norm(ref))))
    _record(f"stages_{_tag(pe)}", st)
    assert_stages(res, FP16, "relu", guard=False)
    assert st["grad_rel_l2"] < 2e-2 and st["grad_cosine"] > 0.9995, st


def _eval_points_at_training_rows(m, ctx, lv, ws):
    """the sample points of one training level, formed like the kernel's load_point, and their view directions"""
    dev = ws.device
    o, d, v = (torch.from_numpy(a).to(dev) for a in ctx["rays"])
    z = L.workspace_view(ws, lv, "z").reshape(-1)
    s = torch.arange(lv["M_rays"], device=dev)
    ray = s // lv["N"]
    return (o[ray] + z[s][:, None] * d[ray]).contiguous(), v[ray].contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize("pe", GPU_VARIANTS, ids=_tag)
def test_evaluators_match_the_training_forward(pe):
    """fp16: the render, point, grid and cell-mean forwards are bit-identical to the saving training forward; fp16x3:
    within the fp16x3 bound of an fp64 evaluation"""
    from plenoctree_b200 import ops
    from plenoctree_b200.nerf.models import Rays
    sh, R = 3, 24
    m = _model(pe, sh, R, nsp=0)
    state, ctx = _train_call(m, R)
    ws = m.workspace(True)
    views = L.train_workspace_views(m.cfg, R, False)
    # render: the same draws give the same per-sample rgbs on both levels
    o, d, v = ctx["rays"]
    m.workspace(False).fill_(0xFF)
    m(Rays(o, d, v), t_rand=ctx["t_rand"], u=ctx["u"])
    torch.cuda.synchronize()
    wr = m.workspace(False)
    rviews = L.train_workspace_views(m.cfg, R, False, training=False)
    for lv, rv in zip(views["levels"], rviews["levels"]):
        a = L.workspace_view(ws, lv, "rgbs")[:lv["M_rays"]]
        b = L.workspace_view(wr, rv, "rgbs")[:rv["M_rays"]]
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), _tag(pe)
    # points: eval_points / eval_points_raw at the fine level's sample points
    lv = views["levels"][-1]
    pts, vd = _eval_points_at_training_rows(m, ctx, lv, ws)
    train_rgbs = L.workspace_view(ws, lv, "rgbs")[:lv["M_rays"]]
    rgb, sig = m.eval_points(pts, vd)
    assert torch.equal(torch.cat([rgb, sig], 1).view(torch.int32), train_rgbs.view(torch.int32))
    raw_rgb, raw_sig = m.eval_points_raw(pts)
    assert torch.equal(raw_sig.clamp_min(0)[:, 0], train_rgbs[:, 3])
    # cells: one sample per cell is the raw output itself
    cells = ops.eval_cells_mean(m.blobs[1], sh, pts, 1, posenc=m.posenc)
    assert torch.equal(cells, torch.cat([raw_rgb, raw_sig], 1))
    # grid: the voxel centres, formed like load_point, through eval_points_raw
    reso, off, scl = 16, (0.5, 0.5, 0.5), (0.5, 0.5, 0.5)    # power-of-two scale: torch divides by a reciprocal
    grgb, gsig = ops.eval_grid(m.blobs[1], sh, reso, off, scl, want_rgb=True, posenc=m.posenc)
    ii = (torch.arange(reso, device="cuda", dtype=torch.float32) + 0.5) * (1.0 / reso)
    gx, gy, gz = torch.meshgrid(ii, ii, ii, indexing="ij")
    gp = torch.stack([(g.reshape(-1) - o_) / s_ for g, o_, s_ in zip((gx, gy, gz), off, scl)], 1).contiguous()
    prgb, psig = m.eval_points_raw(gp)
    assert torch.equal(grgb, prgb) and torch.equal(gsig, psig[:, 0])
    # fp16x3 against fp64
    rgb3, sig3 = m.eval_points_raw(pts, precision=ops.PREC_FP16X3)
    with torch.no_grad():
        params = PO.unflatten(torch.from_numpy(m.params[m.P:].cpu().numpy()).double(), sh, pe)
        ref_rgb, ref_sig = PO.eval_points_raw(params, pts.cpu().double(), pe)
    err = max(float((rgb3.cpu().double() - ref_rgb).abs().max() / ref_rgb.abs().max()),
              float((sig3.cpu().double() - ref_sig).abs().max() / ref_sig.abs().max()))
    _record(f"eval_x3_rel_{_tag(pe)}", err)
    assert err < 1e-4, err


@pytest.mark.gpu
@pytest.mark.parametrize("degs", [(0, 10), (2, 8)])
def test_legacy_matches_permuted_standard(degs):
    """a legacy-order model and a standard-order model whose Dense_0 / Dense_5 rows are permuted to match compute the
    same network: equal within fp16 operand rounding (the K reduction runs in another order)"""
    from plenoctree_b200.nerf.models import NerfModel
    sh = 3
    leg, std = degs + (True,), degs + (False,)
    fl = np.concatenate(params(sh, 41, leg))
    P = PO.param_count(sh, leg)
    fs = np.concatenate([PO.permute_rows(fl[:P], sh, leg, std), PO.permute_rows(fl[P:], sh, leg, std)])
    ml = NerfModel(sh_deg=sh, max_rays=64, min_deg_point=degs[0], max_deg_point=degs[1], legacy_posenc_order=True)
    ms = NerfModel(sh_deg=sh, max_rays=64, min_deg_point=degs[0], max_deg_point=degs[1])
    ml.set_params(fl)
    ms.set_params(fs)
    pts = torch.from_numpy(np.random.RandomState(5).uniform(-1.5, 1.5, (4096, 3)).astype(np.float32)).cuda()
    with torch.no_grad():
        ref_rgb, ref_sig = PO.eval_points_raw(PO.unflatten(torch.from_numpy(fl[P:]).double(), sh, leg),
                                              pts.cpu().double(), leg)
    a_rgb, a_sig = ml.eval_points_raw(pts)
    b_rgb, b_sig = ms.eval_points_raw(pts)
    # both within fp16 rounding of the same fp64 network, and of each other
    for got, ref in ((a_rgb, ref_rgb), (b_rgb, ref_rgb), (a_sig, ref_sig), (b_sig, ref_sig)):
        assert float((got.cpu().double() - ref).abs().max() / ref.abs().max()) < 5e-3
    d = max(float((a_rgb - b_rgb).abs().max() / b_rgb.abs().max()), float((a_sig - b_sig).abs().max() / b_sig.abs().max()))
    _record(f"legacy_vs_permuted_{degs}", d)
    assert d < 5e-3, d


@pytest.mark.gpu
def test_explicit_default_descriptor_is_the_null_descriptor():
    """every entry point with an explicit (0, 10, 0) descriptor gives bit-identical results to NULL"""
    from plenoctree_b200 import _lib
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    sh, R = 3, 24
    d = _lib.NetDesc(0, 10, 0, 0)
    dp = ctypes.addressof(d)
    flat = torch.from_numpy(np.concatenate(params(sh, 3, (0, 10, False)))).cuda()
    P = flat.numel() // 2
    nb = int(lib.pob_packed_bytes(sh))
    b0, b1 = torch.zeros(nb, dtype=torch.uint8, device="cuda"), torch.full((nb,), 7, dtype=torch.uint8, device="cuda")
    check(lib.pob_pack_weights(ptr(flat[:P]), sh, ptr(b0), stream_ptr()))
    check(lib.pob_pack_weights_pe(ptr(flat[:P]), sh, dp, ptr(b1), stream_ptr()))
    assert torch.equal(b0, b1)
    pts = torch.from_numpy(np.random.RandomState(1).uniform(-2, 2, (5000, 3)).astype(np.float32)).cuda()
    vd = torch.nn.functional.normalize(pts, dim=1).contiguous()
    for prec in (1, 3):
        a = torch.empty(5000, 48, device="cuda"), torch.empty(5000, device="cuda")
        b = torch.empty(5000, 48, device="cuda"), torch.empty(5000, device="cuda")
        check(lib.pob_eval_points_raw(ptr(b0), sh, ptr(pts), 5000, ptr(a[0]), ptr(a[1]), prec, stream_ptr()))
        check(lib.pob_eval_points_raw_pe(ptr(b0), sh, dp, ptr(pts), 5000, ptr(b[0]), ptr(b[1]), prec, stream_ptr()))
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        x, y = torch.empty(5000, 4, device="cuda"), torch.empty(5000, 4, device="cuda")
        check(lib.pob_eval_points(ptr(b0), sh, ptr(pts), ptr(vd), 5000, ptr(x), prec, stream_ptr()))
        check(lib.pob_eval_points_pe(ptr(b0), sh, dp, ptr(pts), ptr(vd), 5000, ptr(y), 0, prec, stream_ptr()))
        assert torch.equal(x, y)
        off = (ctypes.c_float * 3)(0.5, 0.5, 0.5)
        scl = (ctypes.c_float * 3)(0.4, 0.4, 0.4)
        g1, g2 = torch.empty(8 * 16 * 16, device="cuda"), torch.empty(8 * 16 * 16, device="cuda")
        check(lib.pob_eval_grid(ptr(b0), sh, 16, 4, 8, 16, 16, off, scl, None, ptr(g1), prec, stream_ptr()))
        check(lib.pob_eval_grid_pe(ptr(b0), sh, dp, 16, 4, 8, 16, 16, off, scl, None, ptr(g2), prec, stream_ptr()))
        assert torch.equal(g1, g2)
        c1, c2 = torch.empty(1000, 49, device="cuda"), torch.empty(1000, 49, device="cuda")
        check(lib.pob_eval_cells_mean(ptr(b0), sh, ptr(pts), 1000, 5, ptr(c1), prec, stream_ptr()))
        check(lib.pob_eval_cells_mean_pe(ptr(b0), sh, dp, ptr(pts), 1000, 5, ptr(c2), prec, stream_ptr()))
        assert torch.equal(c1, c2)
        h1, h2 = np.empty(5000, np.float32), np.empty(5000, np.float32)
        pts_h = pts.cpu().numpy()
        check(lib.pob_eval_points_raw_host(ptr(b0), sh, ptr(pts_h), 5000, None, ptr(h1), prec))
        check(lib.pob_eval_points_raw_host_pe(ptr(b0), sh, dp, ptr(pts_h), 5000, None, ptr(h2), prec))
        np.testing.assert_array_equal(h1, h2)
    # the training step and Adam with cfg.posenc NULL and explicit
    grads = []
    for explicit in (False, True):
        m = _model((0, 10, False), sh, R, seed=3)
        if explicit:
            m.cfg.posenc = dp
        state, _ = _train_call(m, R)
        check(lib.pob_adam_update_pe(sh, dp if explicit else None, 2, ptr(m.params), ptr(state.grads), ptr(state.m),
                                     ptr(state.v), 1e-3, 0.0, None, 1.0, 0.0, ptr(m.blobs[0]), ptr(m.blobs[1]),
                                     stream_ptr()))
        torch.cuda.synchronize()
        grads.append((state.grads.clone(), m.params.clone(), m.blobs[1].clone()))
    for a, b in zip(*grads):
        assert torch.equal(a, b)
    # a refused descriptor fails loudly at the boundary
    bad = _lib.NetDesc(0, 11, 0, 0)
    assert lib.pob_eval_points_raw_pe(ptr(b0), sh, ctypes.addressof(bad), ptr(pts), 16, None, ptr(g1), 1,
                                      stream_ptr()) != 0
    assert b"max_deg" in lib.pob_last_error()


@pytest.mark.gpu
def test_x3_training_with_posenc():
    """the fp16x3 training step with a narrower legacy encoder reaches the fp64 oracle's gradient closely"""
    pe, sh, R = (2, 8, True), 3, 24
    m = _model(pe, sh, R)
    state, ctx = _train_call(m, R, precision=3)
    g = state.grads.double().cpu().numpy()
    ref = _oracle_grad(m, ctx, pe, sh, precision=3)
    rel = float(np.linalg.norm(g - ref) / np.linalg.norm(ref))
    _record("x3_grad_rel_l2_2_8_legacy", rel)
    assert rel < 1e-3, rel


@pytest.mark.gpu
def test_cli_chain_with_posenc_flags(tmp_path):
    """nerf_sh.train with max_deg_point 8 and legacy_posenc_order learns a synthetic scene and its checkpoint reloads;
    nerf_sh.eval, octree.extraction, octree.optimization and octree.evaluation run on that model"""
    from tests.support.model_flags import _set_flags
    from plenoctree_b200.nerf import checkpoints as C, datasets as D
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf.utils import generate_rays, pose_spherical, render_image
    from plenoctree_b200.nerf_sh import eval as EV, train as TR
    from plenoctree_b200.octree import evaluation as OE, extraction as EX, optimization as OP
    sh_deg, W = 3, 48
    ft = np.concatenate([O.init_flat_params(sh_deg, 7001, bias_scale=0.05),
                         O.init_flat_params(sh_deg, 7002, bias_scale=0.05)])
    P = O.param_count(sh_deg)
    for mm in range(2):
        off = mm * P + P - 48 - 1 - 256 * 48 - 256
        ft[off:off + 256] *= 30.0
    teacher = NerfModel(sh_deg=sh_deg, max_rays=4096)
    teacher.set_params(ft)
    cam_x = 0.6911112070083618
    focal = 0.5 * W / np.tan(0.5 * cam_x)
    rs = np.random.RandomState(3)
    splits = {"train": 8, "val": 2, "test": 2}
    poses = {k: [pose_spherical(rs.uniform(-180, 180), rs.uniform(-80, -10), 4.0) for _ in range(n)]
             for k, n in splits.items()}
    images = {}
    for k in splits:
        rays = generate_rays(W, W, focal, np.stack(poses[k]))
        images[k] = [render_image(teacher, Rays(rays.origins[i], rays.directions[i], rays.viewdirs[i]))[0].cpu().numpy()
                     for i in range(splits[k])]
    data_dir, train_dir = str(tmp_path / "scene"), str(tmp_path / "ckpt")
    D.write_blender_scene(data_dir, images, poses, cam_x)
    (tmp_path / "cfg.yaml").write_text("dataset: blender\nfactor: 0\nnum_coarse_samples: 64\nnum_fine_samples: 128\n"
                                       "use_viewdirs: false\nwhite_bkgd: true\nbatch_size: 1024\nsh_deg: 3\n"
                                       "randomized: true\nmax_steps: 300\nmax_deg_point: 8\n"
                                       "legacy_posenc_order: true\n")
    EX._define_cli_flags()
    OP._define_cli_flags()
    FLAGS = _set_flags(train_dir=train_dir, data_dir=data_dir, config=str(tmp_path / "cfg"), save_every=300,
                       print_every=100, render_every=0, sparsity_npoints=1000, lr_init=2e-3, lr_final=2e-4, chunk=4096,
                       noise_std=None, image_batching=True)
    saved = {k: getattr(FLAGS, k) for k in ("is_jaxnerf_ckpt", "init_grid_depth", "samples_per_cell", "masking_mode",
                                             "alpha_thresh", "renderer_step_size", "radius", "output", "eval",
                                             "input", "num_epochs", "val_interval", "lr", "continue_on_decrease")}
    try:
        model, state = TR.main(None)
        assert model.posenc == (0, 8, True) and model.P == PO.param_count(sh_deg, (0, 8, True))
        assert os.path.exists(os.path.join(train_dir, "checkpoint_300")) and state.step == 300
        psnr, _ = EV.main(None)
        fresh = NerfModel(sh_deg=sh_deg, max_rays=4096, max_deg_point=8, legacy_posenc_order=True)
        fresh.init_params(20200823)
        rays = generate_rays(W, W, focal, np.stack(poses["test"]))
        gt = torch.from_numpy(images["test"][0]).cuda()
        r0 = Rays(rays.origins[0], rays.directions[0], rays.viewdirs[0])
        p_init = -10 * np.log10(float(((render_image(fresh, r0)[0] - gt) ** 2).mean()))
        assert psnr > p_init + 2.0, (p_init, psnr)
        # the checkpoint reloads into a model of the same encoder, and is refused by one of the default encoder
        again = NerfModel(sh_deg=sh_deg, max_rays=4096, max_deg_point=8, legacy_posenc_order=True)
        assert C.restore_checkpoint(train_dir, again) == 300
        assert torch.equal(again.params, model.params)
        with pytest.raises(ValueError, match="min_deg_point"):
            C.restore_checkpoint(train_dir, NerfModel(sh_deg=sh_deg, max_rays=64))
        # octree.extraction / optimization / evaluation on the flax checkpoint
        FLAGS.is_jaxnerf_ckpt = True
        FLAGS.init_grid_depth = 5
        FLAGS.samples_per_cell = 8
        FLAGS.masking_mode = "sigma"
        FLAGS.alpha_thresh = 0.01
        FLAGS.renderer_step_size = 1e-3
        FLAGS.radius = "1.5"
        FLAGS.output = str(tmp_path / "tree.npz")
        FLAGS.eval = False
        tree = EX.main(None)
        assert os.path.exists(FLAGS.output) and tree.max_depth == 5
        test_ds = D.get_dataset("test", FLAGS, device="cuda")
        p_tree, s_tree = OE.eval_octree(tree, test_ds, FLAGS)
        assert p_tree > p_init + 1.0 and np.isfinite(s_tree), (p_init, psnr, p_tree)
        FLAGS.input = FLAGS.output
        FLAGS.output = str(tmp_path / "tree_opt.npz")
        FLAGS.num_epochs = 2
        FLAGS.val_interval = 1
        FLAGS.lr = 1e7 * (W * W) / (800.0 * 800.0) / 4
        FLAGS.continue_on_decrease = True
        OP.main(None)
        _record("cli_chain_0_8_legacy", dict(psnr_init=p_init, psnr_300=psnr, psnr_tree=p_tree))
    finally:
        FLAGS.config = None
        FLAGS.min_deg_point, FLAGS.max_deg_point, FLAGS.legacy_posenc_order = 0, 10, False
        for k, v in saved.items():
            setattr(FLAGS, k, v)

"""Trunk activations of the flag net_activation (elu, softplus, tanh besides relu) through every layer: the oracle
against the executed reference (tests/golden/ref_net_activation.npz from tests/golden/make_golden_net_activation.py),
the flag's scope, the C ABI descriptor and, on the GPU, the training kernels stage by stage, the inference forwards,
the whole gradient and the command-line chain.

The stage checks follow test_train_stages.py / test_train_x3.py: every stage is compared with an fp64 evaluation whose
inputs are the kernels' own saved tiles.  The forward bar adds f's fp32 error (4 * 2^-24 * |f(z)|, kernels.h) to the
existing allowance: f is 1-Lipschitz, so the pre-activation's fp32 accumulation error passes through it unamplified.
The data gradient is held to fp64 dH_l * f'(h_l), with f' formed in fp64 from the kernel's saved h_l.
"""
import ctypes
import functools
import os

import numpy as np
import pytest
import torch

from plenoctree_b200 import layouts as L
from oracle import net_activation_oracle as NA
from tests.support.mlp_stages import BWD_ALLOW, CASES, FP16, X3, Case, _centre_sigma, operands, stage_case
from tests.support.model_flags import _act64, _scope_args
from tests.support.records import record

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ACTS = ("elu", "softplus", "tanh")
# weight-gradient kernels in the production step, max |err| / sum |a b| per tensor: a smooth trunk's h_l are dense
# (relu leaves about half of them 0), and the error of an fp32 accumulator grows with its count of sequential MMA
# additions, ~12 000 per fine-level accumulator there (~1 560 tiles per CTA x 8 k16 steps): a worst case of
# 12 000 * 2^-24 = 7.2e-4.  test_train_stages.py's 1e-4 was measured on relu; the other cases keep it.
WG_EPS_W_PRODUCTION = 1e-3
# fp16x3 whole gradient of a softplus trunk against fp64, relative L2 (test_gradient_vs_fp64_oracle): [1.0e-4, against
# the fp32 oracle's 6.1e-6 and the fp16 step's 5.9e-3]
SOFTPLUS_X3_REL = 3e-4

_record = functools.partial(record, "parity_net_activation.json")


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


# =====================================================================================================================
# CPU: oracle, golden, scope, ABI
# =====================================================================================================================
def _golden():
    from oracle import nerf_sh_oracle as O
    g = np.load(os.path.join(HERE, "golden", "ref_net_activation.npz"))
    sh = int(g["sh_deg"])
    flats = []
    for s in g["seeds"]:
        f = O.init_flat_params(sh, int(s), bias_scale=0.05)
        off = 0
        for j, (a, b) in enumerate(O.layer_dims(sh)):
            if j < 8:
                f[off:off + a * b] *= float(g["trunk_scale"])
            elif j == 8:
                f[off:off + a * b] *= float(g["sigma_scale"])
            off += a * b + b
        flats.append(f)
    return g, sh, flats


def test_oracle_with_relu_is_the_oracle():
    """net_activation="relu" (either case) reproduces the oracle's default bit for bit: forward, loss and gradient"""
    from oracle import nerf_sh_oracle as O
    from tests.support.mlp_stages import _setup
    fc, ff, rays, px, t_rand, u, sp = _setup(2, 8, 32, 16, 5)
    cfg = dict(num_coarse_samples=64, num_fine_samples=32, near=2.0, far=6.0, white_bkgd=True, sparsity_weight=1e-2,
               sparsity_length=0.05, weight_decay_mult=0.1)
    base = O.loss_and_grads(fc, ff, 2, rays, px, cfg, t_rand, u, sp)
    for name in ("relu", "ReLU"):
        got = NA.loss_and_grads(fc, ff, 2, rays, px, cfg, t_rand, u, sp, net_activation=name)
        assert {k: v for k, v in got[0].items() if k != "_z_fine"} == {k: v for k, v in base[0].items() if k != "_z_fine"}
        np.testing.assert_array_equal(got[0]["_z_fine"], base[0]["_z_fine"])
        np.testing.assert_array_equal(got[1], base[1])
        np.testing.assert_array_equal(got[2], base[2])
    pts = _t(np.random.RandomState(1).uniform(-1.5, 1.5, size=(50, 3)).astype(np.float32))
    p = O.unflatten(fc, 2)
    for a, b in zip(O.eval_points_raw(p, pts), NA.eval_points_raw(p, pts, "relu")):
        assert torch.equal(a, b)


def test_golden_trunk_spans_both_signs():
    """the golden's trunk: every layer's pre-activations reach below -1 and above +1 for every activation, so the
    activations differ from relu (and from each other) on every layer"""
    from oracle import nerf_sh_oracle as O
    g, sh, flats = _golden()
    params = O.unflatten(flats[1], sh)
    x = O.posenc(_t(g["points"]))
    for act in ACTS:
        f = NA.NET_ACTIVATIONS[act]
        h, inputs = x, x
        for i in range(8):
            z = h @ params[i][0] + params[i][1]
            assert float(z.min()) < -1.0 and float(z.max()) > 1.0, (act, i, float(z.min()), float(z.max()))
            h = f(z)
            if i == 4:
                h = torch.cat([h, inputs], -1)


@pytest.mark.parametrize("act", ACTS)
def test_oracle_forward_matches_executed_reference(act):
    """NerfModel.__call__ with nn.elu / nn.softplus / nn.tanh, both levels, deterministic and with injected draws:
    the oracle within test_oracle.py's tolerances; with relu it misses them by far"""
    from oracle import nerf_sh_oracle as O
    g, sh, flats = _golden()
    pc, pf = (O.unflatten(f, sh) for f in flats)
    rays = (_t(g["origins"]), _t(g["directions"]), _t(g["viewdirs"]))
    worst_relu = 0.0
    for tag, t_rand, u in (("det", None, None), ("rand", _t(g["t_rand"]), _t(g["u"]))):
        for name in (act, "relu"):
            with torch.no_grad():
                ret = NA.nerf_forward(pc, pf, sh, rays, 64, 128, 2.0, 6.0, True, t_rand=t_rand, u=u,
                                     net_activation=name)
            for lvl, (rgb, disp, acc) in zip(("coarse", "fine"), ret):
                tol = 2e-5 if lvl == "coarse" else 5e-4
                want_rgb, want_acc = g[f"{act}_call_{tag}_{lvl}_rgb"], g[f"{act}_call_{tag}_{lvl}_acc"]
                if name == act:
                    np.testing.assert_allclose(rgb.numpy(), want_rgb, rtol=0, atol=tol)
                    np.testing.assert_allclose(acc.numpy(), want_acc, rtol=0, atol=tol)
                    want_disp = g[f"{act}_call_{tag}_{lvl}_disp"]
                    ok = np.isfinite(want_disp)
                    np.testing.assert_array_equal(np.isfinite(disp.numpy()), ok)
                    np.testing.assert_allclose(disp.numpy()[ok], want_disp[ok], rtol=20 * tol)
                else:
                    worst_relu = max(worst_relu, float(np.abs(rgb.numpy() - want_rgb).max()) / tol)
    assert worst_relu > 20.0, worst_relu


@pytest.mark.parametrize("act", ACTS)
def test_oracle_loss_matches_executed_reference(act):
    """train_step.loss_fn with the trunk activation, through both MLPs and the sparsity points (raw sigma of the fine
    MLP, which runs the same trunk): within 3e-4"""
    from oracle import nerf_sh_oracle as O
    g, sh, flats = _golden()
    pc, pf = (O.unflatten(f, sh) for f in flats)
    r = np.float32(g["sparsity_radius"])
    sp = (g["sp01"] * np.float32(r - (-r)) + np.float32(-r)).astype(np.float32)
    cfg = dict(num_coarse_samples=64, num_fine_samples=128, near=2.0, far=6.0, white_bkgd=True,
               sparsity_weight=float(g["sparsity_weight"]), sparsity_length=float(g["sparsity_length"]),
               weight_decay_mult=float(g["weight_decay_mult"]))
    rays = (_t(g["origins"]), _t(g["directions"]), _t(g["viewdirs"]))
    with torch.no_grad():
        total, st = NA.loss_fn(pc, pf, sh, rays, _t(g["pixels"]), cfg, _t(g["t_rand"]), _t(g["u"]), _t(sp),
                              net_activation=act)
    for k in ("loss", "loss_c", "loss_sp", "weight_l2", "psnr", "psnr_c"):
        want = float(g[f"{act}_{k}"])
        assert abs(float(st[k]) - want) <= 3e-4 * abs(want) + 1e-9, (act, k, float(st[k]), want)


@pytest.mark.parametrize("act", ACTS)
def test_oracle_matches_torch_twin(act):
    """the torch twin's eval_points_raw with torch.nn.ELU / Softplus / Tanh (both MLPs): within 2e-5"""
    from oracle import nerf_sh_oracle as O
    g, sh, flats = _golden()
    pts = _t(g["points"])
    for lvl, flat in (("coarse", flats[0]), ("fine", flats[1])):
        with torch.no_grad():
            rgb, sig = NA.eval_points_raw(O.unflatten(flat, sh), pts, act)
        np.testing.assert_allclose(rgb.numpy(), g[f"{act}_twin_raw_rgb_{lvl}"], rtol=0, atol=2e-5)
        np.testing.assert_allclose(sig.numpy(), g[f"{act}_twin_raw_sigma_{lvl}"], rtol=0, atol=2e-5 * max(
            1.0, float(np.abs(g[f"{act}_twin_raw_sigma_{lvl}"]).max())))


def test_reference_loader_reproduced():
    """the twin's restore_model_state_from_jaxnerf on a flax checkpoint written by nerf/checkpoints.py: this package's
    torch state_dict holds the same tensors, and the loaded twin's outputs are the oracle's with the activation (the
    checkpoint does not record it)"""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf import checkpoints as C
    g, sh, flats = _golden()
    flat = np.concatenate(flats)
    sd = C.flat_to_torch_state_dict(flat, sh)
    assert sorted(sd.keys()) == [str(k) for k in g["ckpt_state_keys"]]
    for k in ("MLP_0.input_layers.0.weight", "MLP_1.input_layers.5.weight", "MLP_1.rgb_layer.bias"):
        np.testing.assert_array_equal(np.asarray(sd[k])[:4], g["ckpt_sd_" + k.replace(".", "_")])
    pts = _t(g["points"])
    for act in ACTS:
        with torch.no_grad():
            rgb, sig = NA.eval_points_raw(O.unflatten(flats[1], sh), pts, act)
        np.testing.assert_allclose(rgb.numpy(), g[f"{act}_ckpt_raw_rgb_fine"], rtol=0, atol=2e-5)
        np.testing.assert_array_equal(g[f"{act}_ckpt_raw_rgb_fine"], g[f"{act}_twin_raw_rgb_fine"])


def test_check_scope_net_activation():
    """check_scope (every CLI's check) accepts the built trunk activations under both namings in any case, and
    refuses gelu / swish / silu with the pre-activation reason and other names as not built"""
    from plenoctree_b200.nerf import flags as F
    for names, code in ((("relu", "ReLU", "RELU"), 0), (("elu", "ELU", "Elu"), 1), (("softplus", "Softplus"), 2),
                        (("tanh", "Tanh", "TANH"), 3)):
        for name in names:
            F.check_scope(_scope_args(net_activation=name))
            F.check_scope(_scope_args(net_activation=name, sigma_activation="Softplus", rgb_activation="Sigmoid"))
            assert F.net_activation_code(name) == code
    for bad in ("gelu", "GELU", "swish", "silu", "SiLU"):
        with pytest.raises(NotImplementedError, match="pre-activation"):
            F.check_scope(_scope_args(net_activation=bad))
    for bad in ("sigmoid", "leaky_relu", "softmax", "relu6", "LeakyReLU"):
        with pytest.raises(NotImplementedError, match="not built"):
            F.check_scope(_scope_args(net_activation=bad))


def test_check_scope_other_flags_whatever_the_trunk():
    """every other flag is checked the same way whatever the trunk activation"""
    from plenoctree_b200.nerf import flags as F
    for net in ("relu", "elu", "Tanh"):
        for mn in range(11):
            for mx in range(mn, 11):
                F.check_scope(_scope_args(net_activation=net, min_deg_point=mn, max_deg_point=mx))
        for mn, mx in ((0, 11), (-1, 10), (5, 4), (0, 16), (11, 11)):
            with pytest.raises(NotImplementedError, match="min_deg_point"):
                F.check_scope(_scope_args(net_activation=net, min_deg_point=mn, max_deg_point=mx))
        for kw in (dict(net_depth=6), dict(net_width=128), dict(skip_layer=3), dict(use_viewdirs=True),
                   dict(sg_dim=4), dict(rgb_activation="relu"), dict(sigma_activation="elu"),
                   dict(sigma_activation="tanh")):
            with pytest.raises(NotImplementedError):
                F.check_scope(_scope_args(net_activation=net, **kw))
        with pytest.raises(ValueError, match="llff"):
            F.check_scope(_scope_args(net_activation=net, render_path=True))
    args = _scope_args(net_activation="ELU")
    F.check_scope(args)
    assert args.net_activation == "ELU"                    # the caller's flags are left as they are


def test_abi_net_descriptor():
    """the ctypes NetDesc is pob_posenc of the header, field for field; codes match; out-of-range codes are refused
    at the boundary"""
    import re
    from plenoctree_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "plenoctree_b200.h")).read()
    body = re.search(r"typedef struct pob_posenc \{(.*?)\} pob_posenc;", hdr, re.S).group(1)
    fields = re.findall(r"int (\w+);", body)
    assert fields == [f[0] for f in _lib.NetDesc._fields_]
    assert ctypes.sizeof(_lib.NetDesc) == 4 * len(fields) == 16
    for name in ("RELU", "ELU", "SOFTPLUS", "TANH"):
        m = re.search(rf"#define POB_NET_{name} (\d+)", hdr)
        assert int(m.group(1)) == getattr(_lib, f"NET_{name}")
    from plenoctree_b200.nerf import flags as F
    assert F.NET_ACTIVATIONS == {"relu": _lib.NET_RELU, "elu": _lib.NET_ELU, "softplus": _lib.NET_SOFTPLUS,
                                 "tanh": _lib.NET_TANH}
    lib = _lib.lib
    for code in range(4):
        d = _lib.NetDesc(0, 10, 0, code)
        assert lib.pob_param_count_pe(3, ctypes.addressof(d)) == lib.pob_param_count(3)    # layout unchanged
    for bad in (-1, 4, 100):
        d = _lib.NetDesc(0, 10, 0, bad)
        assert lib.pob_param_count_pe(3, ctypes.addressof(d)) == -1
        assert b"net_activation" in lib.pob_last_error()
    assert _lib.posenc_struct(None) is None and _lib.posenc_struct((0, 10, False), 0) is None
    s = _lib.posenc_struct(None, _lib.NET_TANH)
    assert (s.min_deg, s.max_deg, s.legacy_order, s.net_activation) == (0, 10, 0, 3)
    s = _lib.posenc_struct((2, 8, True), _lib.NET_ELU)
    assert (s.min_deg, s.max_deg, s.legacy_order, s.net_activation) == (2, 8, 1, 1)


def test_model_carries_the_activation_without_gpu_state():
    """get_model_state passes net_activation; checkpoints do not change (the flat layout is the relu model's)"""
    from plenoctree_b200.nerf import checkpoints as C
    from oracle import nerf_sh_oracle as O
    flat = O.init_flat_params(3, 3, bias_scale=0.05)
    assert C.param_count(3) == flat.size
    tree = C.flat_to_flax_params(np.concatenate([flat, flat]), 3)
    np.testing.assert_array_equal(C.flax_params_to_flat(tree, 3), np.concatenate([flat, flat]))


# =====================================================================================================================
# GPU
# =====================================================================================================================


def _stage_case(case, act, precision, wg_w_bar=None):
    tag = f"stages_{act}_{'fp16x3' if precision == X3 else 'fp16'}_"
    return stage_case(case.replace(act=act, precision=precision, centre=True),
                      lambda name, res: _record(tag + name, res), guard=False, wg_w_bar=wg_w_bar)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [1, X3], ids=["fp16", "fp16x3"])
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_net_activation_train_stages(case, act, precision):
    _stage_case(case, act, precision)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [1, X3], ids=["fp16", "fp16x3"])
@pytest.mark.parametrize("act", ACTS)
def test_net_activation_train_stages_production_step(act, precision):
    from plenoctree_b200._lib import RenderConfig, lib
    from plenoctree_b200.nerf.models import ctypes_ref
    need = int(lib.pob_train_workspace_bytes(ctypes_ref(RenderConfig(3, 64, 128, 1, 4096, 10000)), precision))
    free, _ = torch.cuda.mem_get_info()
    if free < need + (8 << 30):
        pytest.skip(f"needs {need / 2**30:.1f} GB of workspace + ~8 GB for the reference; {free / 2**30:.1f} GB free")
    _stage_case(Case(3, 4096, 64, 128, 10000), act, precision, wg_w_bar=WG_EPS_W_PRODUCTION)


@pytest.mark.gpu
@pytest.mark.parametrize("act", ACTS)
def test_relu_mask_mutation_fails_the_data_gradient_bar(act):
    """applying the relu mask of h_l in place of f'(h_l) misses the data-gradient bar by far"""
    res = _stage_case(Case(3, 96, 64, 128, 300), act, FP16)
    worst = min(r["stages"]["bwd_excess_relu_mask_mutation"] for k, r in res.items() if k.startswith("MLP"))
    _record(f"relu_mask_mutation_{act}", dict(min_excess=worst, bar=BWD_ALLOW[FP16]))
    assert worst > 10 * BWD_ALLOW[FP16], worst


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [1, X3], ids=["fp16", "fp16x3"])
def test_relu_code_is_bit_identical_to_null(precision):
    """an explicit descriptor with net_activation = 0 is the NULL descriptor, bit for bit: training workspace tiles,
    gradient, render rows, points, grid and cell means"""
    from plenoctree_b200 import _lib, ops
    from plenoctree_b200.nerf.models import Rays
    case = Case(3, 64, 64, 128, 200, precision=precision, centre=True)
    outs = []
    null_struct = ops.posenc_struct
    for explicit in (False, True):
        model = case.model()
        if explicit:
            model._posenc_struct = _lib.NetDesc(0, 10, 0, _lib.NET_RELU)
            model.cfg.posenc = ctypes.addressof(model._posenc_struct)
            # every ops call below passes an explicit {0, 10, 0, 0} descriptor instead of NULL
            ops.posenc_struct = lambda pe, net=0: _lib.NetDesc(0, 10, 0, int(net))
        try:
            state, ctx = case.run(model, fill=0xFF)
            ws = model.workspace(True, precision)
            views = L.train_workspace_views(model.cfg, ctx["n"], True, precision=precision)
            tiles = {f"{i}_{k}": L.workspace_view(ws, lv, k).clone() for i, lv in enumerate(views["levels"])
                     for k in ("H", "E", "DZ", "DO", "mask", "rgbs")}
            o, d, v = ctx["rays"]
            r = model(Rays(o, d, v), randomized=True, t_rand=ctx["t_rand"], u=ctx["u"], precision=precision)
            pts = torch.from_numpy(np.random.RandomState(3).uniform(-1.5, 1.5, (3000, 3)).astype(np.float32)).cuda()
            vd = torch.nn.functional.normalize(pts.flip(1), dim=1).contiguous()
            blob = model._blob(False)
            raw = ops.eval_points_raw(blob, 3, pts, precision=precision)
            rgbs = ops.eval_points(blob, 3, pts, vd, precision=precision)
            grid = ops.eval_grid(blob, 3, 32, (0.5, 0.5, 0.5), (0.4, 0.4, 0.4), want_rgb=True, precision=precision)
            cells = ops.eval_cells_mean(blob, 3, pts.reshape(-1, 6, 3).contiguous(), 6, precision=precision)
            torch.cuda.synchronize()
        finally:
            ops.posenc_struct = null_struct
        outs.append(dict(grad=state.grads.clone(), tiles=tiles, render=[t.clone() for lvl in r for t in lvl],
                         raw=raw, rgbs=rgbs, grid=grid, cells=cells))
    a, b = outs
    assert torch.equal(a["grad"], b["grad"])
    for k in a["tiles"]:
        assert torch.equal(a["tiles"][k], b["tiles"][k]), k
    for x, y in zip(a["render"], b["render"]):
        assert torch.equal(x, y)
    for k in ("raw", "rgbs", "grid"):
        for x, y in zip(a[k], b[k]):
            assert torch.equal(x, y), k
    assert torch.equal(a["cells"], b["cells"])


@pytest.mark.gpu
@pytest.mark.parametrize("act", ACTS)
def test_inference_forwards_match_training_rows(act):
    """fp16: render rows, eval_points, eval_points_raw (relu of raw sigma), the grid sweep and one-sample cell means
    are bit-identical to the training forward's rows at the same points.  fp16x3: render rows bit-identical to the x3
    training rows, and eval_points_raw within 1e-5 relative of an fp64 evaluation with the hi + lo operands."""
    from plenoctree_b200 import ops
    from plenoctree_b200.nerf.models import Rays
    case = Case(3, 64, 64, 128, 0, act=act, centre=True)
    rep = {}
    for precision in (1, X3):
        model = case.model()
        state, ctx = case.replace(precision=precision).run(model, fill=0xFF)
        ws = model.workspace(True, precision)
        views = L.train_workspace_views(model.cfg, ctx["n"], False, precision=precision)
        o, d, v = ctx["rays"]
        model(Rays(o, d, v), randomized=True, t_rand=ctx["t_rand"], u=ctx["u"], precision=precision)
        torch.cuda.synchronize()
        rws = model.workspace(False)
        rviews = L.train_workspace_views(model.cfg, ctx["n"], False, training=False)
        for i, (lv, rlv) in enumerate(zip(views["levels"], rviews["levels"])):
            Mr = lv["M_rays"]
            t_rows = L.workspace_view(ws, lv, "rgbs")[:Mr]
            r_rows = L.workspace_view(rws, rlv, "rgbs")[:Mr]
            assert torch.equal(t_rows.view(torch.int32), r_rows.view(torch.int32)), (act, precision, i)
        lv = views["levels"][-1]
        Mr, N = lv["M_rays"], lv["N"]
        z = L.workspace_view(ws, lv, "z").reshape(-1)[:Mr]
        od, dd, vd = (torch.from_numpy(a).cuda() for a in (o, d, v))
        ray = torch.arange(Mr, device="cuda") // N
        x = (od[ray] + z[:, None] * dd[ray]).contiguous()
        rows = L.workspace_view(ws, lv, "rgbs")[:Mr]
        blob = model._blob(False)
        raw_rgb, raw_sig = ops.eval_points_raw(blob, 3, x, precision=precision, net_activation=model.net_act_code)
        if precision == 1:
            rgbs_rgb, rgbs_sig = ops.eval_points(blob, 3, x, vd[ray].contiguous(), precision=1,
                                                 net_activation=model.net_act_code)
            torch.cuda.synchronize()
            assert torch.equal(rgbs_rgb, rows[:, :3]) and torch.equal(rgbs_sig[:, 0], rows[:, 3]), act
            assert torch.equal(raw_sig[:, 0].clamp_min(0), rows[:, 3]), act
            cells = ops.eval_cells_mean(blob, 3, x[:4096].reshape(-1, 1, 3).contiguous(), 1, precision=1,
                                        net_activation=model.net_act_code)
            assert torch.equal(cells[:, -1], raw_sig[:4096, 0]) and torch.equal(cells[:, :-1], raw_rgb[:4096]), act
            reso = 16
            g_rgb, g_sig = ops.eval_grid(blob, 3, reso, (0.5, 0.5, 0.5), (0.3, 0.3, 0.3), want_rgb=True,
                                         precision=1, net_activation=model.net_act_code)
            # voxel centres as the kernel forms them, in fp32 on the CPU (exact IEEE subtraction and division)
            arr = (torch.arange(reso, dtype=torch.float32) + 0.5) / reso
            c = (arr - torch.tensor(0.5, dtype=torch.float32)) / torch.tensor(0.3, dtype=torch.float32)
            gx = torch.stack(torch.meshgrid(c, c, c, indexing="ij"), -1).reshape(-1, 3).contiguous().cuda()
            p_rgb, p_sig = ops.eval_points_raw(blob, 3, gx, precision=1, net_activation=model.net_act_code)
            torch.cuda.synchronize()
            assert torch.equal(g_sig, p_sig[:, 0]) and torch.equal(g_rgb, p_rgb), act
        else:
            flat = model.params[model.P:].cpu().numpy()
            W, B, Wh, bh = operands(flat, L.K_of(3), "cuda", True)
            # posenc as the kernel forms it: exact fp32 x * 2^j, the cosine's argument added in fp32, sines in fp64
            j = torch.arange(10, device="cuda", dtype=torch.float32)
            xb = (x[:, None, :] * torch.exp2(j)[None, :, None]).reshape(-1, 30)
            arg = torch.cat([xb, xb + torch.tensor(np.float32(np.pi / 2), device="cuda")], 1)
            enc = torch.cat([x.double(), torch.sin(arg.double())], 1)
            h, inputs = enc, enc
            for l in range(8):
                h = _act64(act, h @ W[l] + B[l])
                if l == 4:
                    h = torch.cat([h, inputs], -1)
            heads = h @ Wh + bh
            err = float((raw_sig[:, 0].double() - heads[:, 0]).abs().max() / heads[:, 0].abs().max())
            rep[f"x3_raw_sigma_rel_err_{act}"] = err
            assert err < 1e-5, (act, err)
    _record(f"inference_{act}", rep)


@pytest.mark.gpu
@pytest.mark.parametrize("act", ACTS)
def test_gradient_vs_fp64_oracle(act):
    """the whole gradient against the fp64 oracle with the activation: test_sigma_activation.py's gates"""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf import train as T
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from tests.support.mlp_stages import FLOOR_SLACK, GRAD_GAIN, LOSS_REL, _setup
    R, nf, nsp = 96, 128, 300
    fc, ff, rays, px, t_rand, u, sp = _setup(3, R, nf, nsp, 77)
    for f in (fc, ff):
        _centre_sigma(f, 3, act)
    cfg = dict(num_coarse_samples=64, num_fine_samples=nf, near=2.0, far=6.0, white_bkgd=True,
               sparsity_weight=1e-3, sparsity_length=0.05)
    stats_o, gc, gf = NA.loss_and_grads(fc, ff, 3, rays, px, cfg, t_rand, u, sp, torch.float64, net_activation=act)
    ref = np.concatenate([gc, gf])
    zf = stats_o.pop("_z_fine").astype(np.float32)
    _, gc, gf = NA.loss_and_grads(fc, ff, 3, rays, px, cfg, t_rand, u, sp, torch.float32, z_fine=zf,
                                   net_activation=act)
    ref32 = np.concatenate([gc, gf])
    _, gc, gf = O.loss_and_grads(fc, ff, 3, rays, px, cfg, t_rand, u, sp, torch.float64, z_fine=zf)
    ref_relu = np.concatenate([gc, gf])
    rel = lambda g, r: float(np.linalg.norm(g - r) / np.linalg.norm(r))
    model = NerfModel(sh_deg=3, num_coarse_samples=64, num_fine_samples=nf, max_rays=R, sparsity_npoints=nsp,
                      net_activation=act)
    model.set_params(np.concatenate([fc, ff]))
    rep = {"fp32_oracle_vs_fp64": rel(ref32, ref), "relu_oracle_vs_act": rel(ref_relu, ref)}
    for name, prec in (("fp16", 1), ("fp16x3", X3)):
        state = T.TrainState(model)
        n = T.loss_and_grad(model, state, {"rays": Rays(*rays), "pixels": px}, sparsity_weight=1e-3,
                            sparsity_length=0.05, randomized=True, t_rand=t_rand, u=u, sp_points=sp, z_fine=zf,
                            precision=prec)
        torch.cuda.synchronize()
        g = state.grads.double().cpu().numpy()
        st = T.stats_from_raw(state.stats_raw, n, 1e-3, nsp, True)
        rep[name] = dict(grad_rel_l2=rel(g, ref), grad_rel_l2_vs_fp32_oracle=rel(g, ref32),
                         cosine=float(np.dot(g, ref) / (np.linalg.norm(g) * np.linalg.norm(ref))),
                         loss_rel=abs(st.loss - stats_o["loss"]) / stats_o["loss"],
                         loss_c_rel=abs(st.loss_c - stats_o["loss_c"]) / stats_o["loss_c"],
                         loss_sp_abs=abs(st.loss_sp - stats_o["loss_sp"]))
    rep["gain_vs_fp32_oracle"] = rep["fp16"]["grad_rel_l2_vs_fp32_oracle"] / rep["fp16x3"]["grad_rel_l2_vs_fp32_oracle"]
    _record(f"gradient_vs_fp64_oracle_{act}", rep)
    x, h = rep["fp16x3"], rep["fp16"]
    assert x["loss_rel"] < LOSS_REL and x["loss_c_rel"] < LOSS_REL, rep
    assert x["loss_sp_abs"] < LOSS_REL * max(abs(stats_o["loss_sp"]), 1e-6) + 1e-8, rep
    if act == "softplus":
        # f'(h) = 1 - exp(-h) ~ h for the small h of strongly negative pre-activations, and the hi + lo pair holds h
        # to 2^-25 absolute (fp16 subnormals), not relative as fp32 does: those units' dZ lose relative precision
        assert x["grad_rel_l2"] <= SOFTPLUS_X3_REL, rep
    else:
        assert x["grad_rel_l2"] <= FLOOR_SLACK * rep["fp32_oracle_vs_fp64"], rep
    assert rep["gain_vs_fp32_oracle"] >= GRAD_GAIN, rep
    assert h["loss_rel"] < 5e-3 and h["loss_c_rel"] < 5e-3, rep
    # fp16 sparsity loss: test_sigma_activation.py's 2e-3 relative; a softplus trunk's raw sigma carries the larger
    # fp16 error of its dense positive h ([4.7e-3 relative, 1.8e-7 absolute on loss_sp = 3.8e-5])
    sp_rel = 1e-2 if act == "softplus" else 2e-3
    assert h["loss_sp_abs"] < sp_rel * max(abs(stats_o["loss_sp"]), 1e-6) + 1e-7, rep
    assert h["grad_rel_l2"] < 2e-2 and h["cosine"] > 0.9995, rep
    assert rep["relu_oracle_vs_act"] > 100 * rep["fp16x3"]["grad_rel_l2"], rep


@pytest.mark.gpu
def test_cli_train_eval_mesh_extract_elu(tmp_path):
    """nerf_sh.train --net_activation elu learns a synthetic scene, then nerf_sh.eval, nerf_sh.gen_mesh and
    octree.extraction run on its checkpoint with the same flag"""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf import datasets as D, flags as F
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf.utils import generate_rays, pose_spherical, render_image
    from plenoctree_b200.nerf_sh import eval as EV, gen_mesh as GM, train as TR
    from plenoctree_b200.octree import extraction as EX
    sh_deg, W = 3, 48
    ft = np.concatenate([O.init_flat_params(sh_deg, 7001, bias_scale=0.05), O.init_flat_params(sh_deg, 7002, bias_scale=0.05)])
    P = O.param_count(sh_deg)
    for m in range(2):
        off = m * P + P - 48 - 1 - 256 * 48 - 256
        ft[off:off + 256] *= 30.0
    teacher = NerfModel(sh_deg=sh_deg, max_rays=4096)
    teacher.set_params(ft)
    cam_x = 0.6911112070083618
    focal = 0.5 * W / np.tan(0.5 * cam_x)
    rs = np.random.RandomState(3)
    splits = {"train": 8, "val": 2, "test": 2}
    poses = {k: [pose_spherical(rs.uniform(-180, 180), rs.uniform(-80, -10), 4.0) for _ in range(n)] for k, n in splits.items()}
    images = {}
    for k in splits:
        rays = generate_rays(W, W, focal, np.stack(poses[k]))
        images[k] = [render_image(teacher, Rays(rays.origins[i], rays.directions[i], rays.viewdirs[i]))[0].cpu().numpy()
                     for i in range(splits[k])]
    data_dir, train_dir = str(tmp_path / "scene"), str(tmp_path / "ckpt")
    D.write_blender_scene(data_dir, images, poses, cam_x)
    (tmp_path / "cfg.yaml").write_text("dataset: blender\nfactor: 0\nnum_coarse_samples: 64\nnum_fine_samples: 128\n"
                                       "use_viewdirs: false\nwhite_bkgd: true\nbatch_size: 1024\nsh_deg: 3\n"
                                       "randomized: true\nmax_steps: 200\nnet_activation: elu\n")
    EX._define_cli_flags()
    F.define_flags()
    FLAGS = F.FLAGS
    if not FLAGS.is_parsed():
        FLAGS.mark_as_parsed()
    new = dict(train_dir=train_dir, data_dir=data_dir, config=str(tmp_path / "cfg"), save_every=200, print_every=100,
               render_every=0, sparsity_npoints=1000, lr_init=2e-3, lr_final=2e-4, chunk=4096, noise_std=None,
               image_batching=True, is_jaxnerf_ckpt=True, init_grid_depth=5, samples_per_cell=8, masking_mode="sigma",
               alpha_thresh=1e-6, renderer_step_size=1e-3, radius="1.5", eval=False, output=None,
               reso="48 48 48", c1="-1.5", c2="1.5", iso=6.0, coarse=False, point_chunk=65536)
    old = {k: getattr(FLAGS, k) for k in list(new) + ["net_activation", "max_steps"]}
    try:
        for k, v in new.items():
            setattr(FLAGS, k, v)
        model, state = TR.main(None)
        assert model.net_act_code == 1 and state.step == 200
        psnr, _ = EV.main(None)
        fresh = NerfModel(sh_deg=sh_deg, max_rays=4096, net_activation="elu")
        fresh.init_params(20200823)
        rays = generate_rays(W, W, focal, np.stack(poses["test"]))
        gt = torch.from_numpy(images["test"][0]).cuda()
        p_init = -10 * np.log10(float(((render_image(fresh, Rays(rays.origins[0], rays.directions[0],
                                                                  rays.viewdirs[0]))[0] - gt) ** 2).mean()))
        # the surface at half the trained density's maximum over the mesh box
        ax = torch.linspace(-1.5, 1.5, 32, device="cuda")
        box = torch.stack(torch.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3).contiguous()
        _, sig = model.eval_points_raw(box, want_rgb=False)
        FLAGS.iso = 0.5 * float(sig.max())
        mesh = GM.main(None)
        assert os.path.getsize(mesh) > 0
        FLAGS.config = None
        FLAGS.net_activation = "elu"
        FLAGS.output = str(tmp_path / "tree_elu.npz")
        EX.main(None)
        tree = dict(np.load(FLAGS.output))
        _record("cli_elu", dict(psnr_init=p_init, psnr_200_steps=psnr, tree_keys=sorted(tree)))
        assert psnr > p_init + 2.0, (p_init, psnr)
        assert len(tree) > 0
    finally:
        for k, v in old.items():
            setattr(FLAGS, k, v)

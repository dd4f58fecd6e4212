"""What the MLP entry points of the C ABI refuse, in which order and with which message, and what a successful call
launches.

Each table lists one entry point's checks in the order the library makes them, as (bad arguments, exact
pob_last_error text).  Row i is called with its own bad arguments and those of every later row (an argument that two
rows set keeps the earlier row's value), so its check must come before all the later ones.  The CPU tables stop at
the device query (the SM count); the GPU tables carry on behind it, and no refusal there may launch a kernel.  A
successful call launches a fixed number of kernels, each counted by pob_launch_count and, except the output packing
of pob_render_rays and the projection's own kernel, timed under one phase of pob_timing_read."""
import ctypes

import numpy as np
import pytest

from plenoctree_b200 import _lib
from plenoctree_b200._lib import NetDesc, RenderConfig, TrainHParams, lib

FAKE = 0x1000                      # a non-NULL pointer that no check before a refusal dereferences
BAD_PE = NetDesc(3, 2, 0, 0)       # min_deg > max_deg
ELU_PE = NetDesc(0, 10, 0, _lib.NET_ELU)
PE_MSG = ("posenc needs 0 <= min_deg <= max_deg <= 10 (width 3 + 6 (max_deg - min_deg) <= 63, the 64-column posenc "
          "tile with its constant-one bias column), legacy_order 0 or 1 and net_activation one of POB_NET_RELU, "
          "POB_NET_ELU, POB_NET_SOFTPLUS, POB_NET_TANH")
SH_MSG = "sh_deg must be in [-1, 4]"
PREC_MSG = "precision must be POB_PREC_FP16 or POB_PREC_FP16X3"
RESET = "pob_sample_coarse: NULL pointer"
PHASES = ("fwd", "bwd", "wgrad", "render", "optim")   # POB_PH_*


def _ref(s):
    return None if s is None else ctypes.addressof(s)


def _cfg(a):
    """the pob_render_config of the arguments a (kept alive in a)"""
    if a["cfg_null"]:
        return None
    c = RenderConfig(a["sh_deg"], a["nc"], a["nf"], 1, a["max_rays"], a["nsp"])
    c.sigma_activation = a["sigma_act"]
    c.posenc = _ref(a["posenc"])
    a["_cfg"] = c
    return ctypes.addressof(c)


CFG = dict(cfg_null=False, sh_deg=3, nc=8, nf=16, max_rays=64, nsp=32, sigma_act=0, posenc=None)
CFG_ROWS = [
    (dict(cfg_null=True), "config is NULL"),
    (dict(sh_deg=5), SH_MSG),
    (dict(nc=2), "num_coarse_samples must be in [3, 1024]"),
    (dict(nf=1020), "num_coarse_samples + num_fine_samples must be <= 1024"),
    (dict(max_rays=0), "max_rays must be positive"),
    (dict(nsp=-1), "sparsity_npoints must be >= 0"),
    (dict(posenc=BAD_PE), PE_MSG),
    (dict(sigma_act=2), "sigma_activation must be POB_SIGMA_RELU or POB_SIGMA_SOFTPLUS"),
]


def _specs(P):
    """name -> (where, call(args) -> rc, failing rc, base arguments, CPU rows, GPU rows).  P: pointer values (FAKE
    here; device buffers on the GPU, where the GPU rows also need P['ws16'], a plain allocation of the fp16 training
    workspace of CFG)."""
    X = P["x"]
    f3 = ctypes.c_float * 3
    ev = dict(packed=X, sh=3, posenc=None, prec=_lib.PREC_FP16)
    ev_rows = [(dict(sh=5), SH_MSG), (dict(packed=None), "packed weights pointer is NULL"), (dict(prec=2), PREC_MSG)]
    render = dict(CFG, pk_c=X, pk_f=X, o=X, d=X, v=X, n=8, zb=X, u=X, zf=None, out_c=X, out_f=X, ws=X,
                  prec=_lib.PREC_FP16)
    train = dict(CFG, flags=0, hp=(0.1, 0.05, 1024.0), pk_c=X, pk_f=X, o=X, d=X, v=X, px=X, n=8, zb=X, u=X, zf=None,
                 sp=X, g=X, stats=X, ws=X, params=X, prec=_lib.PREC_FP16)

    def hp(a):
        if a["hp"] is None:
            return None
        a["_hp"] = TrainHParams(*a["hp"])
        return ctypes.addressof(a["_hp"])

    return {
        "pob_param_count_pe": (
            "pob_param_count", lambda a: lib.pob_param_count_pe(a["sh"], _ref(a["posenc"])), -1,
            dict(sh=3, posenc=None),
            [(dict(sh=5), None), (dict(sh=-2), None), (dict(posenc=BAD_PE), PE_MSG)], []),
        "pob_pack_weights_pe": (
            "pob_pack_weights",
            lambda a: lib.pob_pack_weights_pe(a["flat"], a["sh"], _ref(a["posenc"]), a["packed"], None), 1,
            dict(flat=X, sh=3, posenc=None, packed=X),
            [(dict(sh=5), SH_MSG), (dict(posenc=BAD_PE), PE_MSG), (dict(flat=None), "NULL pointer"),
             (dict(packed=None), "NULL pointer")], []),
        "pob_workspace_bytes": (
            "pob_workspace_bytes", lambda a: lib.pob_workspace_bytes(_cfg(a), 1), -1, dict(CFG), CFG_ROWS, []),
        "pob_train_workspace_bytes": (
            "pob_train_workspace_bytes", lambda a: lib.pob_train_workspace_bytes(_cfg(a), a["prec"]), -1,
            dict(CFG, prec=_lib.PREC_FP16X3), CFG_ROWS + [(dict(prec=2), PREC_MSG)], []),
        "pob_render_rays": (
            "pob_render_rays",
            lambda a: lib.pob_render_rays(_cfg(a), a["pk_c"], a["pk_f"], a["o"], a["d"], a["v"], a["n"], a["zb"], None,
                                          a["u"], 1, a["zf"], a["out_c"], a["out_f"], a["ws"], a["prec"], None), 1,
            render,
            CFG_ROWS + [(dict(pk_c=None), "packed weights pointer is NULL"), (dict(prec=2), PREC_MSG)],
            [(dict(n=-1), "n_rays exceeds cfg->max_rays"), (dict(n=65), "n_rays exceeds cfg->max_rays"),
             (dict(o=None), "NULL pointer"), (dict(d=None), "NULL pointer"), (dict(v=None), "NULL pointer"),
             (dict(zb=None), "NULL pointer"), (dict(ws=None), "NULL pointer"), (dict(out_c=None), "NULL pointer"),
             (dict(pk_f=None), "fine level needs packed_fine, u (or z_fine) and out_fine"),
             (dict(u=None), "fine level needs packed_fine, u (or z_fine) and out_fine"),
             (dict(out_f=None), "fine level needs packed_fine, u (or z_fine) and out_fine")]),
        "pob_loss_and_grad_flags": (
            "pob_loss_and_grad",
            lambda a: lib.pob_loss_and_grad_flags(
                _cfg(a), hp(a), a["pk_c"], a["pk_f"], a["o"], a["d"], a["v"], a["px"], a["n"], a["zb"], None, a["u"],
                1, a["zf"], a["sp"], a["g"], a["stats"], a["ws"], None, a["params"], a["prec"], a["flags"], None), 1,
            train,
            [(dict(flags=2), "unknown bits in flags")] + CFG_ROWS +
            [(dict(hp=None), "hparams is NULL"), (dict(pk_c=None), "packed weights pointer is NULL"),
             (dict(prec=2), PREC_MSG)],
            [(dict(n=0), "n_rays out of range"), (dict(n=65), "n_rays out of range"),
             (dict(o=None), "NULL pointer"), (dict(px=None), "NULL pointer"), (dict(ws=None), "NULL pointer"),
             (dict(g=None), "NULL pointer"), (dict(stats=None), "NULL pointer"),
             (dict(prec=_lib.PREC_FP16X3, params=None), "POB_PREC_FP16X3 needs params_dev (the flat fp32 parameters)"),
             (dict(pk_f=None), "fine level needs packed_fine and u (or z_fine)"),
             (dict(u=None), "fine level needs packed_fine and u (or z_fine)"),
             (dict(sp=None), "sparsity term needs sp_points"),
             (dict(hp=(0.1, 0.05, 0.0)), "loss_scale must be positive"),
             (dict(prec=_lib.PREC_FP16X3, ws=FAKE), "workspace is not a device allocation"),
             (dict(prec=_lib.PREC_FP16X3, ws=P.get("ws16")),
              "workspace too small for this precision (pob_train_workspace_bytes)")]),
        "pob_eval_points_raw_pe": (
            "pob_eval_points_raw",
            lambda a: lib.pob_eval_points_raw_pe(a["packed"], a["sh"], _ref(a["posenc"]), a["pts"], a["m"], X,
                                                 a["sig"], a["prec"], None), 1,
            dict(ev, pts=X, m=100, sig=X), ev_rows,
            [(dict(posenc=BAD_PE), PE_MSG), (dict(m=-1), "negative point count"), (dict(pts=None), "NULL pointer"),
             (dict(sig=None), "NULL pointer")]),
        "pob_eval_points_pe": (
            "pob_eval_points",
            lambda a: lib.pob_eval_points_pe(a["packed"], a["sh"], _ref(a["posenc"]), a["pts"], a["vd"], a["m"],
                                             a["out"], a["sact"], a["prec"], None), 1,
            dict(ev, pts=X, vd=X, m=100, out=X, sact=0), ev_rows,
            [(dict(posenc=BAD_PE), PE_MSG),
             (dict(sact=2), "sigma_activation must be POB_SIGMA_RELU or POB_SIGMA_SOFTPLUS"),
             (dict(m=-1), "negative point count"), (dict(pts=None), "NULL pointer"), (dict(out=None), "NULL pointer"),
             (dict(vd=None), "viewdirs required when sh_deg >= 0 (models.py:199)")]),
        "pob_eval_cells_mean_pe": (
            "pob_eval_cells_mean",
            lambda a: lib.pob_eval_cells_mean_pe(a["packed"], a["sh"], _ref(a["posenc"]), a["pts"], a["n"], a["S"],
                                                 a["out"], a["prec"], None), 1,
            dict(ev, pts=X, n=10, S=8, out=X), ev_rows,
            [(dict(posenc=BAD_PE), PE_MSG), (dict(n=-1), "bad sizes"), (dict(S=0), "bad sizes"),
             (dict(pts=None), "NULL pointer"), (dict(out=None), "NULL pointer")]),
        "pob_eval_grid_pe": (
            "pob_eval_grid",
            lambda a: lib.pob_eval_grid_pe(a["packed"], a["sh"], _ref(a["posenc"]), a["reso"], a["x0"], a["nx"], 16,
                                           16, a["off"], a["scale"], X, a["sig"], a["prec"], None), 1,
            dict(ev, reso=16, x0=0, nx=4, off=f3(0.5, 0.5, 0.5), scale=f3(0.3, 0.3, 0.3), sig=X), ev_rows,
            [(dict(posenc=BAD_PE), PE_MSG), (dict(reso=12), "reso must be a power of two (extraction.py:246,290)"),
             (dict(x0=-1), "slab out of range"), (dict(nx=17), "slab out of range"),
             (dict(off=None), "NULL pointer"), (dict(scale=None), "NULL pointer"), (dict(sig=None), "NULL pointer")]),
        "pob_eval_points_raw_host_pe": (
            "pob_eval_points_raw_host",
            lambda a: lib.pob_eval_points_raw_host_pe(a["packed"], a["sh"], _ref(a["posenc"]), a["pts"], a["m"], None,
                                                      a["sig"], a["prec"]), 1,
            dict(ev, pts=FAKE, m=100, sig=FAKE), ev_rows,
            [(dict(posenc=BAD_PE), PE_MSG), (dict(m=-1), "negative point count"), (dict(pts=None), "NULL pointer"),
             (dict(sig=None), "NULL pointer")]),
        "pob_sh_proj_points": (
            "pob_sh_proj_points",
            lambda a: lib.pob_sh_proj_points(a["packed"], _ref(a["posenc"]), a["pts"], a["m"], a["hw"], X, X, X,
                                             a["sig"], None), 1,
            dict(packed=X, posenc=None, pts=X, m=100, hw=X, sig=X),
            [(dict(packed=None), "packed weights pointer is NULL")],
            [(dict(posenc=BAD_PE), PE_MSG), (dict(posenc=ELU_PE), "the vanilla trunk of the projection is relu"),
             (dict(m=-1), "negative point count"), (dict(pts=None), "NULL pointer"), (dict(hw=None), "NULL pointer"),
             (dict(sig=None), "NULL pointer")]),
        "pob_adam_update_pe": (
            "pob_adam_update",
            lambda a: lib.pob_adam_update_pe(a["sh"], _ref(a["posenc"]), a["n"], a["params"], a["g"], a["m"], a["v"],
                                             1e-3, 1.0, None, 1.0, 0.0, a["pk_c"], a["pk_f"], None), 1,
            dict(sh=3, posenc=None, n=2, params=X, g=X, m=X, v=X, pk_c=X, pk_f=X),
            [(dict(sh=-2), SH_MSG), (dict(posenc=BAD_PE), PE_MSG), (dict(n=3), "num_mlps must be 1 or 2"),
             (dict(params=None), "NULL pointer"), (dict(g=None), "NULL pointer"), (dict(v=None), "NULL pointer"),
             (dict(pk_c=None), "NULL pointer"), (dict(pk_f=None), "NULL pointer")], []),
    }


def _check_rows(name, spec, rows, on_gpu):
    where, call, bad_rc, base, _, _ = spec
    for i, (_, what) in enumerate(rows):
        args = dict(base)
        for over, _ in reversed(rows[i:]):
            args.update(over)
        lib.pob_sample_coarse(None, None, 0, 0, None, None)
        assert lib.pob_last_error().decode() == RESET
        n0 = lib.pob_launch_count()
        rc = call(args)
        msg = lib.pob_last_error().decode()
        assert rc == bad_rc, (name, i, what, rc, msg)
        assert msg == (RESET if what is None else f"{where}: {what}"), (name, i, msg)
        if on_gpu:
            assert lib.pob_launch_count() == n0, (name, i, what)


@pytest.mark.parametrize("name", sorted(_specs({"x": FAKE})))
def test_refusals_before_the_device_query(name):
    """the checks each MLP entry point makes before it asks for the SM count: exact message, in order"""
    spec = _specs({"x": FAKE})[name]
    _check_rows(name, spec, spec[4], False)


@pytest.mark.gpu
def test_refusals_launch_nothing():
    """every check of each MLP entry point, the device query passing: exact message, in order, and no kernel
    counted"""
    import torch
    buf = torch.zeros(1 << 22, dtype=torch.float32, device="cuda")
    lib.cudaMalloc.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_size_t]
    lib.cudaFree.argtypes = [ctypes.c_void_p]
    ws16 = ctypes.c_void_p()
    c = RenderConfig(3, 8, 16, 1, 64, 32)
    assert lib.cudaMalloc(ctypes.byref(ws16), int(lib.pob_train_workspace_bytes(ctypes.addressof(c), 1))) == 0
    try:
        for name, spec in sorted(_specs({"x": buf.data_ptr(), "ws16": ws16.value}).items()):
            _check_rows(name, spec, spec[4] + spec[5], True)
        torch.cuda.synchronize()
    finally:
        lib.cudaFree(ws16)


# =====================================================================================================================
# what a successful call launches
# =====================================================================================================================
def _launches(fn):
    """(kernels counted, {phase: timed launches}) of fn()"""
    import torch
    torch.cuda.synchronize()
    lib.pob_timing_enable(1)
    try:
        n0 = lib.pob_launch_count()
        fn()
        torch.cuda.synchronize()
        n = lib.pob_launch_count() - n0
        ms, cnt = (ctypes.c_double * 5)(), (ctypes.c_longlong * 5)()
        assert lib.pob_timing_read(ms, cnt) == 5
    finally:
        lib.pob_timing_enable(0)
    return n, {p: int(k) for p, k in zip(PHASES, cnt) if k}


def _rays(R, nc, nf, seed=3):
    import torch
    from plenoctree_b200.nerf.models import Rays
    g = torch.Generator(device="cuda").manual_seed(seed)
    o = torch.rand(R, 3, device="cuda", generator=g) * 0.2
    d = torch.nn.functional.normalize(torch.rand(R, 3, device="cuda", generator=g) - 0.5, dim=1)
    d[:, 2] -= 2.0
    v = torch.nn.functional.normalize(d, dim=1)
    t = torch.rand(R, nc, device="cuda", generator=g)
    u = torch.rand(R, nf, device="cuda", generator=g) if nf else None
    px = torch.rand(R, 3, device="cuda", generator=g)
    return Rays(o, d, v), t, u, px


def _model(nc, nf, nsp, R=64):
    from plenoctree_b200.nerf.models import NerfModel
    m = NerfModel(sh_deg=3, num_coarse_samples=nc, num_fine_samples=nf, max_rays=R, sparsity_npoints=nsp)
    m.init_params(5)
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("levels, z_fine, want", [
    (1, False, (4, dict(fwd=1, render=2))),
    (2, False, (8, dict(fwd=2, render=4))),
    (2, True, (7, dict(fwd=2, render=3))),
])
def test_render_launches(levels, z_fine, want):
    """pob_render_rays: per level sample (coarse draw or fine resample; a caller's z_fine is copied instead), forward
    and composite, then one untimed output pack per level"""
    import torch
    nc, nf = 16, (32 if levels == 2 else 0)
    model = _model(nc, nf, 0)
    rays, t, u, _ = _rays(64, nc, nf)
    zf = None
    if z_fine:
        zf = torch.sort(2.0 + 4.0 * torch.rand(64, nc + nf, device="cuda"), dim=1).values
    assert _launches(lambda: model(rays, randomized=True, t_rand=t, u=u, z_fine=zf)) == want


@pytest.mark.gpu
@pytest.mark.parametrize("levels, precision, sparsity, want", [
    (2, _lib.PREC_FP16, True, (15, dict(fwd=2, bwd=2, wgrad=2, render=7, optim=2))),
    (2, _lib.PREC_FP16, False, (14, dict(fwd=2, bwd=2, wgrad=2, render=6, optim=2))),
    (2, _lib.PREC_FP16X3, True, (21, dict(fwd=2, bwd=2, wgrad=6, render=7, optim=4))),
    (2, _lib.PREC_FP16X3, False, (20, dict(fwd=2, bwd=2, wgrad=6, render=6, optim=4))),
    (1, _lib.PREC_FP16, True, (8, dict(fwd=1, bwd=1, wgrad=1, render=4, optim=1))),
    (1, _lib.PREC_FP16X3, True, (11, dict(fwd=1, bwd=1, wgrad=3, render=4, optim=2))),
])
def test_training_launches(levels, precision, sparsity, want):
    """pob_loss_and_grad_flags: x3 weight residuals (one per MLP), the render forward of every level, one composite
    backward per level, the sparsity gradient, then per MLP data gradient, weight gradient (three passes in x3) and
    reduction"""
    import torch
    from plenoctree_b200.nerf import train as T
    nc, nf = 16, (32 if levels == 2 else 0)
    model = _model(nc, nf, 96)
    state = T.TrainState(model)
    rays, t, u, px = _rays(64, nc, nf)
    sp = torch.rand(96, 3, device="cuda") * 3.0 - 1.5
    batch = {"rays": rays, "pixels": px}
    got = _launches(lambda: T.loss_and_grad(model, state, batch, sparsity_weight=1e-3 if sparsity else 0.0,
                                            t_rand=t, u=u, sp_points=sp, precision=precision))
    assert got == want
    assert torch.isfinite(state.grads).all()


@pytest.mark.gpu
def test_evaluator_and_projection_launches():
    """each evaluator, the host evaluator and the projection's point stage (one forward, then its own untimed
    kernel): one counted launch per kernel, the forward timed under fwd"""
    import torch
    from oracle import projection_oracle as PJ
    from plenoctree_b200 import ops
    from plenoctree_b200._lib import ptr
    from plenoctree_b200.octree.projection import VanillaNerf
    model = _model(16, 0, 0)
    blob = model.blobs[0]
    x = torch.rand(1000, 3, device="cuda") * 2 - 1
    vd = torch.nn.functional.normalize(torch.rand(1000, 3, device="cuda") - 0.5, dim=1)
    one = (1, dict(fwd=1))
    for prec in (_lib.PREC_FP16, _lib.PREC_FP16X3):
        assert _launches(lambda: ops.eval_points_raw(blob, 3, x, precision=prec)) == one
        assert _launches(lambda: ops.eval_points_raw(blob, 3, x, want_rgb=False, precision=prec)) == one
        assert _launches(lambda: ops.eval_points(blob, 3, x, vd, precision=prec)) == one
        assert _launches(lambda: ops.eval_cells_mean(blob, 3, x, 10, precision=prec)) == one
        assert _launches(lambda: ops.eval_grid(blob, 3, 16, (0.5, 0.5, 0.5), (0.3, 0.3, 0.3), precision=prec)) == one
    xh = x.cpu().numpy()
    sig = np.zeros(1000, np.float32)
    assert _launches(lambda: _lib.check(lib.pob_eval_points_raw_host_pe(ptr(blob), 3, None, xh.ctypes.data, 1000,
                                                                         None, sig.ctypes.data, 1))) == one
    assert np.isfinite(sig).all() and sig.any()
    vn = VanillaNerf({"MLP_0": PJ.init_params(46)}, (0, 10, False), 4, num_fine_samples=0)
    ws = torch.empty(int(lib.pob_sh_proj_points_workspace_bytes(1000)), dtype=torch.uint8, device="cuda")
    a, s = torch.empty(1000, 128, device="cuda"), torch.empty(1000, device="cuda")
    assert _launches(lambda: _lib.check(lib.pob_sh_proj_points(ptr(vn.sigma_blob), None, ptr(x), 1000, ptr(vn.head_w),
                                                               ptr(vn.head_b), ptr(ws), ptr(a), ptr(s),
                                                               _lib.stream_ptr()))) == (2, dict(fwd=1))


@pytest.mark.gpu
@pytest.mark.parametrize("mlps", [1, 2])
def test_adam_launches(mlps):
    """pob_adam_update_pe: one Adam launch over every MLP's parameters, then one weight pack per MLP, all under
    optim"""
    from plenoctree_b200.nerf import train as T
    from plenoctree_b200._lib import ptr
    model = _model(16, 32 if mlps == 2 else 0, 0)
    state = T.TrainState(model)
    state.grads.normal_()
    assert _launches(lambda: _lib.check(lib.pob_adam_update_pe(
        3, None, mlps, ptr(model.params), ptr(state.grads), ptr(state.m), ptr(state.v), 1e-3, 1.0, None, 1.0, 0.0,
        ptr(model.blobs[0]), ptr(model.blobs[1]) if mlps == 2 else None, None))) == (1 + mlps, dict(optim=1 + mlps))

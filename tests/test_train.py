"""GPU parity of value_and_grad(loss_fn) + Adam against the CPU oracle's autograd."""
import functools

import numpy as np
import pytest
import torch

from tests.support.mlp_stages import _setup
from tests.support.records import record

pytestmark = pytest.mark.gpu


_record = functools.partial(record, "parity_train.json")


def _layer_report(g, ref, sh_deg):
    from plenoctree_b200 import layouts as L
    w_off, b_off, total = L.flat_offsets(L.K_of(sh_deg))
    dims = L.layer_dims(L.K_of(sh_deg))
    rep = {}
    for i, (cin, cout) in enumerate(dims):
        for nm, a, n in (("w", w_off[i], cin * cout), ("b", b_off[i], cout)):
            x, y = g[a:a + n], ref[a:a + n]
            rel = float(np.linalg.norm(x - y) / max(1e-30, np.linalg.norm(y)))
            rep[f"Dense_{i}.{nm}"] = rel
    return rep


@pytest.mark.parametrize("sh_deg,R,nf,nsp", [(3, 96, 128, 300), (3, 64, 0, 0), (4, 40, 128, 64)])
def test_loss_and_grad_vs_oracle(sh_deg, R, nf, nsp):
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf import train as T
    fc, ff, rays, px, t_rand, u, sp = _setup(sh_deg, R, nf, nsp, 77)
    cfg = dict(num_coarse_samples=64, num_fine_samples=nf, near=2.0, far=6.0, white_bkgd=True,
               sparsity_weight=1e-3 if nsp else 0.0, sparsity_length=0.05)
    stats_o, gc_o, gf_o = O.loss_and_grads(fc, ff, sh_deg, rays, px, cfg, t_rand, u, sp)
    stats_o.pop("_z_fine")
    model = NerfModel(sh_deg=sh_deg, num_coarse_samples=64, num_fine_samples=nf, max_rays=R, sparsity_npoints=nsp)
    model.set_params(np.concatenate([fc, ff]) if nf else fc)
    state = T.TrainState(model)
    batch = {"rays": Rays(*rays), "pixels": px}
    n = T.loss_and_grad(model, state, batch, sparsity_weight=cfg["sparsity_weight"], sparsity_length=0.05,
                        randomized=True, t_rand=t_rand, u=u, sp_points=sp)
    torch.cuda.synchronize()
    g = state.grads.cpu().numpy()
    assert np.isfinite(g).all()
    P = model.P
    rep = {"MLP_0": _layer_report(g[:P], gc_o, sh_deg)}
    if nf:
        rep["MLP_1"] = _layer_report(g[P:], gf_o, sh_deg)
    st = T.stats_from_raw(state.stats_raw, n, cfg["sparsity_weight"], nsp, nf > 0)
    rep["stats"] = dict(gpu=st._asdict(), oracle=stats_o)
    _record(f"sh{sh_deg}_R{R}_nf{nf}_nsp{nsp}", rep)
    # loss values (fp16 operands incl. biases, free-running fine level on 40-96 rays): 5e-3 relative
    assert abs(st.loss - stats_o["loss"]) / stats_o["loss"] < 5e-3
    if nf:
        assert abs(st.loss_c - stats_o["loss_c"]) / stats_o["loss_c"] < 5e-3
    if nsp:
        assert abs(st.loss_sp - stats_o["loss_sp"]) < 2e-3 * max(abs(stats_o["loss_sp"]), 1e-6) + 1e-7
    # (a) against the fp32 oracle, free running.  fp16 operands flip ~4e-4 of the ReLU masks and move the
    # fine-level samples, so early layers carry per-tensor errors of a few percent on a random-init field;
    # the bar is on the whole gradient: relative L2 < 2e-2, cosine > 0.9995, and tight heads for MLP_0.
    ref_all = np.concatenate([gc_o, gf_o]) if nf else gc_o
    tot = float(np.linalg.norm(g - ref_all) / np.linalg.norm(ref_all))
    cos = float(np.dot(g, ref_all) / (np.linalg.norm(g) * np.linalg.norm(ref_all)))
    _record(f"sh{sh_deg}_R{R}_nf{nf}_nsp{nsp}_total", dict(rel_l2=tot, cosine=cos))
    assert tot < 2e-2 and cos > 0.9995, (tot, cos)
    assert rep["MLP_0"]["Dense_9.w"] < 5e-3 and rep["MLP_0"]["Dense_8.w"] < 5e-3
    # (b) against the oracle with the SAME operand precision (fp16-rounded GEMM operands, fp32 accumulate,
    # loss-scaled fp16 gradient chain) and the same fine-level depths: isolates kernel logic from precision.
    # Even this emulation is chaotic at the percent level for the early layers: a pre-activation within
    # rounding distance of zero flips its ReLU mask, and the emulation evaluated in fp32 vs fp64 already
    # differs by ~2e-2 on Dense_0 (measured; DESIGN.md "gradient parity").  Bars: heads < 1e-2 (no mask
    # upstream of them flips the result), trunk tensors < 0.1, whole gradient < 2e-2.
    scale = T.default_loss_scale(R)
    with O.emulate_fp16_operands(loss_scale=scale):
        stats_e, gc_e, gf_e = O.loss_and_grads(fc, ff, sh_deg, rays, px, cfg, t_rand, u, sp)
    T.loss_and_grad(model, state, batch, sparsity_weight=cfg["sparsity_weight"], sparsity_length=0.05,
                    randomized=True, t_rand=t_rand, u=u, sp_points=sp, z_fine=stats_e["_z_fine"])
    torch.cuda.synchronize()
    g2 = state.grads.cpu().numpy()
    rep2 = {"MLP_0": _layer_report(g2[:P], gc_e, sh_deg)}
    if nf:
        rep2["MLP_1"] = _layer_report(g2[P:], gf_e, sh_deg)
    _record(f"sh{sh_deg}_R{R}_nf{nf}_nsp{nsp}_vs_fp16_emulation", rep2)
    ref_e = np.concatenate([gc_e, gf_e]) if nf else gc_e
    tot_e = float(np.linalg.norm(g2 - ref_e) / np.linalg.norm(ref_e))
    _record(f"sh{sh_deg}_R{R}_nf{nf}_nsp{nsp}_vs_fp16_emulation_total", dict(rel_l2=tot_e))
    assert tot_e < 2e-2, tot_e
    for mlp in rep2:
        for name, rel in rep2[mlp].items():
            bar = 1e-2 if name.startswith(("Dense_8", "Dense_9")) else 0.1
            assert rel < bar, (mlp, name, rel)


def test_adam_update_and_repack():
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf.models import NerfModel
    from plenoctree_b200.nerf import train as T
    from plenoctree_b200._lib import check, lib, ptr
    sh_deg = 3
    model = NerfModel(sh_deg=sh_deg, max_rays=64)
    model.init_params(3)
    state = T.TrainState(model)
    rs = np.random.RandomState(0)
    p = model.params.cpu().numpy().copy()
    m = np.zeros_like(p)
    v = np.zeros_like(p)
    for step in range(3):
        g = (rs.normal(size=p.shape) * 1e-3).astype(np.float32)
        state.grads.copy_(torch.from_numpy(g))
        check(lib.pob_adam_update(sh_deg, 2, ptr(model.params), ptr(state.grads), ptr(state.m), ptr(state.v),
                                  5e-4, float(step), None, 0.5, 0.0, ptr(model.blobs[0]), ptr(model.blobs[1]), None))
        p, m, v = O.adam_step(p, 0.5 * g, m, v, float(step), 5e-4)
    torch.cuda.synchronize()
    np.testing.assert_allclose(model.params.cpu().numpy(), p, rtol=2e-5, atol=1e-7)
    # weight decay (train.py:101-114: loss += weight_decay_mult * sum(theta^2)/numel): g += coef * theta with
    # coef = 2 * weight_decay_mult / numel, here a large value so that the term matters; lr / step from the device
    coef = 0.25
    for step in range(3, 5):
        g = (rs.normal(size=p.shape) * 1e-3).astype(np.float32)
        state.grads.copy_(torch.from_numpy(g))
        state.lr_step.copy_(torch.tensor([3e-4, float(step)]))
        check(lib.pob_adam_update(sh_deg, 2, ptr(model.params), ptr(state.grads), ptr(state.m), ptr(state.v),
                                  123.0, -7.0, ptr(state.lr_step), 0.5, coef, ptr(model.blobs[0]),
                                  ptr(model.blobs[1]), None))
        p, m, v = O.adam_step(p, 0.5 * g + np.float32(coef) * p, m, v, float(step), 3e-4)
    torch.cuda.synchronize()
    np.testing.assert_allclose(model.params.cpu().numpy(), p, rtol=2e-5, atol=1e-7)
    # the packed blob follows the new parameters
    from plenoctree_b200 import ops
    pts = torch.from_numpy(rs.uniform(-1, 1, size=(300, 3)).astype(np.float32)).cuda()
    rgb, sig = model.eval_points_raw(pts, precision=ops.PREC_FP16X3)
    with torch.no_grad():
        rgb_o, sig_o = O.eval_points_raw(O.unflatten(p[model.P:], sh_deg), pts.cpu())
    assert float((rgb.cpu() - rgb_o).abs().max() / rgb_o.abs().max()) < 1e-4


def test_training_reduces_loss():
    """a few hundred steps on a fixed synthetic batch: the loss must go down (teacher = constant colour)."""
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf import train as T
    from tests.support.mlp_stages import _rays
    R = 512
    o, d, v = _rays(R, 4)
    px = np.tile(np.array([[0.8, 0.3, 0.1]], np.float32), (R, 1))
    model = NerfModel(sh_deg=3, max_rays=R, sparsity_npoints=1000)
    model.init_params(1)
    state = T.TrainState(model)
    batch = {"rays": Rays(o, d, v), "pixels": px}
    first = T.train_step(model, state, batch, 5e-4, sync_stats=True)
    for _ in range(60):
        T.train_step(model, state, batch, 5e-4)
    last = T.train_step(model, state, batch, 5e-4, sync_stats=True)
    assert np.isfinite(last.loss) and last.loss < 0.5 * first.loss, (first, last)


def test_loss_and_grad_with_sigma_noise():
    """row a4 in training: the relu mask of sigma follows the NOISED pre-activation (train.py:70 -> models.py:274)."""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf import train as T
    sh_deg, R, nf = 3, 64, 128
    fc, ff, rays, px, t_rand, u, _ = _setup(sh_deg, R, nf, 0, 99)
    rs = np.random.RandomState(3)
    noise = (rs.normal(size=(R, 64)).astype(np.float32) * 0.5, rs.normal(size=(R, 64 + nf)).astype(np.float32) * 0.5)
    cfg = dict(num_coarse_samples=64, num_fine_samples=nf, near=2.0, far=6.0, white_bkgd=True, sparsity_weight=0.0,
               sparsity_length=0.05)
    stats_o, gc_o, gf_o = O.loss_and_grads(fc, ff, sh_deg, rays, px, cfg, t_rand, u, None, sigma_noise=noise)
    _, gc_p, gf_p = O.loss_and_grads(fc, ff, sh_deg, rays, px, cfg, t_rand, u, None)
    ref = np.concatenate([gc_o, gf_o])
    plain = np.concatenate([gc_p, gf_p])
    assert np.linalg.norm(ref - plain) / np.linalg.norm(plain) > 0.05   # noise changes the gradient visibly
    model = NerfModel(sh_deg=sh_deg, num_coarse_samples=64, num_fine_samples=nf, max_rays=R)
    model.set_params(np.concatenate([fc, ff]))
    state = T.TrainState(model)
    T.loss_and_grad(model, state, {"rays": Rays(*rays), "pixels": px}, sparsity_weight=0.0, randomized=True,
                    t_rand=t_rand, u=u, z_fine=stats_o["_z_fine"], sigma_noise=noise)
    torch.cuda.synchronize()
    g = state.grads.cpu().numpy()
    tot = float(np.linalg.norm(g - ref) / np.linalg.norm(ref))
    cos = float(np.dot(g, ref) / (np.linalg.norm(g) * np.linalg.norm(ref)))
    _record("sigma_noise_grad", dict(rel_l2=tot, cosine=cos))
    assert tot < 2e-2 and cos > 0.9995, (tot, cos)


@pytest.mark.gpu
def test_training_curve_matches_oracle():
    """N optimisation steps from identical parameters, batches and random draws: the GPU path (fp16 operands, fp32
    accumulate / parameters / Adam) against the fp32 CPU oracle (loss_fn + autograd + flax-Adam restatement).  Band:
    every step's loss (both levels) within 0.2 % of the oracle's (measured <= 8e-4), the accumulated parameter update
    with cosine > 0.99 and relative L2 < 0.15 (measured 0.994 / 0.107): Adam divides every gradient by its own running
    magnitude, so parameters whose gradient is near zero — where fp16 operand rounding decides the sign — move as far
    as all others; the update direction must not drift."""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf import train as T
    sh_deg, R, nf, nsp, steps, lr = 3, 48, 128, 64, 6, 5e-4
    fc, ff, rays, px, _, _, _ = _setup(sh_deg, R, nf, nsp, 91)
    cfg = dict(num_coarse_samples=64, num_fine_samples=nf, near=2.0, far=6.0, white_bkgd=True,
               sparsity_weight=1e-3, sparsity_length=0.05)
    model = NerfModel(sh_deg=sh_deg, num_coarse_samples=64, num_fine_samples=nf, max_rays=R, sparsity_npoints=nsp)
    p0 = np.concatenate([fc, ff])
    model.set_params(p0)
    state = T.TrainState(model)
    rs = np.random.RandomState(5)
    mo = [np.zeros_like(fc), np.zeros_like(ff)]
    vo = [np.zeros_like(fc), np.zeros_like(ff)]
    curve = []
    for step in range(steps):
        t_rand = rs.uniform(size=(R, 64)).astype(np.float32)
        u = rs.uniform(size=(R, nf)).astype(np.float32)
        sp = rs.uniform(-1.5, 1.5, size=(nsp, 3)).astype(np.float32)
        stats_o, gc, gf = O.loss_and_grads(fc, ff, sh_deg, rays, px, cfg, t_rand, u, sp)
        fc, mo[0], vo[0] = O.adam_step(fc, gc, mo[0], vo[0], float(step), lr)
        ff, mo[1], vo[1] = O.adam_step(ff, gf, mo[1], vo[1], float(step), lr)
        st = T.train_step(model, state, {"rays": Rays(*rays), "pixels": px}, lr, sparsity_weight=1e-3,
                          sparsity_length=0.05, t_rand=t_rand, u=u, sp_points=sp, sync_stats=True)
        curve.append(dict(step=step, loss_gpu=st.loss, loss_oracle=float(stats_o["loss"]),
                          loss_c_gpu=st.loss_c, loss_c_oracle=float(stats_o["loss_c"])))
        assert abs(st.loss - stats_o["loss"]) / stats_o["loss"] < 2e-3, curve[-1]
        assert abs(st.loss_c - stats_o["loss_c"]) / stats_o["loss_c"] < 2e-3, curve[-1]
    dp_gpu = model.params.cpu().numpy() - p0
    dp_ref = np.concatenate([fc, ff]) - p0
    rel = float(np.linalg.norm(dp_gpu - dp_ref) / np.linalg.norm(dp_ref))
    cos = float(np.dot(dp_gpu, dp_ref) / (np.linalg.norm(dp_gpu) * np.linalg.norm(dp_ref)))
    _record("training_curve_6_steps", dict(curve=curve, update_rel_l2=rel, update_cosine=cos))
    assert rel < 0.15 and cos > 0.99, (rel, cos)


@pytest.mark.gpu
def test_draw_uniforms_philox():
    """pob_draw_uniforms: U[0,1) jitter / inverse-CDF draws and U[-r,r) sparsity points of a step from one Philox
    launch: ranges, moments, determinism in (seed, step), fresh numbers per step, device-side step override."""
    from plenoctree_b200._lib import check, lib, ptr
    n_t, n_u, n_sp = 4096 * 64 + 3, 4096 * 128 + 1, 3 * 10000
    def draw(seed, step, step_dev=None):
        t = torch.empty(n_t, device="cuda"); u = torch.empty(n_u, device="cuda"); sp = torch.empty(n_sp, device="cuda")
        check(lib.pob_draw_uniforms(seed, float(step), ptr(step_dev), ptr(t), n_t, ptr(u), n_u, ptr(sp), n_sp, 1.5, None))
        torch.cuda.synchronize()
        return t, u, sp
    t, u, sp = draw(7, 3)
    for x in (t, u):
        assert float(x.min()) >= 0.0 and float(x.max()) < 1.0
        assert abs(float(x.mean()) - 0.5) < 2e-3 and abs(float(x.var()) - 1.0 / 12.0) < 2e-3
    assert float(sp.min()) >= -1.5 and float(sp.max()) < 1.5 and abs(float(sp.mean())) < 0.03
    assert abs(float(torch.corrcoef(torch.stack([t[:100000], u[:100000]]))[0, 1])) < 0.02     # streams are independent
    t2, u2, sp2 = draw(7, 3)
    assert torch.equal(t, t2) and torch.equal(u, u2) and torch.equal(sp, sp2)
    t3, _, _ = draw(7, 4)
    t4, _, _ = draw(8, 3)
    assert not torch.equal(t, t3) and not torch.equal(t, t4)
    t5, _, _ = draw(7, 999, step_dev=torch.tensor([4.0], device="cuda"))      # the device step wins
    assert torch.equal(t5, t3)


@pytest.mark.gpu
def test_graphed_train_step_matches_eager():
    """GraphedTrainStep (one CUDA graph per step: Philox draws keyed by the device-side step, kernels, Adam with
    lr / step from the device buffer) must reproduce the eager train_step sequence: parameters and Adam moments bit
    for bit, with the host queueing all replays ahead of the device (the (lr, step) staging ring is what is tested)."""
    from plenoctree_b200.nerf.models import NerfModel, Rays
    from plenoctree_b200.nerf import train as T
    R = 256
    fc, ff, rays, px, _, _, _ = _setup(3, R, 128, 0, 33)
    b12 = torch.from_numpy(np.concatenate([rays[0], rays[1], rays[2], px], axis=1)).cuda()
    lrs = [5e-4, 4e-4, 3e-4, 2e-4]
    outs = []
    for graphed in (False, True):
        model = NerfModel(sh_deg=3, max_rays=R, sparsity_npoints=1000)
        model.set_params(np.concatenate([fc, ff]))
        state = T.TrainState(model)
        if graphed:
            g = T.GraphedTrainStep(model, state, R)
            assert state.step == 0
            for lr in lrs:
                g.step(b12, lr)
        else:
            batch = {"rays": Rays(b12[:, 0:3], b12[:, 3:6], b12[:, 6:9]), "pixels": b12[:, 9:12]}
            for lr in lrs:
                T.train_step(model, state, batch, lr)
        torch.cuda.synchronize()
        assert state.step == len(lrs)
        outs.append((model.params.clone(), state.m.clone(), state.v.clone(), state.stats_raw.clone()))
    for name, a, b in zip(("params", "m", "v"), *[o[:3] for o in outs]):
        assert torch.equal(a, b), name
    # the loss sums are float atomics over the rays (order varies from launch to launch): equal to rounding only
    assert torch.allclose(outs[0][3], outs[1][3], rtol=1e-4, atol=1e-3)
    assert not torch.equal(outs[0][0], torch.from_numpy(np.concatenate([fc, ff])).cuda())

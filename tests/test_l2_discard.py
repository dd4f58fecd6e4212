"""POB_TRAIN_DISCARD_SAVED_GRADS: the weight gradient drops each dZ / dO tile from L2 once it has loaded it.

The flag only states that the caller will not read those tiles: every result the call returns, and every other byte
of the workspace, must be what the call leaves without it.  train_step (and GraphedTrainStep) always set it;
loss_and_grad keeps the tiles unless asked (keep_saved_tiles)."""
import pytest
import torch

from plenoctree_b200 import _lib
from tests.support.model_flags import FILL, NF, NSP, RAYS, _batch, _call, _equal_outside, _model, _saved_grad_ranges


def test_unknown_flag_bit_refused():
    """refused at the boundary, before any argument is looked at"""
    args = [None] * 8 + [1] + [None] * 3 + [0] + [None] * 7 + [_lib.PREC_FP16]
    rc = _lib.lib.pob_loss_and_grad_flags(*args, 2, None)
    assert rc != 0
    assert b"flags" in _lib.lib.pob_last_error()


CASES = {   # sh_deg, nf, nsp, near, far, loss_and_grad keywords
    "sh16_production": (3, NF, NSP, 2.0, 6.0, dict(sparsity_length=0.05, sparsity_radius=1.5)),
    "sh25_tt": (4, NF, NSP, 0.0, 4.0, dict(sparsity_length=0.2, sparsity_radius=5.0)),
    "single_level_sparsity": (3, 0, 3000, 2.0, 6.0, dict(sparsity_length=0.05, sparsity_radius=1.5)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_discard_leaves_results_and_other_regions(case):
    """gradient bit-identical; loss sums equal to the rounding of their float atomics; every workspace byte outside
    the DZ / DO images identical (a discard outside the loaded ranges would leave undefined bytes there)"""
    from plenoctree_b200.nerf import train as T
    sh_deg, nf, nsp, near, far, kw = CASES[case]
    model = _model(sh_deg, nf, nsp, near, far)
    state = T.TrainState(model)
    batch, _ = _batch(RAYS, 11)
    g0, s0, w0 = _call(model, state, batch, True, **kw)
    g1, s1, w1 = _call(model, state, batch, False, **kw)
    assert torch.isfinite(g0).all()
    assert torch.equal(g0, g1)
    assert torch.allclose(s0, s1, rtol=1e-5, atol=0)
    ranges = _saved_grad_ranges(model, RAYS, nsp > 0)
    assert _equal_outside(w0, w1, ranges)
    # the kept tiles were written: no DZ / DO range still holds the fill pattern everywhere
    for a, b in ranges:
        assert not bool((w0[a:b] == FILL).all())


@pytest.mark.gpu
def test_fp16x3_ignores_the_flag():
    """fp16x3's weight-gradient passes read dZ twice: the flag is accepted and changes nothing, DZ included"""
    from plenoctree_b200.nerf import train as T
    R = 1024
    model = _model(3, NF, 2000, R=R)
    state = T.TrainState(model)
    batch, _ = _batch(R, 12)
    g0, s0, w0 = _call(model, state, batch, True, precision=_lib.PREC_FP16X3)
    g1, s1, w1 = _call(model, state, batch, False, precision=_lib.PREC_FP16X3)
    assert torch.equal(g0, g1)
    assert torch.allclose(s0, s1, rtol=1e-5, atol=0)
    assert torch.equal(w0, w1)


@pytest.mark.gpu
def test_train_step_and_graph_match_a_keep_tiles_loop():
    """eager train_step and GraphedTrainStep (both discard) against loss_and_grad with the tiles kept + Adam:
    params, m and v bit for bit"""
    from plenoctree_b200.nerf import train as T
    R, nsp = 1024, 1000
    lrs = [5e-4, 4e-4, 3e-4]
    batch, b12 = _batch(R, 13)
    outs = []
    for mode in ("keep_loop", "train_step", "graphed"):
        model = _model(3, NF, nsp, R=R)
        state = T.TrainState(model)
        graph = T.GraphedTrainStep(model, state, R) if mode == "graphed" else None
        for lr in lrs:
            if mode == "graphed":
                graph.step(b12, lr)
            elif mode == "train_step":
                T.train_step(model, state, batch, lr)
            else:
                T.loss_and_grad(model, state, batch, keep_saved_tiles=True)
                _lib.check(_lib.lib.pob_adam_update_pe(
                    model.sh_deg, model.cfg.posenc, model.num_mlps, _lib.ptr(model.params), _lib.ptr(state.grads),
                    _lib.ptr(state.m), _lib.ptr(state.v), float(lr), float(state.step), None, 1.0, 0.0,
                    _lib.ptr(model.blobs[0]), _lib.ptr(model.blobs[1]), _lib.stream_ptr()))
                state.step += 1
        torch.cuda.synchronize()
        outs.append((model.params.clone(), state.m.clone(), state.v.clone()))
    for mode, o in zip(("train_step", "graphed"), outs[1:]):
        for name, a, b in zip(("params", "m", "v"), outs[0], o):
            assert torch.equal(a, b), f"{mode}: {name}"

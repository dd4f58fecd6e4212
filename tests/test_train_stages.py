"""Stage-by-stage parity of the training kernels (saving forward, data gradient, weight gradient + reduce).

tests/test_train.py compares whole gradients with an oracle, and its bars are loose by necessity: a pre-activation
within rounding distance of zero flips a ReLU mask between any two implementations (DESIGN.md "Gradient parity").
Here every intermediate of one pob_loss_and_grad call is read back from the caller-owned workspace (layouts.py:
train_workspace_views), and each stage is compared with an fp64 evaluation whose inputs are the GPU's own
previous-stage tiles and masks, with the fp16 operands the kernels use: no mask can flip between GPU and reference,
so the bars sit at the precision of the arithmetic (half an fp16 ulp for the rounding of the stored value plus an
fp32 accumulation allowance of a stated multiple of 2^-24 * sum |a*w|).
"""
import functools

import numpy as np
import pytest
import torch

from plenoctree_b200 import layouts as L
from tests.support.mlp_stages import CASES, Case, FP16, assert_stages, check_call, stage_case
from tests.support.records import record

_record = functools.partial(record, "parity_train_stages.json")


# =====================================================================================================================
# CPU: the workspace mirror and the tile / mask codecs
# =====================================================================================================================
def test_workspace_mirror_matches_library():
    """train_workspace_views() reproduces carve(): same total as pob_workspace_bytes over SH degrees, one and two
    levels, sparsity point counts and capacities; no buffer overlaps the next one for any call size."""
    from plenoctree_b200._lib import RenderConfig, lib
    from plenoctree_b200.nerf.models import ctypes_ref
    n = 0
    for sh in range(-1, 5):
        for nc, nf in ((3, 0), (64, 0), (3, 5), (64, 128), (64, 192), (256, 0), (100, 156)):
            for nsp in (0, 1, 300, 10000):
                for R in (1, 40, 4096):
                    cfg = RenderConfig(sh, nc, nf, 1, R, nsp)
                    want = int(lib.pob_workspace_bytes(ctypes_ref(cfg), 1))
                    for n_rays in sorted({1, (R + 1) // 2, R}):
                        for sp_on in (False, True):
                            v = L.train_workspace_views(cfg, n_rays, sp_on)
                            assert v["total"] == want, (sh, nc, nf, nsp, R)
                            assert len(v["levels"]) == (2 if nf else 1)
                            ext = []
                            for lv in v["levels"]:
                                for name in ("z", "rgbs", "weights", "comp", "disp", "acc", "G", "H", "E", "DZ",
                                             "DO", "mask"):
                                    off, shape = lv[name]
                                    ext.append((off, off + int(np.prod(shape)) * (1 if name in ("H", "E", "DZ", "DO") else 4)))
                                assert lv["M"] == n_rays * lv["N"] + (nsp if sp_on and lv is v["levels"][-1] else 0)
                                assert lv["rows"] % 512 == 0 and lv["rows"] >= lv["M"] > lv["rows"] - 512
                            ext.sort()
                            for (a0, a1), (b0, _) in zip(ext, ext[1:] + [(v["partials"][0], 0)]):
                                assert a0 % 1024 == 0 and a1 <= b0
                            n += 1
    assert n > 1000


def test_render_workspace_mirror_matches_library():
    """train_workspace_views(training=False) reproduces carve() for pob_render_rays: same total as
    pob_workspace_bytes(cfg, 0) (the sparsity point count must not change it), six buffers per level, no overlap."""
    from plenoctree_b200._lib import RenderConfig, lib
    from plenoctree_b200.nerf.models import ctypes_ref
    n = 0
    for sh in range(-1, 5):
        for nc, nf in ((3, 0), (64, 0), (3, 5), (64, 128), (64, 192), (256, 0), (100, 156)):
            for nsp in (0, 300):
                for R in (1, 40, 4096):
                    cfg = RenderConfig(sh, nc, nf, 1, R, nsp)
                    want = int(lib.pob_workspace_bytes(ctypes_ref(cfg), 0))
                    for n_rays in sorted({1, (R + 1) // 2, R}):
                        v = L.train_workspace_views(cfg, n_rays, True, training=False)
                        assert v["total"] == want, (sh, nc, nf, nsp, R)
                        assert len(v["levels"]) == (2 if nf else 1) and v["partials"] == []
                        ext = []
                        for lv in v["levels"]:
                            assert sorted(k for k in lv if isinstance(lv[k], tuple)) == \
                                ["acc", "comp", "disp", "rgbs", "weights", "z"]
                            assert lv["M"] == lv["M_rays"] == n_rays * lv["N"]
                            for name in ("z", "rgbs", "weights", "comp", "disp", "acc"):
                                off, shape = lv[name]
                                ext.append((off, off + int(np.prod(shape)) * 4))
                        ext.sort()
                        for (a0, a1), (b0, _) in zip(ext, ext[1:] + [(want, 0)]):
                            assert a0 % 1024 == 0 and a1 <= b0
                        n += 1
    assert n > 200


def test_mask_codec_roundtrip():
    """decode_mask inverts mlp_fwd's bit-shifting store (column 32c+2k -> bit 15-k, 32c+2k+1 -> bit 31-k)."""
    rs = np.random.RandomState(0)
    h = rs.normal(size=(300, 256)).astype(np.float16)
    h[h < 0.3] = 0
    h[7] = 0
    h[11] = 1
    words = L.encode_mask_reference(h)
    assert words[7].sum() == 0 and (words[11] == 0xFFFFFFFF).all()
    got = L.decode_mask(torch.from_numpy(words.view(np.int32)))
    assert got.dtype == torch.bool and np.array_equal(got.numpy(), h != 0)
    for j in range(256):                         # one column at a time: exactly one bit of one word
        e = np.zeros((1, 256), np.float16)
        e[0, j] = 1
        w = L.encode_mask_reference(e)[0]
        assert np.count_nonzero(w) == 1 and w[j // 32] == np.uint32(1) << np.uint32(L.mask_bit_of_column()[j % 32])
        assert L.decode_mask(torch.from_numpy(w.view(np.int32)[None]))[0].nonzero().flatten().tolist() == [j]


def test_tile_decoders_roundtrip():
    """the torch gather decoders read back the numpy tile packers (T layout for h, SW128 for dz / dO / posenc)."""
    rs = np.random.RandomState(1)
    m = [rs.normal(size=(128, 256)).astype(np.float16) for _ in range(3)]
    H = torch.from_numpy(np.stack([np.stack([L.pack_t_tile(x)] * 8) for x in m]))
    DZ = torch.from_numpy(np.stack([np.stack([L.pack_a_tile(x)] * 8) for x in m]))
    E = torch.from_numpy(np.stack([L.pack_a_tile(x[:, :64]) for x in m]))
    DO = torch.from_numpy(np.stack([L.pack_a_tile(x[:, :128]) for x in m]))
    cat = np.concatenate(m)
    assert np.array_equal(L.decode_h(H, 3).numpy(), cat)
    assert np.array_equal(L.decode_dz(DZ, 6).numpy(), cat)
    assert np.array_equal(L.decode_e(E).numpy(), cat[:, :64])
    assert np.array_equal(L.decode_do(DO).numpy(), cat[:, :128])


# =====================================================================================================================
# GPU: stage-isolated parity
# =====================================================================================================================


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_train_stages(case):
    stage_case(case, _record)


@pytest.mark.gpu
def test_train_stages_production_step():
    """the bench.py step: 4096 rays x (64 + 128) samples + 10 000 sparsity points, ~6 200 fine-level tiles (~47 per
    forward / dgrad CTA, ~890 per wgrad CTA): ring phases and accumulators carried across many tiles."""
    case = Case(3, 4096, 64, 128, 10000)
    from plenoctree_b200._lib import RenderConfig, lib
    from plenoctree_b200.nerf.models import ctypes_ref
    need = int(lib.pob_workspace_bytes(ctypes_ref(RenderConfig(3, 64, 128, 1, 4096, 10000)), 1))
    free, _ = torch.cuda.mem_get_info()
    if free < need + (6 << 30):
        pytest.skip(f"the production step needs {need / 2**30:.1f} GB of workspace + ~6 GB for the reference; "
                    f"{free / 2**30:.1f} GB free on this (shared) device")
    stage_case(case, _record, guard=False)


@pytest.mark.gpu
def test_workspace_hygiene():
    """nothing the call reads is left over from earlier contents of the workspace: a 0xFF-filled (NaN) and a zeroed
    workspace give bit-identical gradients, and a call after a larger one on the same workspace matches a fresh
    workspace bit for bit and passes the stage checks."""
    case = Case(3, 96, 64, 128, 300)
    outs = []
    for fill in (0xFF, 0):
        model = case.model()
        state, _ = case.run(model, fill=fill)
        outs.append((state.grads.clone(), state.stats_raw.clone()))
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.allclose(outs[0][1], outs[1][1], rtol=1e-4, atol=1e-3)   # float atomics over rays: rounding only
    small = Case(3, 96, 64, 128, 300, seed=23)
    model = small.model()
    small.run(model, n=96, fill=0xFF)
    state, ctx = small.run(model, n=40)                   # stale tiles of the 96-ray call behind and between
    fresh = small.model()
    state_f, _ = small.run(fresh, n=40, fill=0)
    assert torch.equal(state.grads, state_f.grads)
    res = check_call(model, state, ctx, FP16)
    _record("stale_workspace_R96_then_R40", res)
    assert_stages(res, FP16, "relu")

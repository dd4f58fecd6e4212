"""GPU parity of the fused point evaluator (csrc/mlp_fwd.cu) through the C ABI:
against the committed golden vectors of the reference's torch twin, against the CPU oracle on
seeded inputs, ragged sizes, and the extraction grid sweep."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "gpurun_out")

# Tolerances (relative to the largest reference magnitude of the compared tensor).
#   FP16X3: error-compensated operands, fp32-class accuracy -> 1e-4 (north-star bar is 1e-3)
#   FP16  : 10-bit-mantissa operands (TF32-class, like the reference's default-precision XLA GPU
#           path), fp32 accumulate -> the north-star bar itself, 1e-3 of the largest magnitude, elementwise on the
#           raw pre-activation outputs (measured on an H100: max 5.6e-4 .. 8.5e-4).
#           On arbitrary random points (no golden vectors; thousands of points, every SH degree) the largest single
#           error of the 10-layer fp16 chain reaches ~2e-3: those tests use TOL_FP16_ANY.
TOL_X3 = 1e-4
TOL_FP16 = 1e-3
TOL_FP16_ANY = 3e-3


def _record(name, payload):
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, "parity_eval_points.json")
    data = {}
    if os.path.exists(path):
        try:
            data = json.load(open(path))
        except Exception:
            data = {}
    data[name] = payload
    json.dump(data, open(path, "w"), indent=1)


def _relmax(got, want):
    return float(np.abs(got - want).max() / max(1e-9, np.abs(want).max()))


def _rms(got, want):
    return float(np.sqrt(((got - want) ** 2).mean()) / max(1e-9, np.sqrt((want ** 2).mean())))


def _blob(flat, sh_deg):
    from plenoctree_b200 import ops
    return ops.pack_weights(torch.from_numpy(flat).cuda(), sh_deg)


def test_pack_kernel_images_match_numpy_model():
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import layouts as L
    for sh_deg in (3, 4, 0):
        flat = O.init_flat_params(sh_deg, 5, bias_scale=0.1)
        blob = _blob(flat, sh_deg).cpu().numpy()
        ref = L.pack_reference(flat, sh_deg)
        lay = L.blob_layout(L.K_of(sh_deg))
        for key, nbytes in (("w_hi", lay["fwd_bytes"]), ("w_lo", lay["fwd_bytes"]), ("wt_hi", lay["bwd_bytes"])):
            got = blob[lay[key]:lay[key] + nbytes]
            assert np.array_equal(got, ref[key]), f"{key} image mismatch (sh_deg={sh_deg})"


@pytest.mark.parametrize("name,sh_deg", [("eval_points_sh16.npz", 3), ("eval_points_sh25.npz", 4)])
def test_eval_points_raw_vs_reference_golden(golden_dir, name, sh_deg):
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    g = np.load(os.path.join(golden_dir, name))
    seed = int(g["seed"])
    pts = torch.from_numpy(g["points"]).cuda()
    stats = {}
    for tag, s in (("fine", seed + 1), ("coarse", seed)):
        blob = _blob(O.init_flat_params(sh_deg, s, bias_scale=0.05), sh_deg)
        for prec, pname, tol in ((ops.PREC_FP16X3, "fp16x3", TOL_X3), (ops.PREC_FP16, "fp16", TOL_FP16)):
            rgb, sig = ops.eval_points_raw(blob, sh_deg, pts, precision=prec)
            torch.cuda.synchronize()
            rgb, sig = rgb.cpu().numpy(), sig.cpu().numpy()
            e = dict(rgb_max=_relmax(rgb, g[f"raw_rgb_{tag}"]), sig_max=_relmax(sig, g[f"raw_sigma_{tag}"]),
                     rgb_rms=_rms(rgb, g[f"raw_rgb_{tag}"]), sig_rms=_rms(sig, g[f"raw_sigma_{tag}"]))
            stats[f"{tag}_{pname}"] = e
            _record(f"{name}:{tag}:{pname}", e)
            assert e["rgb_max"] < tol and e["sig_max"] < tol, (tag, pname, e)


@pytest.mark.parametrize("m", [1, 127, 128, 129, 255, 256, 257, 1000, 148 * 256 * 2 + 77])
def test_ragged_sizes_and_sigma_only(m):
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    from plenoctree_b200._lib import check, lib, ptr, stream_ptr
    sh_deg = 3
    flat = O.init_flat_params(sh_deg, 11, bias_scale=0.05)
    blob = _blob(flat, sh_deg)
    rs = np.random.RandomState(m)
    pts_np = rs.uniform(-1.5, 1.5, size=(m, 3)).astype(np.float32)
    pts = torch.from_numpy(pts_np).cuda()
    for prec, tol in ((ops.PREC_FP16X3, TOL_X3), (ops.PREC_FP16, TOL_FP16_ANY)):
        rgb, sig = ops.eval_points_raw(blob, sh_deg, pts, precision=prec)
        _, sig_only = ops.eval_points_raw(blob, sh_deg, pts, want_rgb=False, precision=prec)
        # the same call into outputs with 64 guard rows behind them: detects out-of-bounds row writes
        guard = torch.full((m + 64, 48), 7.0, device="cuda")
        sguard = torch.full((m + 64,), 7.0, device="cuda")
        check(lib.pob_eval_points_raw(ptr(blob), sh_deg, ptr(pts), m, ptr(guard), ptr(sguard), prec, stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(sig, sig_only)
        assert torch.equal(guard[:m], rgb) and torch.equal(sguard[:m], sig[:, 0])
        assert bool((guard[m:] == 7.0).all()) and bool((sguard[m:] == 7.0).all())
        idx = np.unique(np.concatenate([np.arange(min(m, 300)), np.arange(max(0, m - 300), m)]))
        with torch.no_grad():
            rgb_o, sig_o = O.eval_points_raw(O.unflatten(flat, sh_deg), torch.from_numpy(pts_np[idx]))
        assert _relmax(rgb.cpu().numpy()[idx], rgb_o.numpy()) < tol
        assert _relmax(sig.cpu().numpy()[idx], sig_o.numpy()) < tol
        assert torch.isfinite(rgb).all() and torch.isfinite(sig).all()


def test_empty_input_is_a_noop():
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    blob = _blob(O.init_flat_params(3, 1), 3)
    rgb, sig = ops.eval_points_raw(blob, 3, torch.zeros((0, 3), device="cuda"))
    assert rgb.shape == (0, 48) and sig.shape == (0, 1)


@pytest.mark.parametrize("sh_deg", [0, 1, 2, 3, 4])
def test_eval_points_rgb_sigma_all_degrees(sh_deg):
    """NerfModel.eval_points: SH evaluation at the view direction + sigmoid/relu in the epilogue."""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    flat = O.init_flat_params(sh_deg, 21 + sh_deg, bias_scale=0.05)
    blob = _blob(flat, sh_deg)
    rs = np.random.RandomState(sh_deg)
    m = 777
    pts = rs.uniform(-1.5, 1.5, size=(m, 3)).astype(np.float32)
    vd = rs.normal(size=(m, 3)).astype(np.float32)
    vd /= np.linalg.norm(vd, axis=-1, keepdims=True)
    K = (sh_deg + 1) ** 2
    with torch.no_grad():
        raw_rgb, raw_sig = O.eval_points_raw(O.unflatten(flat, sh_deg), torch.from_numpy(pts))
        rgb_o = torch.sigmoid(O.eval_sh(sh_deg, raw_rgb.reshape(m, 3, K), torch.from_numpy(vd)))
        sig_o = torch.relu(raw_sig)
    for prec, tol in ((ops.PREC_FP16X3, TOL_X3), (ops.PREC_FP16, TOL_FP16_ANY)):
        rgb, sig = ops.eval_points(blob, sh_deg, torch.from_numpy(pts).cuda(), torch.from_numpy(vd).cuda(),
                                   precision=prec)
        torch.cuda.synchronize()
        assert np.abs(rgb.cpu().numpy() - rgb_o.numpy()).max() < tol
        assert _relmax(sig.cpu().numpy(), sig_o.numpy()) < tol


def test_grid_sweep_matches_reference_grid_formula():
    """octree/extraction.py:296-304 voxel centres, x-major flattening; slab offsets; bit-identical to
    evaluating the same coordinates as explicit points."""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    sh_deg = 3
    flat = O.init_flat_params(sh_deg, 31, bias_scale=0.05)
    blob = _blob(flat, sh_deg)
    reso = 32
    radius = torch.tensor([1.5, 1.3, 1.1])
    center = torch.tensor([0.1, -0.2, 0.05])
    scale = 0.5 / radius
    offset = 0.5 * (1.0 - center / radius)
    arr = (torch.arange(0, reso, dtype=torch.float32) + 0.5) / reso
    xx, yy, zz = (arr - offset[0]) / scale[0], (arr - offset[1]) / scale[1], (arr - offset[2]) / scale[2]
    grid = torch.stack(torch.meshgrid(xx, yy, zz, indexing="ij")).reshape(3, -1).T.contiguous()
    rgb_p, sig_p = ops.eval_points_raw(blob, sh_deg, grid.cuda(), precision=ops.PREC_FP16)
    rgb_g, sig_g = ops.eval_grid(blob, sh_deg, reso, offset.tolist(), scale.tolist(), want_rgb=True)
    torch.cuda.synchronize()
    assert torch.equal(sig_g, sig_p[:, 0]) and torch.equal(rgb_g, rgb_p)
    # slab [8, 20) equals the corresponding rows
    _, sig_s = ops.eval_grid(blob, sh_deg, reso, offset.tolist(), scale.tolist(), x0=8, nx=12)
    torch.cuda.synchronize()
    assert torch.equal(sig_s, sig_p[8 * reso * reso:20 * reso * reso, 0])


@pytest.mark.parametrize("S", [256, 32, 8, 5])
def test_cell_mean_extraction_step2(S):
    """octree/extraction.py:367-394: mean over samples_per_cell points of cat([raw_rgb, raw_sigma])."""
    from oracle import nerf_sh_oracle as O
    from plenoctree_b200 import ops
    sh_deg = 3
    flat = O.init_flat_params(sh_deg, 41, bias_scale=0.05)
    blob = _blob(flat, sh_deg)
    n_cells = 97
    rs = np.random.RandomState(S)
    centers = rs.uniform(-1.4, 1.4, size=(n_cells, 1, 3)).astype(np.float32)
    pts = (centers + rs.uniform(-0.003, 0.003, size=(n_cells, S, 3))).astype(np.float32)
    with torch.no_grad():
        rgb, sig = O.eval_points_raw(O.unflatten(flat, sh_deg), torch.from_numpy(pts.reshape(-1, 3)))
        want = torch.cat([rgb, sig], -1).reshape(n_cells, S, -1).mean(1).numpy()
    for prec, tol in ((ops.PREC_FP16X3, TOL_X3), (ops.PREC_FP16, TOL_FP16)):
        got = ops.eval_cells_mean(blob, sh_deg, torch.from_numpy(pts).cuda(), S, precision=prec)
        torch.cuda.synchronize()
        assert got.shape == (n_cells, 49)
        assert _relmax(got.cpu().numpy(), want) < tol

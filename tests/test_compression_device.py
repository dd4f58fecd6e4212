"""Palette quantisation of compressed trees on the device (octree/quantize.py, csrc/quantize.cu) against the numpy
median_cut / compress_tree, which stay the definition.

CPU: the restatement in tests/support/median_cut_ref.py matches median_cut bit for bit, every fixture tells the
host's orders from perturbed ones, and the CLI's --device cpu writes what the host compressor writes.
GPU: maps and palettes equal to the host's for edge cases, whole trees, the CLI, renders of the written files,
determinism across runs and SM counts, and the C entry point's refusals.
"""
import ctypes
import os

import numpy as np
import pytest

from plenoctree_b200.octree import compression as C
from tests.support.median_cut_ref import fixtures, median_cut_ref, same

VARIANTS = [dict(tie="reverse"), dict(axis="last")]
WEIGHTED_VARIANTS = [dict(total="sequential"), dict(cum="pairwise")]


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(fixtures()))
def test_restatement_matches_the_host_and_fixture_is_sensitive(name):
    pts, bits, w = fixtures()[name]
    host = C.median_cut(pts, bits, w)
    assert same(host, median_cut_ref(pts, bits, w))
    for v in VARIANTS + (WEIGHTED_VARIANTS if w is not None else []):
        assert not same(host, median_cut_ref(pts, bits, w, **v)), f"{name} does not separate {v}"


def test_reduceat_restatement_on_adversarial_segments():
    from tests.support.median_cut_ref import reduceat_sum
    rs = np.random.RandomState(3)
    for _ in range(40):
        n = int(rs.randint(1, 5000))
        a = rs.standard_normal(n) * np.exp(rs.standard_normal(n) * 8)
        starts = np.unique(np.r_[0, rs.randint(0, n, size=5)])
        ends = np.r_[starts[1:], n]
        for s, e, v in zip(starts, ends, np.add.reduceat(a, starts)):
            assert reduceat_sum(a[s:e]) == v


def _tiny_tree(seed=0, N=2, nodes=40, basis=4):
    rs = np.random.RandomState(seed)
    data = np.concatenate([rs.normal(0, 0.5, size=(nodes, N, N, N, 3 * basis)),
                           rs.uniform(0, 6, size=(nodes, N, N, N, 1))], axis=-1).astype(np.float16)
    return {"data": data, "child": np.zeros((nodes, N, N, N), np.int32), "n_internal": np.int64(nodes),
            "data_format": f"SH{basis}", "invradius3": np.ones(3, np.float32), "offset": np.zeros(3, np.float32)}


def _cli(tmp_path, z, device, extra=()):
    src = tmp_path / "tree.npz"
    np.savez_compressed(src, **z)
    out = tmp_path / f"out_{device}"
    C.main([str(src), "--out_dir", str(out), "--bits", "6", "--device", device, *extra])
    return dict(np.load(out / "tree.npz"))


def _same_files(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape, k
        assert x.tobytes() == y.tobytes(), k


def test_cli_cpu_writes_what_the_host_compressor_writes(tmp_path):
    z = _tiny_tree()
    got = _cli(tmp_path, z, "cpu", ("--retain", "1", "--weighted"))
    want = C.compress_tree(dict(z), 6, 2.0, 1, True)
    _same_files(got, want)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _dev(pts, bits, w=None):
    from plenoctree_b200.octree import quantize as Q
    return Q.median_cut(pts, bits, w)


def _check(pts, bits, w=None):
    host = C.median_cut(pts, bits, w)
    dev = _dev(pts, bits, w)
    assert np.array_equal(host[1], dev[1])
    assert host[0].tobytes() == dev[0].tobytes()
    assert host[0].astype(np.float16).tobytes() == dev[0].astype(np.float16).tobytes()


def _edge_cases():
    rs = np.random.RandomState(11)
    g = rs.normal(size=(3000, 3)).astype(np.float32)
    two = np.where(rs.rand(500, 3) < 0.5, 1.0, 2.0).astype(np.float32)
    heavy = g[:2000].copy()
    heavy[:1500, 0] = 0.25
    nan = g[:700].copy()
    nan[3, 1] = np.nan
    inf = g[:700].copy()
    inf[:, 2] = np.inf
    inf[::3, 2] = -np.inf
    c = {"n0": np.zeros((0, 3), np.float32), "n1": g[:1], "n2": g[:2], "identical": np.ones((257, 3), np.float32),
         "two_values": two, "heavy_duplicates": heavy, "nan": nan, "inf_axis": inf, "all_pos_inf": inf[1::3]}
    for name, (p, b, w) in fixtures().items():
        c["fx_" + name] = p
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [0, 1, 8, 15, 16])
@pytest.mark.parametrize("weighted", [False, True])
def test_median_cut_edge_cases_match_the_host(bits, weighted):
    rs = np.random.RandomState(bits)
    for name, p in _edge_cases().items():
        w = rs.uniform(0, 1, size=len(p)) if weighted and len(p) else None
        _check(p, bits, w)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(fixtures()))
def test_median_cut_fixtures_match_the_host(name):
    p, b, w = fixtures()[name]
    for bits in (b, 16):
        _check(p, bits, w)


@pytest.mark.gpu
def test_median_cut_weights_zero_tiny_huge_tied():
    rs = np.random.RandomState(5)
    p = (rs.randint(-8, 8, size=(4000, 3)) / 8).astype(np.float32)
    for w in (np.zeros(4000), np.full(4000, 1e-300), np.full(4000, 1e300), np.full(4000, 0.5),
              rs.uniform(0, 1, 4000) * 10.0 ** rs.randint(-200, 200, 4000)):
        for bits in (1, 8, 16):
            _check(p, bits, w)


@pytest.mark.gpu
def test_median_cut_above_2_pow_24_points():
    rs = np.random.RandomState(2)
    n = (1 << 24) + 4099
    p = (rs.randint(-512, 512, size=(n, 3)) / 64).astype(np.float32)
    _check(p, 2)


def _tree_dict(depth, sh_dim):
    import torch
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "scripts"))
    from bench_octree import build_tree
    tree, _, _ = build_tree(depth, torch.device("cuda"), sh_dim=sh_dim)
    return tree.state()


@pytest.mark.gpu
@pytest.mark.parametrize("sh_dim", [16, 25])
def test_compress_tree_matches_the_host(sh_dim):
    z = _tree_dict(4, sh_dim)
    for retain, weighted in ((0, False), (2, False), (0, True), (2, True)):
        want = C.compress_tree(dict(z), 16, 2.0, retain, weighted)
        got = C.compress_tree(dict(z), 16, 2.0, retain, weighted, device="cuda")
        _same_files(got, want)


@pytest.mark.gpu
def test_cli_auto_and_cuda_write_the_cpu_files_and_render_alike(tmp_path, capsys):
    import torch
    from plenoctree_b200.octree import Rays, VolumeRenderer, load_tree
    z = _tree_dict(3, 16)
    files = {}
    for dev in ("cpu", "auto", "cuda"):
        files[dev] = _cli(tmp_path, z, dev, ("--weighted",))
        files[dev + "_out"] = capsys.readouterr().out.replace(f"out_{dev}", "out")
    for dev in ("auto", "cuda"):
        _same_files(files[dev], files["cpu"])
        assert files[dev + "_out"] == files["cpu_out"]
    rs = np.random.RandomState(0)
    o = torch.from_numpy(rs.uniform(-0.2, 0.2, size=(4096, 3)).astype(np.float32) + np.float32([0, 0, -2.5]))
    d = torch.from_numpy(rs.normal(size=(4096, 3)).astype(np.float32) * 0.2 + np.float32([0, 0, 1]))
    d = d / d.norm(dim=1, keepdim=True)
    imgs = [VolumeRenderer(load_tree(files[k]), 1e-3).forward(Rays(o, d, d)) for k in ("cpu", "cuda")]
    assert torch.equal(imgs[0], imgs[1])


@pytest.mark.gpu
def test_deterministic_across_runs_and_sm_counts(monkeypatch):
    from plenoctree_b200.octree import quantize as Q
    rs = np.random.RandomState(9)
    p = (rs.randint(-64, 64, size=(3, 200000, 3)) / 32).astype(np.float32)
    w = rs.uniform(0, 1, size=200000)
    runs = []
    for sms in (None, "16", "66", "132", None):
        if sms is None:
            monkeypatch.delenv("POB_SM_COUNT", raising=False)
        else:
            monkeypatch.setenv("POB_SM_COUNT", sms)
        for weights in (None, w):
            pal, idx = Q.median_cut_batch(p, 16, weights)
            runs.append((weights is None, pal.cpu().numpy().tobytes(), idx.cpu().numpy().tobytes()))
    for r in runs[2:]:
        assert r == runs[0] if r[0] else r == runs[1]


@pytest.mark.gpu
def test_refusals_name_the_problem_and_launch_nothing(monkeypatch):
    import torch
    from plenoctree_b200._lib import lib
    n = 100
    pts = torch.zeros((1, n, 3), device="cuda")
    pal = torch.zeros((1 << 16) * 3, device="cuda")
    mp = torch.zeros(n, dtype=torch.int16, device="cuda")
    wsb = lib.pob_quantize_workspace_bytes(1, n, 0)
    ws = torch.zeros(wsb + 256, dtype=torch.uint8, device="cuda")
    P = lambda t: t.data_ptr()  # noqa: E731
    base = dict(points=P(pts), weights=None, nb=1, n=n, bits=4, pal=P(pal), map=P(mp), ws=P(ws), wsb=wsb)

    def call(**kw):
        a = dict(base, **kw)
        return lib.pob_quantize_median_cut(a["points"], a["weights"], a["nb"], a["n"], a["bits"], a["pal"], a["map"],
                                           a["ws"], a["wsb"], None)

    cases = [(dict(bits=-1), "bits must be in"), (dict(bits=17), "bits must be in"),
             (dict(points=None), "NULL pointer"), (dict(pal=None), "NULL pointer"), (dict(map=None), "NULL pointer"),
             (dict(ws=None), "NULL pointer"), (dict(ws=P(ws) + 8), "not 256-byte aligned"),
             (dict(wsb=wsb - 1), "smaller than"), (dict(n=1 << 31), "2^31"), (dict(nb=0), "n_basis >= 1")]
    torch.cuda.synchronize()
    n0 = lib.pob_launch_count()
    for kw, msg in cases:
        assert call(**kw) != 0
        assert msg in lib.pob_last_error().decode(), (kw, lib.pob_last_error())
    monkeypatch.setenv("POB_SM_COUNT", "3")
    assert call() != 0 and "POB_SM_COUNT" in lib.pob_last_error().decode()
    assert lib.pob_launch_count() == n0
    monkeypatch.delenv("POB_SM_COUNT")
    assert lib.pob_quantize_workspace_bytes(1, 1 << 31, 0) == -1
    # a valid call is timed under its own phase
    lib.pob_timing_enable(1)
    assert call() == 0
    torch.cuda.synchronize()
    ms, cnt = (ctypes.c_double * 6)(), (ctypes.c_longlong * 6)()
    assert lib.pob_timing_read_phases(6, ms, cnt) == 6
    lib.pob_timing_enable(0)
    assert cnt[5] == lib.pob_launch_count() - n0 and list(cnt[:5]) == [0] * 5

"""Compressed PlenOctrees (octree.compression output) rendered and evaluated as stored: n3tree.read_compressed /
load_tree, QuantTree, pob_octree_render_quant / pob_octree_render_depth_quant (csrc/octree.cu, QuantFetch).

- CPU: the loader reads what compression.compress_tree writes (quantised with retain 0 and 2, weighted and not, and
  --noquant), refuses bad files with a ValueError naming the key, and leaves ordinary tree.npz files to N3Tree.load;
  the ctypes descriptor matches the header field by field; the C entry points validate the descriptor.
- GPU: on the production-depth trees of tests/test_octree_march.py (and an SH25 shell built the same way), the
  compressed tree renders bit-identically (rgb, depth, acc and the visit counters) to the fp32 tree that
  compression.decompress_data rebuilds from the same file: explicit rays and perspective slabs, fast on and off.  The
  fp32 march is held to fp64 there, so identity carries that bound over.
- End to end: octree.evaluation on a compressed file prints the PSNR / SSIM of its decompressed tree.npz and writes the
  same images; octree.optimization refuses a compressed input.
"""
import ctypes
import os
import re

import numpy as np
import pytest

from oracle import octree_oracle as OO
from plenoctree_b200 import _lib
from plenoctree_b200.octree import compression as C
from plenoctree_b200.octree.n3tree import N3Tree, compressed_layout, read_compressed
from tests.support.octree_scenes import CASES, _pair, _state, _tree, f32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------------------
# files
# ---------------------------------------------------------------------------------------------------------


def _small_tree(N, fmt, seed):
    from tests.support.octree_scenes import _fill, _to_world
    rs = np.random.RandomState(seed)
    K = 1 if fmt == "RGBA" else int(fmt[2:])
    otree = OO.N3Tree(N=N, data_dim=4 if fmt == "RGBA" else 3 * K + 1, depth_limit=3, radius=(1.2, 0.9, 1.0),
                      center=(0.1, -0.1, 0.05), data_format=fmt)
    pts = _to_world(otree, rs.uniform(0.1, 0.9, size=(60, 3)))
    for _ in range(3):
        otree.refine_at(pts)
    _fill(otree, rs, tau_cell=1.5)
    return otree


def _roundtrip(tmp_path, d, name):
    path = str(tmp_path / name)
    np.savez_compressed(path, **d)
    return np.load(path)


# ---------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("retain,weighted", [(0, False), (2, False), (0, True), (2, True)])
def test_reads_quantised_files(tmp_path, retain, weighted):
    z = _state(_small_tree(2, "SH9", 3))
    c = C.compress_tree(dict(z), bits=4, sigma_thresh=2.0, retain=retain, weighted=weighted)
    got = read_compressed(_roundtrip(tmp_path, c, "c.npz"))
    assert got["layout"] == "quant" and repr(got["data_format"]) == "SH9"
    for k in ("child", "sigma", "quant_map", "quant_colors", "offset"):
        assert np.array_equal(got[k], c[k]), k
    assert np.array_equal(got["invradius"], c["invradius3"])
    assert got["quant_colors"].shape == (9 - retain, 16, 3) and got["quant_map"].dtype == np.uint16
    if retain:
        assert np.array_equal(got["data_retained"], c["data_retained"])
    else:
        assert got["data_retained"] is None
    # what the device tree decodes: palette[map] per basis function, the retained ones as stored
    dec = C.decompress_data(c)
    assert dec.shape == z["data"].shape and np.array_equal(dec[..., -1], got["sigma"])
    assert compressed_layout(z) is None


def test_reads_noquant_files(tmp_path):
    z = _state(_small_tree(3, "RGBA", 4))
    c = C.compress_tree(dict(z), quantize=False)
    got = read_compressed(_roundtrip(tmp_path, c, "c.npz"))
    assert got["layout"] == "noquant" and repr(got["data_format"]) == "RGBA"
    assert np.array_equal(got["data"], z["data"]) and np.array_equal(got["child"], z["child"])


def _bad(c, **changes):
    d = dict(c)
    for k, v in changes.items():
        if v is None:
            d.pop(k)
        else:
            d[k] = v
    return d


def test_refuses_bad_files_naming_the_key():
    z = _state(_small_tree(2, "SH4", 5))
    c = C.compress_tree(dict(z), bits=3, sigma_thresh=2.0, retain=1)
    read_compressed(c)
    qmap = c["quant_map"].copy()
    qmap[2].reshape(-1)[17] = 8                                            # palette has 2^3 entries
    with pytest.raises(ValueError, match=r"'quant_map'\[2\] holds index 8"):
        read_compressed(_bad(c, quant_map=qmap))
    with pytest.raises(ValueError, match="'quant_map'"):
        read_compressed(_bad(c, quant_map=c["quant_map"][:, :-1]))
    with pytest.raises(ValueError, match="'quant_colors'"):
        read_compressed(_bad(c, quant_map=c["quant_map"][:2]))             # one map plane short of the palettes
    with pytest.raises(ValueError, match="'quant_colors' .* do not add up"):
        read_compressed(_bad(c, quant_map=c["quant_map"][:2], quant_colors=c["quant_colors"][:2]))
    with pytest.raises(ValueError, match="'sigma'"):
        read_compressed(_bad(c, sigma=c["sigma"][:-1]))
    with pytest.raises(ValueError, match="'child'"):
        read_compressed(_bad(c, child=None))
    with pytest.raises(ValueError, match="'quant_colors'"):
        read_compressed(_bad(c, quant_colors=c["quant_colors"][:, :6]))
    with pytest.raises(ValueError, match="'data_retained'"):
        read_compressed(_bad(c, data_retained=c["data_retained"][:, :-1]))
    child = c["child"].copy()
    child.reshape(-1)[np.flatnonzero(child)[0]] = 10 ** 6
    with pytest.raises(ValueError, match="'child'"):
        read_compressed(_bad(c, child=child))
    n = C.compress_tree(dict(z), quantize=False)
    with pytest.raises(ValueError, match="'data'"):
        read_compressed(_bad(n, data=n["data"][..., :-1]))


def test_ordinary_files_stay_with_n3tree_load(tmp_path):
    """tree.npz is not a compressed layout (load_tree hands it to N3Tree.load unchanged); N3Tree.load refuses the
    compressed layouts with a message instead of failing on a missing bookkeeping key"""
    z = _state(_small_tree(2, "SH4", 6))
    assert compressed_layout(_roundtrip(tmp_path, z, "tree.npz")) is None
    for name, c in (("q.npz", C.compress_tree(dict(z), bits=2)), ("n.npz", C.compress_tree(dict(z), quantize=False))):
        _roundtrip(tmp_path, c, name)
        with pytest.raises(ValueError, match="compressed PlenOctree"):
            N3Tree.load(str(tmp_path / name))


def _header_struct(name):
    src = open(os.path.join(ROOT, "include", "plenoctree_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), src, flags=re.S).group(1)
    fields = []
    for decl in body.split(";"):
        decl = " ".join(decl.split())
        if not decl:
            continue
        m = re.match(r"(.*?)(\w+)(\[(\d+)\])?$", decl)
        fields.append((m.group(2), m.group(1).strip(), int(m.group(4)) if m.group(4) else None))
    return fields


def test_ctypes_descriptor_matches_the_header():
    want = _header_struct("pob_octree_quant")
    got = _lib.OctreeQuant._fields_
    assert [f[0] for f in want] == [g[0] for g in got]
    for (name, ctype, count), (_, ct) in zip(want, got):
        if "*" in ctype:
            assert ct is ctypes.c_void_p, name
        elif count is not None:
            assert ctype == "float" and ct._type_ is ctypes.c_float and ct._length_ == count, name
        elif ctype == "int64_t":
            assert ct is ctypes.c_int64, name
        else:
            assert ctype == "int" and ct is ctypes.c_int, name
    # natural C layout: ctypes pads like the compiler does
    assert ctypes.sizeof(_lib.OctreeQuant) == 96 and _lib.OctreeQuant.sigma_dev.offset == 40


def _desc(**kw):
    t = _lib.OctreeQuant()
    t.child_dev, t.sigma_dev, t.map_dev, t.palette_dev = 256, 512, 768, 1024
    t.n_nodes, t.N, t.basis_dim, t.format, t.retain, t.bits = 10, 2, 16, 1, 0, 16
    for k, v in kw.items():
        setattr(t, k, v)
    return t


@pytest.mark.parametrize("change,msg", [
    (dict(bits=0), "bits must be in [1, 16]"), (dict(bits=17), "bits must be in [1, 16]"),
    (dict(retain=-1), "retain must be in [0, basis_dim]"), (dict(retain=17), "retain must be in [0, basis_dim]"),
    (dict(N=9), "N must be in [2, 8]"), (dict(N=1), "N must be in [2, 8]"),
    (dict(n_nodes=2 ** 29), "leaf index must fit 32 bits"), (dict(format=2), "unsupported data format"),
    (dict(basis_dim=5), "SH basis_dim"), (dict(format=0), "RGBA trees have basis_dim 1"),
    (dict(retain=2), "retained pointer is NULL"), (dict(map_dev=None), "map/palette pointer is NULL"),
    (dict(sigma_dev=None), "child/sigma pointer is NULL")])
def test_c_entry_points_validate_the_descriptor(change, msg):
    from plenoctree_b200.octree.renderer import VolumeRenderer
    t = _desc(**change)
    o = VolumeRenderer(None)._opts(False)
    for fn, outs in ((_lib.lib.pob_octree_render_quant, (1024, None)),
                     (_lib.lib.pob_octree_render_depth_quant, (1024, 1024, 1024, None))):
        rc = fn(ctypes.byref(t), ctypes.byref(o), 256, 256, 256, 1, None, 0, 0, *outs, None)
        assert rc != 0
        assert msg in _lib.lib.pob_last_error().decode()


# ---------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------
CASE_IDS = [(name, i) for name in CASES for i in range(len(CASES[name]))]


def _rays(otree, pts, n=512, seed=0):
    rs = np.random.RandomState(seed)
    rad = 0.5 / otree.invradius.astype(np.float64)
    cen = (0.5 - otree.offset.astype(np.float64)) / otree.invradius.astype(np.float64)
    u = rs.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    o = cen + 3.0 * rad.max() * u
    tgt = pts[rs.randint(0, pts.shape[0], n)] + rs.uniform(-0.02, 0.02, (n, 3)) * rad
    d = (tgt - o) / np.linalg.norm(tgt - o, axis=1, keepdims=True)
    d[: n // 8] *= -1.0                                                   # some miss the box
    inside = pts[rs.randint(0, pts.shape[0], n // 2)]                     # rays starting in occupied cells
    di = rs.normal(size=inside.shape)
    di /= np.linalg.norm(di, axis=1, keepdims=True)
    return np.concatenate([o, inside]).astype(f32), np.concatenate([d, di]).astype(f32)


def _forward(r, o, d, fast, return_depth):
    import torch
    from plenoctree_b200.octree import Rays
    cnt = torch.zeros(2, dtype=torch.int64, device="cuda")
    with torch.no_grad():
        out = r.forward(Rays(torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(d)), fast=fast, counters=cnt,
                        return_depth=return_depth)
    return (out if return_depth else (out,)) + (cnt,)


@pytest.mark.gpu
@pytest.mark.parametrize("name,i", CASE_IDS)
def test_renders_bit_identical_to_the_decompressed_tree(name, i):
    import torch
    from tests.support.octree_scenes import CAM_F, CAM_H, CAM_W, _cameras
    from plenoctree_b200.octree import QuantTree, VolumeRenderer
    q, ref = _pair(name, i)
    assert isinstance(q, QuantTree) and q.retain == CASES[name][i][1] and q.bits == CASES[name][i][0]
    otree, pts = _tree(name)
    o, d = _rays(otree, pts)
    contributing = 0
    for step, bg in ((1e-5, 1.0), (1e-3, 0.25)):
        rq, rf = VolumeRenderer(q, step, bg), VolumeRenderer(ref, step, bg)
        for fast in (False, True):
            for depth in (False, True):
                got, want = _forward(rq, o, d, fast, depth), _forward(rf, o, d, fast, depth)
                for a, b in zip(got, want):
                    assert torch.equal(a, b), (step, fast, depth)
                contributing += int(got[-1][1])
        for c2w in _cameras(otree):
            with torch.no_grad():
                for fast in (False, True):
                    full = rq.render_persp(c2w, CAM_W, CAM_H, CAM_F, fast=fast, return_depth=True)
                    want = rf.render_persp(c2w, CAM_W, CAM_H, CAM_F, fast=fast, return_depth=True)
                    slabs = [rq.render_persp(c2w, CAM_W, CAM_H, CAM_F, fast=fast, rows=(a, b - a), return_depth=True)
                             for a, b in ((0, 7), (7, 8), (8, CAM_H))]
                    rgb = rq.render_persp(c2w, CAM_W, CAM_H, CAM_F, fast=fast)
                    assert torch.equal(rgb, want[0]), fast
                    for k in range(3):
                        assert torch.equal(full[k], want[k]), (fast, k)
                        assert torch.equal(torch.cat([s[k] for s in slabs]), want[k]), (fast, k)
    assert contributing > 1000


@pytest.mark.gpu
def test_device_bytes_and_refusals():
    import torch
    from plenoctree_b200.octree import Rays, VolumeRenderer
    q, ref = _pair("n2_d8_sh16", 0)
    fp32_bytes = ref.data[:ref.n_internal].nbytes + ref.child[:ref.n_internal].nbytes
    # SH16, 16 bits: 16 x 2 B of indices + 4 B sigma + 4 B child per leaf against 49 x 4 B + 4 B, plus 16 palettes of
    # 2^16 x 3 fp16 entries
    leaves = ref.n_internal * 8
    assert q.device_bytes() == leaves * (16 * 2 + 4 + 4) + 16 * 65536 * 6
    assert fp32_bytes == leaves * (49 * 4 + 4)
    r = VolumeRenderer(q, 1e-3)
    with pytest.raises(ValueError, match="read-only"):
        q.parameters()
    with pytest.raises(ValueError, match="read-only"):
        r.train_persp(np.eye(4, dtype=f32), torch.zeros(8, 8, 3), 8, 8, 10.0)
    # a --noquant file: an fp32 tree that renders like the original, and refuses gradients
    from plenoctree_b200.octree import load_tree
    from tests.support.octree_scenes import to_device_tree
    otree, pts = _tree("n3_d4_sh16")
    z = _state(otree)
    nq = load_tree(C.compress_tree(dict(z), quantize=False))
    orig = to_device_tree(otree)
    orig.data[:otree.n_internal] = torch.from_numpy(z["data"].astype(f32)).cuda()
    o, d = _rays(otree, pts, n=256)
    for a, b in zip(_forward(VolumeRenderer(nq, 1e-3), o, d, False, True),
                    _forward(VolumeRenderer(orig, 1e-3), o, d, False, True)):
        assert torch.equal(a, b)
    with pytest.raises(ValueError, match="read-only"):
        nq.parameters()
    nq.data.requires_grad_(True)
    rays = Rays(torch.from_numpy(o), torch.from_numpy(d), torch.from_numpy(d))
    with pytest.raises(ValueError, match="read-only"):
        VolumeRenderer(nq, 1e-3).forward(rays)


@pytest.mark.gpu
def test_ordinary_tree_loads_as_before(tmp_path):
    import torch
    from plenoctree_b200.octree import load_tree
    z = _state(_small_tree(2, "SH9", 8))
    np.savez_compressed(str(tmp_path / "tree.npz"), **z)
    a, b = N3Tree.load(str(tmp_path / "tree.npz")), load_tree(str(tmp_path / "tree.npz"))
    assert type(a) is type(b) is N3Tree and not b.read_only
    for k in ("data", "child", "parent_depth", "offset", "invradius"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    assert (a.n_internal, a.depth_limit, a.geom_resize_fact, repr(a.data_format)) == \
        (b.n_internal, b.depth_limit, b.geom_resize_fact, repr(b.data_format))


@pytest.mark.gpu
def test_cli_evaluation_of_compressed_files(tmp_path):
    """octree.evaluation on a quantised file prints the PSNR / SSIM of its decompressed tree saved as tree.npz and
    writes the same images and disparity maps; a --noquant file evaluates like the tree.npz it came from;
    octree.optimization refuses a compressed input"""
    import subprocess
    import sys
    from tests.support.octree_scenes import _cli, _scene
    common = _scene(tmp_path)
    z = dict(np.load(str(tmp_path / "tree.npz")))
    c = C.compress_tree(dict(z), bits=6, sigma_thresh=2.0, retain=1)
    np.savez_compressed(str(tmp_path / "q.npz"), **c)
    dec = dict(z, data=C.decompress_data(c).astype(np.float16))          # exact: every value is an fp16 value
    assert np.array_equal(dec["data"].astype(f32), C.decompress_data(c))
    np.savez_compressed(str(tmp_path / "dec.npz"), **dec)
    np.savez_compressed(str(tmp_path / "nq.npz"), **C.compress_tree(dict(z), quantize=False))

    def run(name):
        out = _cli("octree.evaluation", common + [
            "--input", str(tmp_path / f"{name}.npz"), "--write_images", str(tmp_path / f"img_{name}"),
            "--write_disp", str(tmp_path / f"disp_{name}"), "--write_vid", str(tmp_path / f"{name}.mp4")])
        line = [ln for ln in out.splitlines() if ln.startswith("Average PSNR")]
        assert len(line) == 1, out[-2000:]
        return line[0]
    q, d = run("q"), run("dec")
    assert q == d
    for sub in ("img", "disp"):
        names = sorted(os.listdir(tmp_path / f"{sub}_q"))
        assert names == sorted(os.listdir(tmp_path / f"{sub}_dec")) and len(names) == 2
        for f in names:
            assert (tmp_path / f"{sub}_q" / f).read_bytes() == (tmp_path / f"{sub}_dec" / f).read_bytes(), (sub, f)
    assert run("nq") == run("tree")
    r = subprocess.run([sys.executable, "-m", "octree.optimization"] + common + [
        "--input", str(tmp_path / "q.npz"), "--output", str(tmp_path / "o.npz"), "--num_epochs", "1"],
        capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert r.returncode != 0 and "compressed PlenOctree" in r.stderr, r.stderr[-2000:]
    assert not os.path.exists(tmp_path / "o.npz")

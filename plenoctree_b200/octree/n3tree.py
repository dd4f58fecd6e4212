"""Host-side mirror of `svox.N3Tree` for the calls the reference makes (octree/extraction.py:475-509,
octree/optimization.py:167-168,226-243, octree/compression.py:75-95 for the npz keys).

    reference call                                   here
    N3Tree(N, data_dim, init_refine, init_reserve,   N3Tree(...)  same keywords
           geom_resize_fact, depth_limit, radius,
           center, data_format, extra_data, map_location)
    tree[grid].refine()        extraction.py:343-352 tree[points].refine()   (pob_octree_query + sort/unique)
    tree.depths / max_depth    extraction.py:353,358 same
    tree[inds].sample(S)       extraction.py:370     same (uniform points inside the selected leaves)
    tree[inds] = rgba          extraction.py:394     same
    tree[:, -1:].relu_()       extraction.py:503     same
    tree.shrink_to_fit()/save  extraction.py:504-509 same; N3Tree.load for optimization.py:168

Tree arrays live on the GPU as torch tensors (device memory only); leaf lookup runs in the CUDA library
(pob_octree_query); the remaining bookkeeping (unique / sort / index arithmetic) is integer plumbing in torch.
There is no CPU path: constructing a tree needs a CUDA device.
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from .._lib import check, lib, ptr, stream_ptr

FORMAT_RGBA, FORMAT_SH = 0, 1


class DataFormat:
    """svox.helpers.DataFormat: 'RGBA' | 'SH<k>' ('SG<k>' / 'ASG<k>' are outside the scope of this path)."""

    def __init__(self, txt):
        txt = "RGBA" if txt is None else str(txt).strip()
        self.txt = txt
        up = txt.upper()
        if up == "RGBA" or up == "":
            self.format, self.basis_dim = FORMAT_RGBA, 1
        elif up.startswith("SH"):
            self.format, self.basis_dim = FORMAT_SH, int(up[2:])
            if self.basis_dim not in (1, 4, 9, 16, 25):
                raise ValueError(f"unsupported SH basis size in data format {txt!r}")
        else:
            raise NotImplementedError(f"data format {txt!r} (only RGBA and SH<k> are supported)")

    def data_dim(self):
        return 4 if self.format == FORMAT_RGBA else 3 * self.basis_dim + 1

    def __repr__(self):
        return "RGBA" if self.format == FORMAT_RGBA else f"SH{self.basis_dim}"


class N3Tree:
    read_only = False   # True for a tree loaded from a --noquant compressed file (load_tree)

    def __init__(self, N=2, data_dim=4, depth_limit=10, init_reserve=1, init_refine=0, geom_resize_fact=1.5,
                 radius=0.5, center=(0.5, 0.5, 0.5), data_format="RGBA", extra_data=None, map_location="cuda",
                 device=None):
        dev = torch.device(device if device is not None else map_location)
        if dev.type != "cuda":
            raise RuntimeError("plenoctree_b200 N3Tree lives on a CUDA device (there is no CPU path)")
        if extra_data is not None:
            raise NotImplementedError("extra_data (SG/ASG formats) is outside the scope of this path")
        self.device = dev
        self.N = int(N)
        self.data_format = DataFormat(data_format)
        self.data_dim = int(data_dim)
        if self.data_dim != self.data_format.data_dim():
            raise ValueError(f"data_dim {data_dim} does not match data format {self.data_format!r}")
        self.depth_limit = int(depth_limit)
        self.geom_resize_fact = float(geom_resize_fact)
        radius = np.broadcast_to(np.asarray(radius, dtype=np.float32), (3,))
        center = np.broadcast_to(np.asarray(center, dtype=np.float32), (3,))
        self.invradius = torch.from_numpy((np.float32(0.5) / radius).astype(np.float32)).to(dev)
        self.offset = torch.from_numpy((np.float32(0.5) * (np.float32(1.0) - center / radius)).astype(np.float32)).to(dev)
        cap = max(int(init_reserve), 1)
        Nn = self.N
        self.data = torch.zeros((cap, Nn, Nn, Nn, self.data_dim), dtype=torch.float32, device=dev)
        self.child = torch.zeros((cap, Nn, Nn, Nn), dtype=torch.int32, device=dev)
        self.parent_depth = torch.zeros((cap, 2), dtype=torch.int32, device=dev)
        self.n_internal = 1
        self.n_free = 0
        self.grad = None          # dense gradient buffer of `data` (training)
        self._leaves = None
        for _ in range(int(init_refine)):
            self.refine()

    # ---- C view -------------------------------------------------------------------------------------
    def c_struct(self):
        t = _lib.Octree()
        t.data_dev = self.data.data_ptr()
        t.child_dev = self.child.data_ptr()
        t.n_nodes = self.n_internal
        t.N = self.N
        t.data_dim = self.data_dim
        t.basis_dim = self.data_format.basis_dim
        t.format = self.data_format.format
        off = self.offset.cpu().numpy()
        inv = self.invradius.cpu().numpy()
        for a in range(3):
            t.offset[a] = float(off[a])
            t.invradius[a] = float(inv[a])
        return t

    # ---- queries ------------------------------------------------------------------------------------
    @property
    def capacity(self):
        return self.data.shape[0]

    def query_packed(self, points):
        """packed leaf index (node*N^3 + (i*N+j)*N+k) of the leaf holding each world point."""
        if not (isinstance(points, torch.Tensor) and points.is_cuda and points.dtype == torch.float32):
            raise ValueError("points must be a float32 CUDA tensor [n,3]")
        pts = points.reshape(-1, 3).contiguous()
        out = torch.empty(pts.shape[0], dtype=torch.int64, device=self.device)
        t = self.c_struct()
        check(lib.pob_octree_query(ctypes.byref(t), ptr(pts), pts.shape[0], ptr(out), stream_ptr()))
        return out

    def _all_leaves(self):
        if self._leaves is None:
            self._leaves = torch.nonzero(self.child[:self.n_internal] == 0)
        return self._leaves

    @property
    def n_leaves(self):
        return self._all_leaves().shape[0]

    @property
    def depths(self):
        """depth of every leaf, in leaf order (octree/extraction.py:358)."""
        return self.parent_depth[self._all_leaves()[:, 0], 1]

    @property
    def max_depth(self):
        return int(self.parent_depth[:self.n_internal, 1].max().item())

    def _pack(self, leaves):
        N = self.N
        return ((leaves[:, 0] * N + leaves[:, 1]) * N + leaves[:, 2]) * N + leaves[:, 3]

    def _corners_unit(self, leaves):
        """lower corner of each leaf cell in [0,1]^3 and the cell resolution N^(depth+1)."""
        N = self.N
        node = leaves[:, 0].clone()
        coord = leaves[:, 1:4].clone()
        mult = torch.ones_like(node)
        pd = self.parent_depth[:self.n_internal].long()
        depth = pd[node, 1]
        for _ in range(int(depth.max().item()) if depth.numel() else 0):
            pk = pd[node, 0]
            up = (node > 0).long()
            mult = mult * N
            pijk = torch.stack([(pk // (N * N)) % N, (pk // N) % N, pk % N], dim=1)
            coord = coord + pijk * (mult * up)[:, None]
            node = pk // (N ** 3)
        res = torch.pow(torch.tensor(float(N), device=self.device, dtype=torch.float64), (depth + 1).double())
        return (coord.double() / res[:, None]).float(), depth

    # ---- refinement ---------------------------------------------------------------------------------
    def _resize_add_cap(self, cap_needed):
        cap_needed = max(cap_needed, int(self.capacity * (self.geom_resize_fact - 1.0)))
        N, D = self.N, self.data_dim
        self.data = torch.cat([self.data, torch.zeros((cap_needed, N, N, N, D), dtype=torch.float32, device=self.device)])
        self.child = torch.cat([self.child, torch.zeros((cap_needed, N, N, N), dtype=torch.int32, device=self.device)])
        self.parent_depth = torch.cat([self.parent_depth, torch.zeros((cap_needed, 2), dtype=torch.int32, device=self.device)])
        self.grad = None

    def parameters(self):
        """svox N3Tree is an nn.Module whose only parameter is `data` (octree/optimization.py:187)."""
        if self.read_only:
            raise ValueError("a compressed PlenOctree is read-only: it has no trainable parameters")
        self.data.requires_grad_(True)
        return [self.data]

    @torch.no_grad()
    def refine(self, packed_sel=None):
        """N3Tree.refine: every selected leaf (sorted packed indices; None = all leaves) below depth_limit becomes an
        internal node appended at the end, in selection order; its N^3 cells inherit the leaf's data."""
        N3 = self.N ** 3
        if packed_sel is None:
            packed_sel = self._pack(self._all_leaves())
        knode = packed_sel // N3
        good = (self.parent_depth[knode, 1] < self.depth_limit) & (self.child.reshape(-1)[packed_sel] == 0)
        key = packed_sel[good]
        n_new = int(key.shape[0])
        if n_new == 0:
            return False
        filled = self.n_internal
        need = filled + n_new - self.capacity
        if need > 0:
            self._resize_add_cap(need)
        knode = key // N3
        new_idx = torch.arange(filled, filled + n_new, device=self.device, dtype=torch.int64)
        self.child[filled:filled + n_new] = 0
        self.child.reshape(-1)[key] = (new_idx - knode).to(torch.int32)
        self.data[filled:filled + n_new] = self.data.reshape(-1, self.data_dim)[key][:, None, None, None, :]
        self.parent_depth[filled:filled + n_new, 0] = key.to(torch.int32)
        self.parent_depth[filled:filled + n_new, 1] = self.parent_depth[knode, 1] + 1
        self.n_internal += n_new
        self._leaves = None
        return True

    # ---- indexing (the subset of N3TreeView the reference uses) ------------------------------------------
    def __getitem__(self, key):
        return N3TreeView(self, key)

    def __setitem__(self, key, value):
        N3TreeView(self, key).set(value)

    # ---- training helpers ---------------------------------------------------------------------------
    def grad_buffer(self):
        if self.grad is None or self.grad.shape != self.data.shape:
            self.grad = torch.zeros_like(self.data)
        return self.grad

    @staticmethod
    def check_sgd_options(momentum, nesterov):
        """torch.optim.SGD's checks on (momentum, nesterov), with its messages; -> momentum as a float."""
        momentum = float(momentum)
        if momentum < 0.0:
            raise ValueError(f"Invalid momentum value: {momentum}")
        if nesterov and momentum <= 0.0:
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        return momentum

    @torch.no_grad()
    def sgd_step(self, lr, momentum=0.0, nesterov=False):
        """torch.optim.SGD(lr, momentum, nesterov=nesterov).step() + zero_grad (octree/optimization.py:180-181,
        205-208).  With momentum the buffer (`_sgd_buf`, zero on first use, like torch's clone of the first gradient)
        lives with this tree across images and epochs; clone() and shrink_to_fit() drop it."""
        momentum = self.check_sgd_options(momentum, nesterov)
        g = self.grad_buffer()
        n = self.n_internal * self.N ** 3 * self.data_dim
        if momentum == 0.0:
            check(lib.pob_octree_sgd_step(ptr(self.data), ptr(g), n, float(lr), stream_ptr()))
            return
        if getattr(self, "_sgd_buf", None) is None or self._sgd_buf.shape != self.data.shape:
            self._sgd_buf = torch.zeros_like(self.data)
        check(lib.pob_octree_sgd_momentum_step(ptr(self.data), ptr(g), ptr(self._sgd_buf), n, float(lr), momentum,
                                               int(bool(nesterov)), stream_ptr()))

    @torch.no_grad()
    def adam_step(self, lr, eps=1e-8):
        """torch.optim.Adam(lr, eps).step() + zero_grad (octree/optimization.py:190-193; eps 1e-4 for fp16 trees)."""
        g = self.grad_buffer()
        if getattr(self, "_adam", None) is None or self._adam[0].shape != self.data.shape:
            self._adam = [torch.zeros_like(self.data), torch.zeros_like(self.data), 0]
        n = self.n_internal * self.N ** 3 * self.data_dim
        check(lib.pob_octree_adam_step(ptr(self.data), ptr(g), ptr(self._adam[0]), ptr(self._adam[1]), n, float(lr),
                                       float(self._adam[2]), float(eps), stream_ptr()))
        self._adam[2] += 1

    # ---- io -----------------------------------------------------------------------------------------
    def shrink_to_fit(self):
        n = self.n_internal
        self.data = self.data[:n].clone()
        self.child = self.child[:n].clone()
        self.parent_depth = self.parent_depth[:n].clone()
        self.grad = None
        self._leaves = None
        self._sgd_buf = None

    def clone(self, device=None):
        t = N3Tree.__new__(N3Tree)
        t.__dict__.update(self.__dict__)
        n = self.n_internal
        t.data = self.data[:n].clone()
        t.child = self.child[:n].clone()
        t.parent_depth = self.parent_depth[:n].clone()
        t.grad = None
        t._leaves = None
        t._adam = None
        t._sgd_buf = None
        return t

    def state(self):
        """payload of N3Tree.save (keys read back by octree/compression.py:75-95 and N3Tree.load)."""
        n = self.n_internal
        d = {
            "data_dim": np.int64(self.data_dim),
            "child": self.child[:n].cpu().numpy(),
            "parent_depth": self.parent_depth[:n].cpu().numpy(),
            "n_internal": np.int64(self.n_internal),
            "n_free": np.int64(self.n_free),
            "invradius3": self.invradius.cpu().numpy(),
            "offset": self.offset.cpu().numpy(),
            "depth_limit": np.int64(self.depth_limit),
            "geom_resize_fact": np.float64(self.geom_resize_fact),
            "data": self.data[:n].half().cpu().numpy(),  # svox stores fp16 ("save CPU memory")
            "data_format": repr(self.data_format),
        }
        return d

    def save(self, path, shrink=True, compress=True):
        if shrink:
            self.shrink_to_fit()
        (np.savez_compressed if compress else np.savez)(path, **self.state())

    @classmethod
    def load(cls, path, map_location="cuda", device=None):
        z = np.load(path)
        if compressed_layout(z) is not None:
            raise ValueError(f"{path} is a compressed PlenOctree (octree.compression output), a read-only final format: "
                             "it can be rendered and evaluated (octree.n3tree.load_tree) but not optimised or refined")
        dev = torch.device(device if device is not None else map_location)
        t = cls.__new__(cls)
        t.device = dev
        t.data_dim = int(z["data_dim"])
        t.child = torch.from_numpy(z["child"].astype(np.int32)).to(dev)
        t.N = int(t.child.shape[-1])
        t.parent_depth = torch.from_numpy(z["parent_depth"].astype(np.int32)).to(dev)
        t.n_internal = int(z["n_internal"])
        t.n_free = int(z["n_free"]) if "n_free" in z.files else 0
        if "invradius3" in z.files:
            inv = z["invradius3"].astype(np.float32)
        else:
            inv = np.full(3, float(z["invradius"]), dtype=np.float32)
        t.invradius = torch.from_numpy(inv).to(dev)
        t.offset = torch.from_numpy(z["offset"].astype(np.float32)).to(dev)
        t.depth_limit = int(z["depth_limit"])
        t.geom_resize_fact = float(z["geom_resize_fact"])
        t.data = torch.from_numpy(z["data"].astype(np.float32)).to(dev)
        t.data_format = DataFormat(str(z["data_format"]) if "data_format" in z.files else None)
        if "extra_data" in z.files:
            raise NotImplementedError("extra_data (SG/ASG formats) is outside the scope of this path")
        t.grad = None
        t._leaves = None
        return t

    def __repr__(self):
        return (f"plenoctree_b200.N3Tree(N={self.N}, data_dim={self.data_dim}, depth_limit={self.depth_limit}, "
                f"capacity:{self.n_internal - self.n_free}/{self.capacity}, data_format={self.data_format!r})")


# ---- compressed trees (octree.compression output) ----------------------------------------------------------
BOOKKEEPING = ("parent_depth", "geom_resize_fact", "n_free", "n_internal", "depth_limit")


def _files(z):
    return set(z.files) if hasattr(z, "files") else set(z.keys())


def compressed_layout(z):
    """'quant' for a quantised octree.compression file (it has quant_map), 'noquant' for a --noquant one (data, but
    none of the refine bookkeeping keys), None for an ordinary tree.npz."""
    files = _files(z)
    if "quant_map" in files:
        return "quant"
    if "data" in files and not files & set(BOOKKEEPING):
        return "noquant"
    return None


class QuantTree:
    """A compressed PlenOctree on the device, as octree.compression writes it: per leaf an fp32 sigma and, per basis
    function k, fp16 RGB coefficients (k < retain) or a uint16 index into that function's fp16 palette.  Read-only:
    VolumeRenderer.forward / render_persp draw it (pob_octree_render_quant); nothing trains or refines it."""
    read_only = True

    def __init__(self, child, sigma, qmap, palette, retained, offset, invradius, data_format, device):
        self.device = device
        self.data_format = data_format
        self.N = int(child.shape[-1])
        self.n_internal = int(child.shape[0])
        self.retain = 0 if retained is None else int(retained.shape[0])
        self.bits = int(palette.shape[1]).bit_length() - 1
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)   # noqa: E731
        self.child = up(child.astype(np.int32))
        self.sigma = up(sigma.astype(np.float32))
        self.map = up(qmap.astype(np.uint16).view(np.int16))           # uint16 bits (torch has no uint16 arithmetic)
        self.palette = up(palette.astype(np.float16))
        self.retained = None if retained is None else up(retained.astype(np.float16))
        self.offset = up(offset.astype(np.float32))
        self.invradius = up(invradius.astype(np.float32))

    def device_bytes(self):
        return sum(t.numel() * t.element_size() for t in (self.child, self.sigma, self.map, self.palette, self.retained)
                   if t is not None)

    def parameters(self):
        raise ValueError("a compressed PlenOctree is read-only: it has no trainable parameters")

    def c_struct(self):
        t = _lib.OctreeQuant()
        t.child_dev = self.child.data_ptr()
        t.n_nodes = self.n_internal
        t.N = self.N
        t.basis_dim = self.data_format.basis_dim
        t.format = self.data_format.format
        t.retain = self.retain
        t.bits = self.bits
        t.sigma_dev = self.sigma.data_ptr()
        t.map_dev = self.map.data_ptr() if self.map.numel() else None
        t.palette_dev = self.palette.data_ptr() if self.palette.numel() else None
        t.retained_dev = None if self.retained is None else self.retained.data_ptr()
        off = self.offset.cpu().numpy()
        inv = self.invradius.cpu().numpy()
        for a in range(3):
            t.offset[a] = float(off[a])
            t.invradius[a] = float(inv[a])
        return t

    def __repr__(self):
        return (f"plenoctree_b200.QuantTree(N={self.N}, nodes={self.n_internal}, data_format={self.data_format!r}, "
                f"bits={self.bits}, retain={self.retain})")


def _key(z, files, key):
    if key not in files:
        raise ValueError(f"compressed tree: missing key {key!r}")
    return np.asarray(z[key])


def _shape(arr, want, key):
    if tuple(arr.shape) != tuple(want):
        raise ValueError(f"compressed tree: {key!r} has shape {tuple(arr.shape)}, expected {tuple(want)}")


def _geometry(z, files):
    """-> child, offset, invradius, DataFormat of a compressed file, checked: child [n, N, N, N] with 2 <= N <= 8, fewer
    than 2^32 leaves, and every internal cell pointing at a node inside the array."""
    child = _key(z, files, "child")
    N = child.shape[-1] if child.ndim == 4 else 0
    if child.ndim != 4 or child.shape[1:] != (N, N, N) or not 2 <= N <= 8 or child.shape[0] < 1 \
            or not np.issubdtype(child.dtype, np.integer):
        raise ValueError(f"compressed tree: 'child' must be an integer array [n_nodes, N, N, N] with N in [2, 8], "
                         f"got {child.dtype} {tuple(child.shape)}")
    n = child.shape[0]
    if n * N ** 3 >= 2 ** 32:
        raise ValueError("compressed tree: 'child' has 2^32 or more leaves")
    c = child.reshape(n, -1).astype(np.int64)
    target = np.arange(n, dtype=np.int64)[:, None] + c
    if ((c != 0) & ((target <= 0) | (target >= n))).any():
        raise ValueError("compressed tree: 'child' points outside the node array")
    inv = (_key(z, files, "invradius3") if "invradius3" in files
           else np.full(3, float(_key(z, files, "invradius")), dtype=np.float32))
    off = _key(z, files, "offset")
    _shape(inv, (3,), "invradius3")
    _shape(off, (3,), "offset")
    fmt = DataFormat(str(z["data_format"]) if "data_format" in files else None)
    if "data_dim" in files and int(z["data_dim"]) != fmt.data_dim():
        raise ValueError(f"compressed tree: 'data_dim' {int(z['data_dim'])} does not match data format {fmt!r}")
    return child, off, inv, fmt


def read_compressed(z):
    """The host arrays of a compressed file (an npz or dict), checked -> dict(layout, child, offset, invradius,
    data_format) plus data (--noquant) or sigma, quant_map, quant_colors, data_retained (None when absent).  These
    arrays come from outside the program and index device memory, so a bad one raises ValueError naming the key:
    shapes against `child`, palette sizes against the data format, and every palette index inside its palette."""
    layout = compressed_layout(z)
    if layout is None:
        raise ValueError("not a compressed PlenOctree: no 'quant_map', and 'data' comes with the refine bookkeeping")
    files = _files(z)
    if "extra_data" in files:
        raise NotImplementedError("extra_data (SG/ASG formats) is outside the scope of this path")
    child, off, inv, fmt = _geometry(z, files)
    leaf_shape = child.shape
    out = dict(layout=layout, child=child, offset=off, invradius=inv, data_format=fmt)
    if layout == "noquant":
        data = _key(z, files, "data")
        _shape(data, leaf_shape + (fmt.data_dim(),), "data")
        out["data"] = data
        return out
    sigma = _key(z, files, "sigma")
    _shape(sigma, leaf_shape, "sigma")
    qmap = _key(z, files, "quant_map")
    colors = _key(z, files, "quant_colors")
    if qmap.ndim != 5 or not np.issubdtype(qmap.dtype, np.integer):
        raise ValueError(f"compressed tree: 'quant_map' must be an integer array [Kq, n_nodes, N, N, N], got "
                         f"{qmap.dtype} {tuple(qmap.shape)}")
    Kq = qmap.shape[0]
    _shape(qmap, (Kq,) + leaf_shape, "quant_map")
    C = colors.shape[1] if colors.ndim == 3 else 0
    if colors.ndim != 3 or C < 2 or C > 65536 or C & (C - 1):
        raise ValueError(f"compressed tree: 'quant_colors' must be [Kq, 2^bits, 3] with 1 <= bits <= 16, got "
                         f"{tuple(colors.shape)}")
    _shape(colors, (Kq, C, 3), "quant_colors")
    retained = None
    if "data_retained" in files:
        retained = np.asarray(z["data_retained"])
        _shape(retained, (retained.shape[0] if retained.ndim else 0,) + leaf_shape + (3,), "data_retained")
    retain = 0 if retained is None else retained.shape[0]
    if retain + Kq != fmt.basis_dim:
        raise ValueError(f"compressed tree: 'quant_colors' ({Kq}) and 'data_retained' ({retain}) basis functions do "
                         f"not add up to the {fmt.basis_dim} of data format {fmt!r}")
    for j in range(Kq):
        lo, hi = int(qmap[j].min()), int(qmap[j].max())
        if lo < 0 or hi >= C:
            raise ValueError(f"compressed tree: 'quant_map'[{j}] holds index {hi if hi >= C else lo}, outside the "
                             f"{C} entries of 'quant_colors'[{j}]")
    out.update(sigma=sigma, quant_map=qmap, quant_colors=colors, data_retained=retained)
    return out


def load_tree(src, map_location="cuda", device=None):
    """Any PlenOctree file (path, or an already loaded npz / dict): an ordinary tree.npz through N3Tree.load, a
    quantised octree.compression file as a QuantTree, a --noquant one as a read-only fp32 N3Tree without the refine
    bookkeeping.  Compressed files are checked by read_compressed first."""
    z = np.load(src) if isinstance(src, (str, bytes)) or hasattr(src, "__fspath__") else src
    if compressed_layout(z) is None:
        return N3Tree.load(src, map_location=map_location, device=device)
    c = read_compressed(z)
    dev = torch.device(device if device is not None else map_location)
    if dev.type != "cuda":
        raise RuntimeError("plenoctree_b200 trees live on a CUDA device (there is no CPU path)")
    child, fmt = c["child"], c["data_format"]
    if c["layout"] == "quant":
        return QuantTree(child, c["sigma"], c["quant_map"], c["quant_colors"], c["data_retained"], c["offset"],
                         c["invradius"], fmt, dev)
    t = N3Tree.__new__(N3Tree)
    t.device = dev
    t.N = int(child.shape[-1])
    t.data_format = fmt
    t.data_dim = fmt.data_dim()
    t.data = torch.from_numpy(c["data"].astype(np.float32)).to(dev)
    t.child = torch.from_numpy(child.astype(np.int32)).to(dev)
    t.parent_depth = None
    t.n_internal = int(child.shape[0])
    t.n_free = 0
    t.depth_limit = None
    t.geom_resize_fact = None
    t.invradius = torch.from_numpy(c["invradius"].astype(np.float32)).to(dev)
    t.offset = torch.from_numpy(c["offset"].astype(np.float32)).to(dev)
    t.grad = None
    t._leaves = None
    t.read_only = True
    return t


class N3TreeView:
    """The part of svox.N3TreeView the reference touches.  key is one of
         float tensor [n,3]           world points -> the leaves holding them   (.refine())
         integer tensor [n]           positions in leaf order                   (.sample(S), assignment)
         (slice(None), channel slice) every leaf, a channel range               (.relu_())"""

    def __init__(self, tree, key):
        self.tree = tree
        self.chan = slice(None)
        if isinstance(key, tuple):
            if len(key) != 2 or key[0] != slice(None):
                raise NotImplementedError("only tree[:, channels] tuple indexing is supported")
            self.chan = key[1]
            self.packed = tree._pack(tree._all_leaves())
        elif isinstance(key, torch.Tensor) and key.is_floating_point():
            self.packed = tree.query_packed(key.to(tree.device))
        elif isinstance(key, torch.Tensor):
            leaves = tree._all_leaves()[key.to(tree.device).long()]
            self.packed = tree._pack(leaves)
        elif isinstance(key, slice) and key == slice(None):
            self.packed = tree._pack(tree._all_leaves())
        else:
            raise NotImplementedError(f"unsupported N3Tree index {type(key)}")

    def _leaves(self):
        N = self.tree.N
        p = self.packed
        return torch.stack([p // N ** 3, (p // (N * N)) % N, (p // N) % N, p % N], dim=1)

    def refine(self):
        """octree/extraction.py:343-352: distinct selected leaves in sorted order (torch.unique(dim=0))."""
        return self.tree.refine(torch.unique(self.packed))

    @property
    def depths(self):
        return self.tree.parent_depth[self.packed // self.tree.N ** 3, 1]

    @property
    def values(self):
        return self.tree.data.reshape(-1, self.tree.data_dim)[self.packed][:, self.chan]

    def sample(self, n_samples, uniforms=None):
        """N3TreeView.sample (octree/extraction.py:370): [n, S, 3] uniform points inside each selected leaf, in
        world coordinates: corner + U[0,1) * cell length."""
        tree = self.tree
        corn_unit, depth = tree._corners_unit(self._leaves())
        corn = (corn_unit - tree.offset) / tree.invradius
        length = torch.pow(float(tree.N), -(depth.float() + 1.0))[:, None] / tree.invradius   # N^-(depth+1)
        if uniforms is None:
            uniforms = torch.rand((corn.shape[0], n_samples, 3), device=tree.device)
        return corn[:, None, :] + uniforms * length[:, None, :]

    @torch.no_grad()
    def set(self, value):
        flat = self.tree.data.reshape(-1, self.tree.data_dim)
        flat[self.packed, self.chan] = value.to(flat.dtype)

    @torch.no_grad()
    def relu_(self):
        flat = self.tree.data.reshape(-1, self.tree.data_dim)
        flat[self.packed, self.chan] = torch.relu(flat[self.packed, self.chan])
        return self

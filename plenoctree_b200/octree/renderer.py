"""Host-side mirror of `svox.VolumeRenderer` for the calls the reference makes.

    reference call                                                   here
    svox.VolumeRenderer(t, step_size=..., ndc=None)                  VolumeRenderer(tree, step_size, ...)
      octree/optimization.py:174, octree/nerf/utils.py:456
    svox.VolumeRenderer(t, ..., ndc=svox.NDCConfig(w, h, focal))     VolumeRenderer(tree, ..., ndc=NDCConfig(w, h,
      forward-facing (LLFF) scenes, octree/optimization.py:170-174    focal)): every call below marches NDC rays
    r.render_persp(c2w, height=H, width=W, fx=focal, fast=False)     render_persp (autograd-aware: the image
      octree/optimization.py:178,202, octree/nerf/utils.py:471        carries a grad_fn that fills tree.data.grad)
    r.forward(rays)  (svox.Rays(origins, dirs, viewdirs))            forward / __call__
    (no svox counterpart)                                            forward / render_persp(..., return_depth=True)
                                                                     -> (rgb, depth, acc) like nerf/utils.py's
                                                                     render_image; disparity(depth, acc) -> disp
    (no svox counterpart)                                            the same forward on a compressed tree
                                                                     (n3tree.load_tree -> QuantTree): no gradients
    mse.backward(); optimizer.step()  optimization.py:205-208        train_persp + N3Tree.sgd_step: one launch for
                                                                     render + clamp-MSE gradient + scatter

All arithmetic is in the CUDA library (csrc/octree.cu) behind include/plenoctree_b200.h; torch carries device
memory, streams and the autograd edge only.

NDC (forward-facing scenes): each world ray is turned into NDC as the reference's convert_to_ndc does (near = 1) and
its direction normalised for the march, while the SH view direction stays the world direction, as the LLFF NeRF-SH
model was trained.  render_persp and forward build these rays with pob_ndc_rays and march them through the
explicit-ray entry points (so gradients, depth and compressed trees work as for world rays); train_persp marches them
inside its fused launch (pob_octree_train_persp_ndc).  Depth is then a distance along the unit NDC direction.
"""
import collections
import ctypes

import numpy as np
import torch

from .. import _lib
from .._lib import check, lib, ptr, stream_ptr

Rays = collections.namedtuple("Rays", ("origins", "dirs", "viewdirs"))
NDCConfig = collections.namedtuple("NDCConfig", ("width", "height", "focal"))     # svox.NDCConfig


def scene_ndc(args, width, height, focal):
    """The NDCConfig the octree CLIs (extraction, optimization, evaluation) march a scene in, or None: a forward-facing
    LLFF scene, i.e. 'llff' in --config and not --spherify, the condition of the reference's extraction and evaluation
    (octree/extraction.py:187, octree/nerf/utils.py:451), under which its datasets hand NeRF-SH NDC rays.  The
    reference's optimization.py:170 tests 'llff' alone, so with --spherify it would optimise in NDC a tree that
    extraction built and evaluation renders in world space; every CLI here uses the one condition instead.  The
    background brightness stays svox's default 1.0 in NDC too, as the reference leaves it."""
    if "llff" in (getattr(args, "config", None) or "") and not getattr(args, "spherify", False):
        return NDCConfig(int(width), int(height), float(focal))
    return None


def make_camera(c2w, width, height, fx, fy=None):
    c2w = c2w.detach().cpu().numpy() if isinstance(c2w, torch.Tensor) else np.asarray(c2w)
    c2w = np.asarray(c2w, dtype=np.float32)
    if c2w.shape not in ((4, 4), (3, 4)):
        raise ValueError("c2w must be [4,4] or [3,4]")
    cam = _lib.Camera()
    for i in range(3):
        for j in range(4):
            cam.c2w[4 * i + j] = float(c2w[i, j])
    cam.fx = float(fx)
    cam.fy = float(fx if fy is None else fy)
    cam.width = float(int(width))
    cam.height = float(int(height))
    return cam


def camera_array(c2ws, width, height, fx, fy=None, device="cuda"):
    """[n,16] float32 device array of pob_camera records (pob_grid_weight_render)."""
    c2ws = np.asarray(c2ws, dtype=np.float32)
    n = c2ws.shape[0]
    out = np.zeros((n, 16), dtype=np.float32)
    out[:, :12] = c2ws[:, :3, :4].reshape(n, 12)
    out[:, 12] = fx
    out[:, 13] = fx if fy is None else fy
    out[:, 14] = int(width)
    out[:, 15] = int(height)
    return torch.from_numpy(out).to(device)


class _RenderFn(torch.autograd.Function):
    """autograd edge: d loss / d tree.data through pob_octree_render_backward."""

    @staticmethod
    def forward(ctx, data, renderer, rays, cam, row0, nrows, opts):
        ctx.renderer, ctx.rays, ctx.cam, ctx.row0, ctx.nrows = renderer, rays, cam, row0, nrows
        return renderer._render_raw(rays, cam, row0, nrows, opts)

    @staticmethod
    def backward(ctx, grad_out):
        r = ctx.renderer
        tree = r.tree
        g = torch.zeros_like(tree.data)
        t = tree.c_struct()
        o = r._opts(False)
        go = grad_out.reshape(-1, 3).contiguous().float()
        if ctx.cam is None:
            ro, rd, rv = ctx.rays
            check(lib.pob_octree_render_backward(ctypes.byref(t), ctypes.byref(o), ptr(ro), ptr(rd), ptr(rv),
                                                 ro.shape[0], None, 0, 0, ptr(go), ptr(g), stream_ptr()))
        else:
            check(lib.pob_octree_render_backward(ctypes.byref(t), ctypes.byref(o), None, None, None, 0,
                                                 ctypes.byref(ctx.cam), ctx.row0, ctx.nrows, ptr(go), ptr(g),
                                                 stream_ptr()))
        return g, None, None, None, None, None, None


class _RenderDepthFn(torch.autograd.Function):
    """autograd edge of (rgb, depth, acc): d loss / d tree.data through pob_octree_render_depth_backward (an output
    whose gradient autograd leaves undefined is passed as NULL, i.e. zero)."""

    @staticmethod
    def forward(ctx, data, renderer, rays, cam, row0, nrows, opts):
        ctx.set_materialize_grads(False)
        ctx.renderer, ctx.rays, ctx.cam, ctx.row0, ctx.nrows = renderer, rays, cam, row0, nrows
        return renderer._render_raw(rays, cam, row0, nrows, opts, return_depth=True)

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_acc):
        r = ctx.renderer
        tree = r.tree
        g = torch.zeros_like(tree.data)
        t = tree.c_struct()
        o = r._opts(False)
        flat = lambda x, c: None if x is None else x.reshape(-1, c).contiguous().float()   # noqa: E731
        gr, gd, ga = flat(g_rgb, 3), flat(g_depth, 1), flat(g_acc, 1)
        if ctx.cam is None:
            ro, rd, rv = ctx.rays
            src = (ptr(ro), ptr(rd), ptr(rv), ro.shape[0], None, 0, 0)
        else:
            src = (None, None, None, 0, ctypes.byref(ctx.cam), ctx.row0, ctx.nrows)
        check(lib.pob_octree_render_depth_backward(ctypes.byref(t), ctypes.byref(o), *src, ptr(gr), ptr(gd), ptr(ga),
                                                   ptr(g), stream_ptr()))
        return g, None, None, None, None, None, None


def disparity(depth, acc):
    """disp = acc / depth where 0 < acc / depth < 1e10 and acc > 1e-10, else 1e10: the rule of the NeRF-SH compositing
    kernel (render.cu, model_utils.volumetric_rendering), so a ray that misses the box gets 1e10."""
    disp = acc / depth
    return torch.where((disp > 0) & (disp < 1e10) & (acc > 1e-10), disp, torch.full_like(disp, 1e10))


class VolumeRenderer:
    def __init__(self, tree, step_size=1e-3, background_brightness=1.0, ndc=None):
        self.tree = tree
        self.step_size = float(step_size)
        self.background_brightness = float(background_brightness)
        self.ndc = None
        if ndc is not None:
            ndc = NDCConfig(*ndc)
            self.ndc = _lib.Ndc(float(ndc.width), float(ndc.height), float(ndc.focal))

    def _ndc_rays(self, rays, cam, row0, nrows):
        """pob_ndc_rays: the NDC rays of explicit world rays (cam None) or of a camera's pixel-row slab"""
        dev = self.tree.device
        if cam is None:
            ro, rd, rv = rays
            n = ro.shape[0]
            src = (ptr(ro), ptr(rd), ptr(rv), n, None, 0, 0)
        else:
            n = nrows * int(cam.width)
            src = (None, None, None, 0, ctypes.byref(cam), row0, nrows)
        out = [torch.empty((n, 3), dtype=torch.float32, device=dev) for _ in range(3)]
        check(lib.pob_ndc_rays(ctypes.byref(self.ndc), *src, *map(ptr, out), stream_ptr()))
        return tuple(out)

    def _opts(self, fast):
        o = _lib.OctreeOpts()
        o.step_size = self.step_size
        o.background_brightness = self.background_brightness
        o.sigma_thresh = 1e-2 if fast else 0.0   # svox VolumeRenderer._get_options(fast)
        o.stop_thresh = 1e-2 if fast else 0.0
        return o

    def _render_raw(self, rays, cam, row0, nrows, opts, counters=None, return_depth=False):
        """-> rgb [n,3] (explicit rays) / [nrows,W,3] (camera slab); with return_depth (rgb, depth, acc), the last two
        of the same shape with 1 channel"""
        tree = self.tree
        t = tree.c_struct()
        quant = isinstance(t, _lib.OctreeQuant)      # a compressed tree (n3tree.QuantTree)
        if cam is None:
            ro, rd, rv = rays
            shape = (ro.shape[0],)
            src = (ptr(ro), ptr(rd), ptr(rv), ro.shape[0], None, 0, 0)
        else:
            shape = (nrows, int(cam.width))
            src = (None, None, None, 0, ctypes.byref(cam), row0, nrows)
        out = torch.empty(shape + (3,), dtype=torch.float32, device=tree.device)
        if not return_depth:
            fn = lib.pob_octree_render_quant if quant else lib.pob_octree_render
            check(fn(ctypes.byref(t), ctypes.byref(opts), *src, ptr(out), ptr(counters), stream_ptr()))
            return out
        depth = torch.empty(shape + (1,), dtype=torch.float32, device=tree.device)
        acc = torch.empty(shape + (1,), dtype=torch.float32, device=tree.device)
        fn = lib.pob_octree_render_depth_quant if quant else lib.pob_octree_render_depth
        check(fn(ctypes.byref(t), ctypes.byref(opts), *src, ptr(out), ptr(depth), ptr(acc), ptr(counters), stream_ptr()))
        return out, depth, acc

    @staticmethod
    def _f32(t, dev):
        if isinstance(t, np.ndarray):
            t = torch.from_numpy(t)
        return t.to(device=dev, dtype=torch.float32).reshape(-1, 3).contiguous()

    def _check_trainable(self, what):
        if getattr(self.tree, "read_only", False):
            raise ValueError(f"{what} needs gradients, and a compressed PlenOctree is read-only (it renders forward "
                             "only)")

    def _render(self, rays, cam, row0, nrows, opts, counters, return_depth):
        data = getattr(self.tree, "data", None)      # a QuantTree has none
        if torch.is_grad_enabled() and data is not None and data.requires_grad:
            self._check_trainable("rendering with tree.data.requires_grad")
            fn = _RenderDepthFn if return_depth else _RenderFn
            return fn.apply(data, self, rays, cam, row0, nrows, opts)
        return self._render_raw(rays, cam, row0, nrows, opts, counters, return_depth)

    def forward(self, rays, fast=False, counters=None, return_depth=False):
        """VolumeRenderer.forward(rays: Rays(origins, dirs, viewdirs)) -> rgb [n,3].  return_depth=True -> (rgb [n,3],
        depth [n,1], acc [n,1]): acc = sum of the compositing weights (background excluded), depth = their sum over
        the segment midpoints z, as the parameter of origin + z * dirs (csrc/octree.cu, trace_forward)."""
        dev = self.tree.device
        r3 = (self._f32(rays.origins, dev), self._f32(rays.dirs, dev), self._f32(rays.viewdirs, dev))
        if self.ndc is not None:
            r3 = self._ndc_rays(r3, None, 0, 0)
        return self._render(r3, None, 0, 0, self._opts(fast), counters, return_depth)

    __call__ = forward

    def render_persp(self, c2w, width=256, height=256, fx=1111.111, fy=None, fast=False, cuda=True, rows=None,
                     counters=None, return_depth=False):
        """render_persp(c2w, width, height, fx) -> [H,W,3] (octree/optimization.py:178,202).  rows=(row0,nrows)
        renders one pixel-row slab (rank sharding of evaluation renders).  return_depth=True -> (rgb [H,W,3],
        depth [H,W,1], acc [H,W,1]), depth along the camera axis (the distance along the pixel's unit ray times
        1 / |(x, y, -1)|), the quantity disparity() turns into nerf_sh.eval's disparity maps."""
        cam = make_camera(c2w, width, height, fx, fy)
        row0, nrows = (0, int(height)) if rows is None else rows
        if self.ndc is None:
            return self._render(None, cam, row0, nrows, self._opts(fast), counters, return_depth)
        out = self._render(self._ndc_rays(None, cam, row0, nrows), None, 0, 0, self._opts(fast), counters,
                           return_depth)
        shape = (nrows, int(width), -1)
        return tuple(x.reshape(shape) for x in out) if return_depth else out.reshape(shape)

    def train_persp(self, c2w, gt, width, height, fx, fy=None, rows=None, want_image=False, sq_err=None):
        """One training image of octree.optimization (octree/optimization.py:201-207) in ONE kernel: render the slab,
        mse = mean((clamp(im,0,1) - gt)^2), scatter d mse / d data into tree.grad_buffer().  gt: [H,W,3] (or the
        slab's rows).  Returns (sum of squared errors as a 1-element float64 device tensor, image or None)."""
        self._check_trainable("train_persp")
        tree = self.tree
        cam = make_camera(c2w, width, height, fx, fy)
        H, W = int(height), int(width)
        row0, nrows = (0, H) if rows is None else rows
        gt = gt.to(device=tree.device, dtype=torch.float32)
        if gt.shape[0] == H and nrows != H:
            gt = gt[row0:row0 + nrows]
        gt = gt.reshape(-1, 3).contiguous()
        if gt.shape[0] != nrows * W:
            raise ValueError("gt does not match the rendered slab")
        g = tree.grad_buffer()
        if sq_err is None:
            sq_err = torch.zeros(1, dtype=torch.float64, device=tree.device)
        out = torch.empty((nrows, W, 3), dtype=torch.float32, device=tree.device) if want_image else None
        t = tree.c_struct()
        o = self._opts(False)
        src = (ctypes.byref(cam),) if self.ndc is None else (ctypes.byref(cam), ctypes.byref(self.ndc))
        fn = lib.pob_octree_train_persp if self.ndc is None else lib.pob_octree_train_persp_ndc
        check(fn(ctypes.byref(t), ctypes.byref(o), *src, row0, nrows, ptr(gt), 1.0 / float(H * W * 3), ptr(g),
                 ptr(sq_err), ptr(out), stream_ptr()))
        return sq_err, out

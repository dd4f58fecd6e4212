"""Host-side mirror of the reference's NeRF-SH model interface for the hot path.

    reference                                              here
    nerf_sh/nerf/models.py::NerfModel.__call__   (:216)    NerfModel.__call__
    nerf_sh/nerf/models.py::eval_points_raw      (:143)    NerfModel.eval_points_raw
    nerf_sh/nerf/models.py::eval_points          (:183)    NerfModel.eval_points
    nerf_sh/nerf/models.py::get_model_state      (:38)     get_model_state
    nerf_sh/train.py::train_step                 (:51)     plenoctree_b200.nerf.train.train_step

All arithmetic happens in the CUDA library behind the C ABI (include/plenoctree_b200.h); torch is
used for device memory, streams and (in train.py) the NCCL all-reduce only.
"""
import math

import numpy as np
import torch

from .. import _lib
from .._lib import PREC_FP16, RenderConfig, check, lib, posenc_ref, posenc_struct, ptr, stream_ptr
from ..layouts import K_of, posenc_width, posenc_valid

from .rays import Rays  # noqa: F401  (nerf_sh/nerf/utils.py:53)


def _cuda_f32(t, name, shape_last=None):
    if isinstance(t, np.ndarray):
        t = torch.from_numpy(np.ascontiguousarray(t, dtype=np.float32)).cuda()
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32):
        raise ValueError(f"{name} must be a float32 CUDA tensor")
    t = t.contiguous()
    if shape_last is not None and t.shape[-1] != shape_last:
        raise ValueError(f"{name} must have last dimension {shape_last}")
    return t


def glorot_uniform_flat(sh_deg, generator=None, posenc=None):
    """Dense kernel_init=glorot_uniform, zero bias (nerf_sh/nerf/model_utils.py:63-65); the fan-in of Dense_0 and
    Dense_5 follows the posenc width of `posenc` (min_deg, max_deg, legacy; None = the default)."""
    from ..layouts import layer_dims
    parts = []
    for cin, cout in layer_dims(K_of(sh_deg), posenc_width(posenc)):
        a = math.sqrt(6.0 / (cin + cout))
        parts.append((torch.rand(cin * cout, generator=generator) * 2 - 1) * a)
        parts.append(torch.zeros(cout))
    return torch.cat(parts).float()


class NerfModel:
    """Nerf NN Model with both coarse and fine MLPs (nerf_sh/nerf/models.py:52-348), SH output head.

    Parameters live in one flat fp32 CUDA tensor `params` = [MLP_0 | MLP_1], each MLP in reference
    order Dense_0..Dense_9 (kernel [in,out] then bias)."""

    def __init__(self, sh_deg=3, num_coarse_samples=64, num_fine_samples=128, near=2.0, far=6.0,
                 white_bkgd=True, lindisp=False, max_rays=4096, sparsity_npoints=0, device="cuda",
                 precision=PREC_FP16, noise_std=None, sigma_activation="relu", min_deg_point=0, max_deg_point=10,
                 legacy_posenc_order=False, net_activation="relu"):
        from .flags import check_samples, net_activation_code, sigma_activation_code
        if not (-1 <= sh_deg <= 4):
            raise ValueError("sh_deg must be in [-1, 4]")
        check_samples(num_coarse_samples, num_fine_samples)
        # flags min_deg_point / max_deg_point / legacy_posenc_order (nerf_sh/nerf/models.py:121-126): the point
        # encoder of both MLPs, which also sets the shapes of Dense_0 [W, 256] and Dense_5 [256 + W, 256]
        self.posenc = (int(min_deg_point), int(max_deg_point), bool(legacy_posenc_order))
        if not posenc_valid(self.posenc):
            raise ValueError("posenc degrees must satisfy 0 <= min_deg_point <= max_deg_point <= 10")
        # flag net_activation (nerf_sh/nerf/models.py:362, model_utils.py:69): the activation after every trunk layer;
        # it rides in the same descriptor, so the parameters and the packed blob do not depend on it
        self.net_activation = str(net_activation)
        self.net_act_code = net_activation_code(net_activation)
        self._posenc_struct = posenc_struct(self.posenc, self.net_act_code)   # None (NULL): default encoder, relu
        # flag sigma_activation (nerf_sh/nerf/models.py:280-281): relu or softplus of the ray samples' raw sigma and
        # of eval_points; raw sigma (eval_points_raw, extraction) and the sparsity term never take it
        self.sigma_activation = str(sigma_activation)
        self.sigma_act_code = sigma_activation_code(sigma_activation)
        self.sh_deg = sh_deg
        self.num_coarse_samples = int(num_coarse_samples)
        self.num_fine_samples = int(num_fine_samples)
        self.near, self.far = float(near), float(far)
        self.white_bkgd = bool(white_bkgd)
        self.lindisp = bool(lindisp)
        self.max_rays = int(max_rays)
        self.sparsity_npoints = int(sparsity_npoints)
        self.precision = precision
        self.noise_std = noise_std   # flag noise_std (nerf_sh/nerf/utils.py:137-142); None = no density noise
        self.device = torch.device(device)
        self.num_mlps = 2 if self.num_fine_samples > 0 else 1
        self.P = int(lib.pob_param_count_pe(sh_deg, posenc_ref(self._posenc_struct)))
        self.params = torch.zeros(self.num_mlps * self.P, dtype=torch.float32, device=self.device)
        nb = int(lib.pob_packed_bytes(sh_deg))
        self.blobs = [torch.zeros(nb, dtype=torch.uint8, device=self.device) for _ in range(self.num_mlps)]
        self.cfg = RenderConfig(sh_deg, self.num_coarse_samples, self.num_fine_samples, int(self.white_bkgd),
                                self.max_rays, self.sparsity_npoints)
        self.cfg.sigma_activation = self.sigma_act_code
        self.cfg.posenc = posenc_ref(self._posenc_struct)
        self._ws = {}
        # un-jittered depth table, computed with the reference expression (model_utils.py:125-129)
        t_vals = torch.linspace(0.0, 1.0, self.num_coarse_samples, dtype=torch.float32)
        if self.lindisp:
            zb = 1.0 / (1.0 / self.near * (1.0 - t_vals) + 1.0 / self.far * t_vals)
        else:
            zb = self.near * (1.0 - t_vals) + self.far * t_vals
        self.z_base = zb.to(self.device)
        # deterministic u of piecewise_constant_pdf (model_utils.py:259-262)
        if self.num_fine_samples > 0:
            self.u_table = torch.linspace(0.0, 1.0 - float(np.finfo(np.float32).eps), self.num_fine_samples,
                                          dtype=torch.float32).to(self.device)
        else:
            self.u_table = None

    # ---- parameters --------------------------------------------------------------------------
    def init_params(self, seed=20200823):
        g = torch.Generator().manual_seed(seed)
        flat = torch.cat([glorot_uniform_flat(self.sh_deg, g, self.posenc) for _ in range(self.num_mlps)])
        self.set_params(flat)

    def set_params(self, flat):
        flat = torch.as_tensor(flat, dtype=torch.float32).reshape(-1)
        if flat.numel() != self.num_mlps * self.P:
            raise ValueError(f"expected {self.num_mlps * self.P} parameters, got {flat.numel()}")
        self.params.copy_(flat.to(self.device))
        self.repack()

    def repack(self):
        for i in range(self.num_mlps):
            check(lib.pob_pack_weights_pe(ptr(self.params[i * self.P:(i + 1) * self.P]), self.sh_deg,
                                          posenc_ref(self._posenc_struct), ptr(self.blobs[i]), stream_ptr()))

    def workspace(self, training, precision=PREC_FP16):
        """device scratch of the render call (training False) or of the training step at `precision`"""
        key = bool(training) if precision == PREC_FP16 else (bool(training), precision)
        if key not in self._ws:
            if training and precision != PREC_FP16:
                nbytes = int(lib.pob_train_workspace_bytes(ctypes_ref(self.cfg), int(precision)))
            else:
                nbytes = int(lib.pob_workspace_bytes(ctypes_ref(self.cfg), int(bool(training))))
            if nbytes < 0:
                raise _lib.PobError(lib.pob_last_error().decode())
            self._ws[key] = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return self._ws[key]

    def _blob(self, coarse):
        return self.blobs[0] if (coarse or self.num_mlps == 1) else self.blobs[1]

    # ---- NerfModel.__call__ ------------------------------------------------------------------
    def _set_sigma_noise(self, n, randomized, sigma_noise):
        """add_gaussian_noise (nerf_sh/nerf/model_utils.py:317-332): when randomized and noise_std is set, raw sigma
        of both levels gets normal(0, noise_std^2) noise.  sigma_noise = (coarse [n,Nc], fine [n,Nc+Nf]) passes the
        already scaled draws explicitly (parity tests).  Returns the tensors (kept alive by the caller)."""
        nc = nf = None
        if sigma_noise is not None:
            nc = _cuda_f32(sigma_noise[0], "sigma_noise[0]", self.num_coarse_samples)
            if self.num_mlps == 2:
                nf = _cuda_f32(sigma_noise[1], "sigma_noise[1]", self.num_coarse_samples + self.num_fine_samples)
        elif randomized and self.noise_std is not None and self.noise_std > 0:
            nc = torch.randn((n, self.num_coarse_samples), device=self.device) * float(self.noise_std)
            if self.num_mlps == 2:
                nf = torch.randn((n, self.num_coarse_samples + self.num_fine_samples),
                                 device=self.device) * float(self.noise_std)
        for t in (nc, nf):
            if t is not None and t.shape[0] != n:
                raise ValueError("sigma_noise must have one row per ray")
        self.cfg.sigma_noise_coarse_dev = ptr(nc)
        self.cfg.sigma_noise_fine_dev = ptr(nf)
        return nc, nf

    def __call__(self, rays, randomized=False, t_rand=None, u=None, precision=None, z_fine=None, sigma_noise=None):
        """-> [(rgb_coarse, disp_coarse, acc_coarse), (rgb, disp, acc)] for up to max_rays rays.

        randomized=True draws the stratified jitter / inverse-CDF uniforms on the device unless
        t_rand [B,Nc] / u [B,Nf] are given explicitly."""
        o = _cuda_f32(rays.origins, "rays.origins", 3)
        d = _cuda_f32(rays.directions, "rays.directions", 3)
        v = _cuda_f32(rays.viewdirs, "rays.viewdirs", 3)
        n = o.shape[0]
        if n > self.max_rays:
            raise ValueError(f"{n} rays exceed max_rays={self.max_rays}; chunk the call (utils.render_image)")
        t_rand, u, upr = self._uniforms(n, randomized, t_rand, u)
        z_fine = None if z_fine is None else _cuda_f32(z_fine, "z_fine")   # keep alive until the launch
        noise = self._set_sigma_noise(n, randomized, sigma_noise)           # noqa: F841  (same)
        ws = self.workspace(False)
        out_c = torch.empty((n, 5), dtype=torch.float32, device=self.device)
        out_f = torch.empty((n, 5), dtype=torch.float32, device=self.device) if self.num_mlps == 2 else None
        check(lib.pob_render_rays(ctypes_ref(self.cfg), ptr(self.blobs[0]),
                                  ptr(self.blobs[1]) if self.num_mlps == 2 else None, ptr(o), ptr(d), ptr(v), n,
                                  ptr(self.z_base), ptr(t_rand), ptr(u), upr,
                                  ptr(z_fine), ptr(out_c), ptr(out_f), ptr(ws), precision or self.precision,
                                  stream_ptr()))
        ret = [(out_c[:, :3], out_c[:, 3], out_c[:, 4])]
        if out_f is not None:
            ret.append((out_f[:, :3], out_f[:, 3], out_f[:, 4]))
        return ret

    def _uniforms(self, n, randomized, t_rand, u):
        if t_rand is not None:
            t_rand = _cuda_f32(t_rand, "t_rand", self.num_coarse_samples)
        elif randomized:
            t_rand = torch.rand((n, self.num_coarse_samples), dtype=torch.float32, device=self.device)
        upr = 0
        if self.num_fine_samples > 0:
            if u is not None:
                u = _cuda_f32(u, "u", self.num_fine_samples)
                upr = 1
            elif randomized:
                u = torch.rand((n, self.num_fine_samples), dtype=torch.float32, device=self.device)
                upr = 1
            else:
                u = self.u_table
        return t_rand, u, upr

    # ---- point evaluation --------------------------------------------------------------------
    def eval_points_raw(self, points, viewdirs=None, coarse=False, want_rgb=True, precision=None):
        from .. import ops
        return ops.eval_points_raw(self._blob(coarse), self.sh_deg, _cuda_f32(points, "points", 3), want_rgb,
                                   precision or self.precision, posenc=self.posenc, net_activation=self.net_act_code)

    def eval_points(self, points, viewdirs=None, coarse=False, precision=None):
        from .. import ops
        if self.sh_deg >= 0 and viewdirs is None:
            raise AssertionError("viewdirs required when sh_deg >= 0")
        vd = None if viewdirs is None else _cuda_f32(viewdirs, "viewdirs", 3)
        return ops.eval_points(self._blob(coarse), self.sh_deg, _cuda_f32(points, "points", 3), vd,
                               precision or self.precision, sigma_activation=self.sigma_act_code,
                               posenc=self.posenc, net_activation=self.net_act_code)


def ctypes_ref(struct):
    import ctypes
    return ctypes.addressof(struct)


def get_model_state(args, device="cuda", seed=20200823, restore=True):
    """models.get_model_state (nerf_sh/nerf/models.py:38-49): builds the model from a flags-like object,
    initialises parameters + Adam moments and, when `restore` and args.train_dir holds a flax-format
    `checkpoint_<step>`, restores parameters / moments / step from the newest one (checkpoints.py)."""
    from .train import TrainState
    model = NerfModel(sh_deg=args.sh_deg, num_coarse_samples=args.num_coarse_samples,
                      num_fine_samples=args.num_fine_samples, near=args.near, far=args.far,
                      white_bkgd=args.white_bkgd, lindisp=getattr(args, "lindisp", False),
                      max_rays=getattr(args, "batch_size", 4096),
                      sparsity_npoints=getattr(args, "sparsity_npoints", 0), device=device,
                      sigma_activation=getattr(args, "sigma_activation", "relu"),
                      min_deg_point=getattr(args, "min_deg_point", 0), max_deg_point=getattr(args, "max_deg_point", 10),
                      legacy_posenc_order=getattr(args, "legacy_posenc_order", False),
                      net_activation=getattr(args, "net_activation", "relu"))
    model.init_params(seed)
    state = TrainState(model)
    if restore and getattr(args, "train_dir", None):
        from . import checkpoints
        checkpoints.restore_checkpoint(args.train_dir, model, state)
    return model, state

"""Vanilla NeRF (use_viewdirs, sh_deg -1) inference: the reference's NerfModel with its view branch
(nerf_sh/nerf/models.py:143-214,216-348, model_utils.py:30-94), as `nerf_sh.eval` / `gen_video` use it for a model
trained or downloaded with `--config nerf_sh/config/misc/og_nerf`.

Per MLP the colour branch raw_rgb = W11 act(W10 [W9 h7 + b9; posenc(viewdir)] + b10) + b11 is split at the condition
layer, as the SH projection splits it (octree/projection.py): Dense_9 has no activation, so
  a_p = h7 (W9 W10_b)                        per sample: heads columns 8..135 of the tensor-core forward
  t_r = W10_e posenc(viewdir_r) + c          per ray, c = b9 W10_b + b10 (pob_render_rays_vanilla tabulates it)
  raw_rgb = W11 act(a_p + t_r) + b11         in the forward's epilogue (include/plenoctree_b200.h)
W9 W10_b and c are formed once here in fp64 (fold_view_branch); the folded head is rounded once, to the fp16 the
tensor cores read.  Inference only: training a vanilla NeRF stays refused (flags.check_scope).
"""
import numpy as np
import torch

from .._lib import PREC_FP16, RenderConfig, ViewBranch, check, lib, posenc_ref, posenc_struct, ptr, stream_ptr
from .models import RaySampler, _cuda_f32, ctypes_ref

POINTS_PER_CALL = 1 << 20        # points per pob_eval_points_vanilla call (a 512 MB view table)


def fold_view_branch(layers):
    """(W9 W10_b [256, 128], b9 W10_b + b10 [128]) of a vanilla MLP [(kernel, bias) x 12], in fp64."""
    k9, b9 = (np.asarray(a, dtype=np.float64) for a in layers[9])
    k10, b10 = (np.asarray(a, dtype=np.float64) for a in layers[10])
    return k9 @ k10[:256], b9 @ k10[:256] + b10


def folded_flat(layers):
    """flat parameters of pob_pack_vanilla: Dense_0..Dense_8 (kernel, bias) in fp32, then W9 W10_b rounded once from
    fp64 to fp16 (held in fp32, so the packing keeps it exactly)."""
    w, _ = fold_view_branch(layers)
    parts = [np.asarray(a, dtype=np.float32).reshape(-1) for k, b in layers[:9] for a in (k, b)]
    parts.append(w.astype(np.float16).astype(np.float32).reshape(-1))
    return np.concatenate(parts)


class VanillaNerfModel(RaySampler):
    """The reference's NerfModel with use_viewdirs (coarse MLP_0, fine MLP_1) on the device.  `mlps` is a vanilla
    parameter set {"MLP_0": [(kernel, bias) x 12], "MLP_1": ...} (checkpoints.vanilla_from_flax_params /
    vanilla_from_torch_state_dict).  It holds packed weights and view-branch arrays only: no optimiser state."""

    def __init__(self, mlps, deg_view=4, num_coarse_samples=64, num_fine_samples=128, near=2.0, far=6.0,
                 white_bkgd=True, lindisp=False, max_rays=4096, device="cuda", noise_std=None, sigma_activation="relu",
                 min_deg_point=0, max_deg_point=10, legacy_posenc_order=False, net_activation="relu"):
        from .flags import MAX_DEG_VIEW, check_posenc, check_samples, net_activation_code, sigma_activation_code
        check_samples(num_coarse_samples, num_fine_samples)
        check_posenc(min_deg_point, max_deg_point)
        if not 0 <= int(deg_view) <= MAX_DEG_VIEW:
            raise ValueError(f"deg_view={deg_view}: 0 <= deg_view <= {MAX_DEG_VIEW} expected")
        self.sh_deg = -1
        self.precision = PREC_FP16
        self.posenc = (int(min_deg_point), int(max_deg_point), bool(legacy_posenc_order))
        self.deg_view = int(deg_view)
        self.net_act_code = net_activation_code(net_activation)
        self.sigma_act_code = sigma_activation_code(sigma_activation)
        self._pe = posenc_struct(self.posenc, self.net_act_code)
        self.num_coarse_samples = int(num_coarse_samples)
        self.num_fine_samples = int(num_fine_samples)
        self.num_mlps = 2 if self.num_fine_samples > 0 else 1
        self.near, self.far = float(near), float(far)
        self.white_bkgd = bool(white_bkgd)
        self.lindisp = bool(lindisp)
        self.max_rays = int(max_rays)
        self.noise_std = noise_std
        self.device = torch.device(device)
        self.step = None
        names = [f"MLP_{i}" for i in range(self.num_mlps)]
        missing = [n for n in names if n not in mlps]
        if missing:
            raise ValueError(f"the parameter set has no {missing[0]} (num_fine_samples={self.num_fine_samples} "
                             f"needs {' and '.join(names)})")
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(self.device)   # noqa: E731
        nb = int(lib.pob_vanilla_packed_bytes())
        self.blobs, self._view_arrays = [], []
        self.view = ViewBranch()
        self.view.deg_view = self.deg_view
        for i, name in enumerate(names):
            layers = mlps[name]
            flat = dev(folded_flat(layers))
            if flat.numel() != int(lib.pob_vanilla_param_count(posenc_ref(self._pe))):
                raise ValueError(f"{name}: Dense_0..Dense_8 do not match the point encoder {self.posenc}")
            blob = torch.zeros(nb, dtype=torch.uint8, device=self.device)
            check(lib.pob_pack_vanilla(ptr(flat), posenc_ref(self._pe), ptr(blob), stream_ptr()))
            _, c = fold_view_branch(layers)
            arrays = (dev(layers[10][0][256:]), dev(c), dev(layers[11][0]), dev(layers[11][1]))
            if arrays[0].shape[0] != 3 + 6 * self.deg_view:
                raise ValueError(f"{name}/Dense_10 has {256 + arrays[0].shape[0]} input rows, deg_view={self.deg_view} "
                                 f"needs {256 + 3 + 6 * self.deg_view}")
            m = self.view.mlp[i]
            m.w10e_dev, m.c_dev, m.w11_dev, m.b11_dev = (ptr(a) for a in arrays)
            self.blobs.append(blob)
            self._view_arrays.append(arrays)   # keeps the descriptor's arrays alive
        self.cfg = RenderConfig(-1, self.num_coarse_samples, self.num_fine_samples, int(self.white_bkgd),
                                self.max_rays, 0)
        self.cfg.sigma_activation = self.sigma_act_code
        self.cfg.posenc = posenc_ref(self._pe)
        self._ws = None
        self._init_depths()

    @classmethod
    def from_flags(cls, args, *, max_rays, device="cuda"):
        """the model of the flags of `args`, restored from args.train_dir: the newest flax `checkpoint_<step>` (a
        jaxnerf checkpoint), else the newest torch `*.ckpt` (checkpoints.restore_vanilla).  `step` is the flax
        checkpoint's step (0 for a torch file)."""
        from . import checkpoints
        pe = (int(args.min_deg_point), int(args.max_deg_point), bool(args.legacy_posenc_order))
        sd = checkpoints.restore_flax_state_dict(args.train_dir)
        if sd is not None:
            mlps = checkpoints.vanilla_from_flax_params(sd["optimizer"]["target"]["params"], pe, args.deg_view)
            step = int((sd["optimizer"].get("state") or {}).get("step", 0))
        else:
            mlps = checkpoints.restore_vanilla(args.train_dir, False, pe, args.deg_view)
            step = 0
        if mlps is None:
            raise ValueError(f"no checkpoint_* or *.ckpt in {args.train_dir}")
        model = cls(mlps, deg_view=args.deg_view, num_coarse_samples=args.num_coarse_samples,
                    num_fine_samples=args.num_fine_samples, near=args.near, far=args.far, white_bkgd=args.white_bkgd,
                    lindisp=args.lindisp, max_rays=max_rays, device=device, noise_std=args.noise_std,
                    sigma_activation=args.sigma_activation, min_deg_point=args.min_deg_point,
                    max_deg_point=args.max_deg_point, legacy_posenc_order=args.legacy_posenc_order,
                    net_activation=args.net_activation)
        model.step = step
        return model

    def workspace(self):
        if self._ws is None:
            n = int(lib.pob_vanilla_workspace_bytes(ctypes_ref(self.cfg)))
            if n < 0:
                check(1)
            self._ws = torch.empty(n, dtype=torch.uint8, device=self.device)
        return self._ws

    def __call__(self, rays, randomized=False, t_rand=None, u=None, z_fine=None, sigma_noise=None, precision=None):
        """NerfModel.__call__ -> [(rgb_coarse, disp_coarse, acc_coarse), (rgb, disp, acc)] for up to max_rays rays
        (the arguments of NerfModel.__call__; precision must be None or PREC_FP16)."""
        if precision not in (None, PREC_FP16):
            raise ValueError("the vanilla forward is fp16 (PREC_FP16)")
        o = _cuda_f32(rays.origins, "rays.origins", 3)
        d = _cuda_f32(rays.directions, "rays.directions", 3)
        v = _cuda_f32(rays.viewdirs, "rays.viewdirs", 3)
        n = o.shape[0]
        if n > self.max_rays:
            raise ValueError(f"{n} rays exceed max_rays={self.max_rays}; chunk the call (utils.render_image)")
        t_rand, u, upr = self._uniforms(n, randomized, t_rand, u)
        z_fine = None if z_fine is None else _cuda_f32(z_fine, "z_fine")   # keep alive until the launch
        noise = self._set_sigma_noise(n, randomized, sigma_noise)           # noqa: F841  (same)
        out_c = torch.empty((n, 5), dtype=torch.float32, device=self.device)
        out_f = torch.empty((n, 5), dtype=torch.float32, device=self.device) if self.num_mlps == 2 else None
        check(lib.pob_render_rays_vanilla(ctypes_ref(self.cfg), ctypes_ref(self.view), ptr(self.blobs[0]),
                                          ptr(self.blobs[1]) if self.num_mlps == 2 else None, ptr(o), ptr(d), ptr(v),
                                          n, ptr(self.z_base), ptr(t_rand), ptr(u), upr, ptr(z_fine), ptr(out_c),
                                          ptr(out_f), ptr(self.workspace()), PREC_FP16, stream_ptr()))
        ret = [(out_c[:, :3], out_c[:, 3], out_c[:, 4])]
        if out_f is not None:
            ret.append((out_f[:, :3], out_f[:, 3], out_f[:, 4]))
        return ret

    def _points(self, points, viewdirs, coarse, raw):
        p = _cuda_f32(points, "points", 3)
        v = _cuda_f32(viewdirs, "viewdirs", 3)
        if v.shape != p.shape:
            raise ValueError("viewdirs must hold one direction per point")
        m = p.shape[0]
        mlp = 0 if (coarse or self.num_mlps == 1) else 1
        # the per-point view table is 512 bytes a point: one POINTS_PER_CALL scratch table serves every chunk
        table = torch.empty((min(m, POINTS_PER_CALL), 128), dtype=torch.float32, device=self.device)
        if raw:
            rgb = torch.empty((m, 3), dtype=torch.float32, device=self.device)
            sigma = torch.empty((m, 1), dtype=torch.float32, device=self.device)
            out = None
        else:
            out = torch.empty((m, 4), dtype=torch.float32, device=self.device)
            rgb = sigma = None
        for i in range(0, m, POINTS_PER_CALL):
            j = min(m, i + POINTS_PER_CALL)
            check(lib.pob_eval_points_vanilla(ptr(self.blobs[mlp]), posenc_ref(self._pe), ctypes_ref(self.view), mlp,
                                              ptr(p[i:j]), ptr(v[i:j]), j - i, ptr(table),
                                              ptr(rgb[i:j]) if raw else None, ptr(sigma[i:j]) if raw else None,
                                              None if raw else ptr(out[i:j]), self.sigma_act_code, stream_ptr()))
        return (rgb, sigma) if raw else (out[:, :3], out[:, 3:4])

    def eval_points_raw(self, points, viewdirs, coarse=False):
        """eval_points_raw(points, viewdirs) (models.py:143-181, octree/nerf/models.py:211-252): (raw_rgb [M, 3],
        raw_sigma [M, 1]) of the fine MLP (the coarse one when `coarse` or without a fine level)."""
        return self._points(points, viewdirs, coarse, True)

    def eval_points(self, points, viewdirs, coarse=False):
        """eval_points (models.py:183-214): (sigmoid(raw_rgb) [M, 3], density activation of raw sigma [M, 1])."""
        return self._points(points, viewdirs, coarse, False)

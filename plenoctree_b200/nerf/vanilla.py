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

from .._lib import PREC_FP16, ViewBranch, check, lib, posenc_ref, ptr, stream_ptr
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


def view_branch(name, layers, deg_view, device):
    """the view-branch arrays of one vanilla MLP on the device: (W10_e [3 + 6 deg_view, 128], c [128], W11 [128, 3],
    b11 [3]), c = b9 W10_b + b10 (fold_view_branch).  A Dense_10 whose rows do not match deg_view is refused before
    anything is uploaded: the kernels read 3 + 6 deg_view rows of W10_e."""
    w10e = np.asarray(layers[10][0], dtype=np.float32)[256:]
    if w10e.shape[0] != 3 + 6 * int(deg_view):
        raise ValueError(f"{name}/Dense_10 has {256 + w10e.shape[0]} input rows, deg_view={deg_view} "
                         f"needs {256 + 3 + 6 * int(deg_view)}")
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)   # noqa: E731
    return dev(w10e), dev(fold_view_branch(layers)[1]), dev(layers[11][0]), dev(layers[11][1])


class VanillaNerfModel(RaySampler):
    """The reference's NerfModel with use_viewdirs (coarse MLP_0, fine MLP_1) on the device.  `mlps` is a vanilla
    parameter set {"MLP_0": [(kernel, bias) x 12], "MLP_1": ...} (checkpoints.vanilla_from_flax_params /
    vanilla_from_torch_state_dict).  It holds packed weights and view-branch arrays only: no optimiser state."""

    def __init__(self, mlps, deg_view=4, num_coarse_samples=64, num_fine_samples=128, near=2.0, far=6.0,
                 white_bkgd=True, lindisp=False, max_rays=4096, device="cuda", noise_std=None, sigma_activation="relu",
                 min_deg_point=0, max_deg_point=10, legacy_posenc_order=False, net_activation="relu"):
        from .flags import MAX_DEG_VIEW, check_posenc
        check_posenc(min_deg_point, max_deg_point)
        if not 0 <= int(deg_view) <= MAX_DEG_VIEW:
            raise ValueError(f"deg_view={deg_view}: 0 <= deg_view <= {MAX_DEG_VIEW} expected")
        super().__init__(-1, num_coarse_samples, num_fine_samples, near, far, white_bkgd, lindisp, max_rays, 0, device,
                         noise_std, sigma_activation, min_deg_point, max_deg_point, legacy_posenc_order,
                         net_activation)
        self.precision = PREC_FP16
        self.deg_view = int(deg_view)
        self.step = None
        names = [f"MLP_{i}" for i in range(self.num_mlps)]
        missing = [n for n in names if n not in mlps]
        if missing:
            raise ValueError(f"the parameter set has no {missing[0]} (num_fine_samples={self.num_fine_samples} "
                             f"needs {' and '.join(names)})")
        nb = int(lib.pob_vanilla_packed_bytes())
        self.blobs, self._view_arrays = [], []
        self.view = ViewBranch()
        self.view.deg_view = self.deg_view
        for i, name in enumerate(names):
            flat = torch.from_numpy(folded_flat(mlps[name])).to(self.device)
            if flat.numel() != int(lib.pob_vanilla_param_count(posenc_ref(self._posenc_struct))):
                raise ValueError(f"{name}: Dense_0..Dense_8 do not match the point encoder {self.posenc}")
            blob = torch.zeros(nb, dtype=torch.uint8, device=self.device)
            check(lib.pob_pack_vanilla(ptr(flat), posenc_ref(self._posenc_struct), ptr(blob), stream_ptr()))
            arrays = view_branch(name, mlps[name], self.deg_view, self.device)
            m = self.view.mlp[i]
            m.w10e_dev, m.c_dev, m.w11_dev, m.b11_dev = (ptr(a) for a in arrays)
            self.blobs.append(blob)
            self._view_arrays.append(arrays)   # keeps the descriptor's arrays alive

    @classmethod
    def from_flags(cls, args, *, max_rays, device="cuda"):
        """the model of the flags of `args`, restored from args.train_dir: the newest flax `checkpoint_<step>` (a
        jaxnerf checkpoint), else the newest torch `*.ckpt` (checkpoints.restore_vanilla).  `step` is the flax
        checkpoint's step (0 for a torch file)."""
        from . import checkpoints
        pe = (int(args.min_deg_point), int(args.max_deg_point), bool(args.legacy_posenc_order))
        for jaxnerf in (True, False):
            mlps, step = checkpoints.restore_vanilla_and_step(args.train_dir, jaxnerf, pe, args.deg_view)
            if mlps is not None:
                break
        else:
            raise ValueError(f"no checkpoint_* or *.ckpt in {args.train_dir}")
        model = cls(mlps, deg_view=args.deg_view, max_rays=max_rays, device=device, noise_std=args.noise_std,
                    **cls.flag_kwargs(args))
        model.step = step
        return model

    @property
    def _pe(self):
        """the encoder descriptor (RaySampler._posenc_struct), by the name the projection's VanillaNerf gives it"""
        return self._posenc_struct

    def workspace(self):
        return self._workspace(None, lambda: lib.pob_vanilla_workspace_bytes(ctypes_ref(self.cfg)))

    def _precision(self, precision):
        if precision not in (None, PREC_FP16):
            raise ValueError("the vanilla forward is fp16 (PREC_FP16)")
        return PREC_FP16

    def _render(self, o, d, v, n, t_rand, u, upr, z_fine, out_c, out_f, precision):
        check(lib.pob_render_rays_vanilla(ctypes_ref(self.cfg), ctypes_ref(self.view), ptr(self.blobs[0]),
                                          ptr(self.blobs[1]) if self.num_mlps == 2 else None, ptr(o), ptr(d), ptr(v),
                                          n, ptr(self.z_base), ptr(t_rand), ptr(u), upr, ptr(z_fine), ptr(out_c),
                                          ptr(out_f), ptr(self.workspace()), precision, stream_ptr()))

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
            check(lib.pob_eval_points_vanilla(ptr(self.blobs[mlp]), posenc_ref(self._posenc_struct),
                                              ctypes_ref(self.view), mlp, ptr(p[i:j]), ptr(v[i:j]), j - i, ptr(table),
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

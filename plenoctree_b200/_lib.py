"""ctypes binding of libplenoctree_b200.so (the C ABI in include/plenoctree_b200.h).

There is no fallback: if the shared library is missing the import raises, and every compute entry
point fails when no sm_90 device is present.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("POB_LIB_PATH") or os.path.join(_HERE, "libplenoctree_b200.so")   # override: kernel A/B experiments

PREC_FP16 = 1
PREC_FP16X3 = 3

TRAIN_DISCARD_SAVED_GRADS = 1   # POB_TRAIN_*: flags of pob_loss_and_grad_flags

SIGMA_RELU = 0        # POB_SIGMA_*: density activation of the ray samples and of eval_points
SIGMA_SOFTPLUS = 1

NET_RELU = 0          # POB_NET_*: trunk activation (pob_posenc.net_activation)
NET_ELU = 1
NET_SOFTPLUS = 2
NET_TANH = 3

_c = ctypes
_vp, _i, _i64, _fp = _c.c_void_p, _c.c_int, _c.c_int64, _c.c_void_p

# name -> (restype, argtypes); must list every symbol the header declares
SIGNATURES = {
    "pob_abi_version": (_i, []),
    "pob_last_error": (_c.c_char_p, []),
    "pob_sm_count": (_i, []),
    "pob_launch_count": (_c.c_longlong, []),
    "pob_timing_enable": (None, [_i]),
    "pob_timing_read": (_i, [_vp, _vp]),
    "pob_timing_read_phases": (_i, [_i, _vp, _vp]),
    "pob_param_count": (_i64, [_i]),
    "pob_packed_bytes": (_i64, [_i]),
    "pob_pack_weights": (_i, [_fp, _i, _vp, _vp]),
    "pob_param_count_pe": (_i64, [_i, _vp]),
    "pob_pack_weights_pe": (_i, [_fp, _i, _vp, _vp, _vp]),
    "pob_eval_points_raw": (_i, [_vp, _i, _fp, _i64, _fp, _fp, _i, _vp]),
    "pob_eval_points": (_i, [_vp, _i, _fp, _fp, _i64, _fp, _i, _vp]),
    "pob_eval_points_act": (_i, [_vp, _i, _fp, _fp, _i64, _fp, _i, _i, _vp]),
    "pob_eval_cells_mean": (_i, [_vp, _i, _fp, _i64, _i, _fp, _i, _vp]),
    "pob_eval_grid": (_i, [_vp, _i, _i, _i, _i, _i, _i, _c.POINTER(_c.c_float), _c.POINTER(_c.c_float),
                           _fp, _fp, _i, _vp]),
    "pob_eval_points_raw_host": (_i, [_vp, _i, _fp, _i64, _fp, _fp, _i]),
    "pob_eval_points_raw_pe": (_i, [_vp, _i, _vp, _fp, _i64, _fp, _fp, _i, _vp]),
    "pob_eval_points_pe": (_i, [_vp, _i, _vp, _fp, _fp, _i64, _fp, _i, _i, _vp]),
    "pob_eval_grid_pe": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _c.POINTER(_c.c_float), _c.POINTER(_c.c_float),
                              _fp, _fp, _i, _vp]),
    "pob_eval_cells_mean_pe": (_i, [_vp, _i, _vp, _fp, _i64, _i, _fp, _i, _vp]),
    "pob_eval_points_raw_host_pe": (_i, [_vp, _i, _vp, _fp, _i64, _fp, _fp, _i]),
    "pob_sample_coarse": (_i, [_fp, _fp, _i, _i, _fp, _vp]),
    "pob_draw_uniforms": (_i, [_c.c_uint64, _c.c_float, _fp, _fp, _i64, _fp, _i64, _fp, _i64, _c.c_float, _vp]),
    "pob_composite": (_i, [_fp, _fp, _fp, _i, _i, _i, _fp, _fp, _fp, _fp, _vp]),
    "pob_composite_bwd": (_i, [_fp, _fp, _fp, _fp, _fp, _i, _i, _i, _c.c_float, _fp, _fp, _vp]),
    "pob_sample_pdf": (_i, [_fp, _fp, _fp, _i, _i, _i, _i, _fp, _vp]),
    "pob_workspace_bytes": (_i64, [_vp, _i]),
    "pob_render_rays": (_i, [_vp, _vp, _vp, _fp, _fp, _fp, _i, _fp, _fp, _fp, _i, _fp, _fp, _fp, _vp, _i, _vp]),
    "pob_loss_and_grad": (_i, [_vp, _vp, _vp, _vp, _fp, _fp, _fp, _fp, _i, _fp, _fp, _fp, _i, _fp, _fp, _fp, _fp,
                               _vp, _vp, _vp]),
    "pob_train_workspace_bytes": (_i64, [_vp, _i]),
    "pob_loss_and_grad_prec": (_i, [_vp, _vp, _vp, _vp, _fp, _fp, _fp, _fp, _i, _fp, _fp, _fp, _i, _fp, _fp, _fp,
                                    _fp, _vp, _vp, _fp, _i, _vp]),
    "pob_loss_and_grad_flags": (_i, [_vp, _vp, _vp, _vp, _fp, _fp, _fp, _fp, _i, _fp, _fp, _fp, _i, _fp, _fp, _fp,
                                     _fp, _vp, _vp, _fp, _i, _i, _vp]),
    "pob_adam_update": (_i, [_i, _i, _fp, _fp, _fp, _fp, _c.c_float, _c.c_float, _fp, _c.c_float, _c.c_float,
                             _vp, _vp, _vp]),
    "pob_adam_update_pe": (_i, [_i, _vp, _i, _fp, _fp, _fp, _fp, _c.c_float, _c.c_float, _fp, _c.c_float,
                                _c.c_float, _vp, _vp, _vp]),
    "pob_octree_render": (_i, [_vp, _vp, _fp, _fp, _fp, _i64, _vp, _i, _i, _fp, _vp, _vp]),
    "pob_octree_render_backward": (_i, [_vp, _vp, _fp, _fp, _fp, _i64, _vp, _i, _i, _fp, _fp, _vp]),
    "pob_octree_render_depth": (_i, [_vp, _vp, _fp, _fp, _fp, _i64, _vp, _i, _i, _fp, _fp, _fp, _vp, _vp]),
    "pob_octree_render_depth_backward": (_i, [_vp, _vp, _fp, _fp, _fp, _i64, _vp, _i, _i, _fp, _fp, _fp, _fp, _vp]),
    "pob_octree_render_quant": (_i, [_vp, _vp, _fp, _fp, _fp, _i64, _vp, _i, _i, _fp, _vp, _vp]),
    "pob_octree_render_depth_quant": (_i, [_vp, _vp, _fp, _fp, _fp, _i64, _vp, _i, _i, _fp, _fp, _fp, _vp, _vp]),
    "pob_octree_train_persp": (_i, [_vp, _vp, _vp, _i, _i, _fp, _c.c_float, _fp, _vp, _fp, _vp]),
    "pob_octree_train_persp_ndc": (_i, [_vp, _vp, _vp, _vp, _i, _i, _fp, _c.c_float, _fp, _vp, _fp, _vp]),
    "pob_ndc_rays": (_i, [_vp, _fp, _fp, _fp, _i64, _vp, _i, _i, _fp, _fp, _fp, _vp]),
    "pob_octree_sgd_step": (_i, [_fp, _fp, _i64, _c.c_float, _vp]),
    "pob_octree_sgd_momentum_step": (_i, [_fp, _fp, _fp, _i64, _c.c_float, _c.c_float, _i, _vp]),
    "pob_octree_adam_step": (_i, [_fp, _fp, _fp, _fp, _i64, _c.c_float, _c.c_float, _c.c_float, _vp]),
    "pob_octree_query": (_i, [_vp, _fp, _i64, _vp, _vp]),
    "pob_grid_weight_render": (_i, [_fp, _i, _vp, _i, _i, _i, _c.POINTER(_c.c_float), _c.POINTER(_c.c_float),
                                    _vp, _fp, _vp, _vp]),
    "pob_grid_weight_render_ndc": (_i, [_fp, _i, _vp, _i, _i, _i, _c.POINTER(_c.c_float), _c.POINTER(_c.c_float),
                                        _vp, _vp, _fp, _vp, _vp]),
    "pob_sh_proj_points_workspace_bytes": (_i64, [_i64]),
    "pob_sh_proj_points": (_i, [_vp, _vp, _fp, _i64, _fp, _fp, _vp, _fp, _fp, _vp]),
    "pob_sh_proj_directions": (_i, [_c.c_uint64, _i64, _i, _i, _i, _i, _i, _fp, _fp, _fp, _fp, _vp]),
    "pob_sh_proj_cells": (_i, [_i64, _i, _i, _fp, _fp, _i, _i, _fp, _fp, _fp, _fp, _fp, _vp]),
    "pob_vanilla_param_count": (_i64, [_vp]),
    "pob_vanilla_packed_bytes": (_i64, []),
    "pob_pack_vanilla": (_i, [_fp, _vp, _vp, _vp]),
    "pob_vanilla_workspace_bytes": (_i64, [_vp]),
    "pob_render_rays_vanilla": (_i, [_vp, _vp, _vp, _vp, _fp, _fp, _fp, _i, _fp, _fp, _fp, _i, _fp, _fp, _fp, _vp, _i,
                                     _vp]),
    "pob_eval_points_vanilla": (_i, [_vp, _vp, _vp, _i, _fp, _fp, _i64, _fp, _fp, _fp, _fp, _i, _vp]),
    "pob_quantize_workspace_bytes": (_i64, [_i64, _i64, _i]),
    "pob_quantize_median_cut": (_i, [_fp, _fp, _i64, _i64, _i, _fp, _fp, _vp, _i64, _vp]),
}


class NetDesc(_c.Structure):
    """pob_posenc, the network beyond sh_deg: the point encoder posenc(x, min_deg, max_deg, legacy_order) and the
    trunk activation net_activation (NET_*).  A NULL pointer is (0, 10, 0, NET_RELU)."""
    _fields_ = [("min_deg", _i), ("max_deg", _i), ("legacy_order", _i), ("net_activation", _i)]


POSENC_DEFAULT = (0, 10, False)   # flags min_deg_point, max_deg_point, legacy_posenc_order of the reference


def posenc_struct(posenc, net_activation=NET_RELU):
    """(min_deg, max_deg, legacy) and a NET_* code -> NetDesc, or None (NULL) for the default encoder with a relu
    trunk, so that a default model calls the library exactly as before the descriptor existed."""
    if (posenc is None or tuple(posenc) == POSENC_DEFAULT) and int(net_activation) == NET_RELU:
        return None
    mn, mx, legacy = POSENC_DEFAULT if posenc is None else posenc
    return NetDesc(int(mn), int(mx), int(bool(legacy)), int(net_activation))


def posenc_ref(struct):
    """pointer argument of a NetDesc (None -> NULL)."""
    return None if struct is None else _c.addressof(struct)


class RenderConfig(_c.Structure):
    _fields_ = [("sh_deg", _i), ("num_coarse_samples", _i), ("num_fine_samples", _i), ("white_bkgd", _i),
                ("max_rays", _i), ("sparsity_npoints", _i), ("sigma_noise_coarse_dev", _vp),
                ("sigma_noise_fine_dev", _vp), ("sigma_activation", _i), ("posenc", _vp)]


class ViewMlp(_c.Structure):
    """pob_view_mlp: the view branch of one vanilla MLP (device fp32 arrays)."""
    _fields_ = [("w10e_dev", _vp), ("c_dev", _vp), ("w11_dev", _vp), ("b11_dev", _vp)]


class ViewBranch(_c.Structure):
    """pob_view_branch: deg_view and the view branch of MLP_0 (coarse) and MLP_1 (fine)."""
    _fields_ = [("deg_view", _i), ("mlp", ViewMlp * 2)]


class TrainHParams(_c.Structure):
    _fields_ = [("sparsity_weight", _c.c_float), ("sparsity_length", _c.c_float), ("loss_scale", _c.c_float)]


class Octree(_c.Structure):
    _fields_ = [("data_dev", _vp), ("child_dev", _vp), ("n_nodes", _i64), ("N", _i), ("data_dim", _i),
                ("basis_dim", _i), ("format", _i), ("offset", _c.c_float * 3), ("invradius", _c.c_float * 3)]


class OctreeQuant(_c.Structure):
    """pob_octree_quant: a compressed (palette-indexed) tree; palette / retained are fp16 bit patterns."""
    _fields_ = [("child_dev", _vp), ("n_nodes", _i64), ("N", _i), ("basis_dim", _i), ("format", _i),
                ("retain", _i), ("bits", _i), ("sigma_dev", _vp), ("map_dev", _vp), ("palette_dev", _vp),
                ("retained_dev", _vp), ("offset", _c.c_float * 3), ("invradius", _c.c_float * 3)]


class OctreeOpts(_c.Structure):
    _fields_ = [("step_size", _c.c_float), ("background_brightness", _c.c_float), ("sigma_thresh", _c.c_float),
                ("stop_thresh", _c.c_float)]


class Ndc(_c.Structure):
    """pob_ndc: svox NDCConfig(width, height, focal) of a forward-facing scene."""
    _fields_ = [("width", _c.c_float), ("height", _c.c_float), ("focal", _c.c_float)]


class Camera(_c.Structure):
    _fields_ = [("c2w", _c.c_float * 12), ("fx", _c.c_float), ("fy", _c.c_float), ("width", _c.c_float),
                ("height", _c.c_float)]


class PobError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -m plenoctree_b200.build` "
            "(there is no CPU fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def check(rc):
    if rc != 0:
        raise PobError(lib.pob_last_error().decode())


def ptr(t):
    """device/host pointer of a torch tensor or numpy array (None -> NULL)."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    return t.ctypes.data


def stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream

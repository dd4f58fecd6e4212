"""Checkpoint bridge (SURVEY §8f rank 1): the flat fp32 parameter / Adam buffers of this package  <->
the two on-disk formats of the reference.

  flax  `checkpoint_<step>`  written by nerf_sh/train.py:237-242,306-310 (flax.training.checkpoints.save_checkpoint
        of utils.TrainState(optimizer)) and read by nerf_sh/nerf/models.py:46-48 and by
        octree/nerf/models.py:66-113 (restore_model_state_from_jaxnerf: ["optimizer"]["target"]["params"],
        Dense_0..7 -> input_layers.i, Dense_8 -> sigma_layer, Dense_9 -> rgb_layer, kernel.T -> weight)
  torch `*.ckpt`             torch.save({"model": state_dict}) read by octree/nerf/models.py:52-63

The flax file is msgpack with numpy arrays as ExtType 1 = packb((shape, dtype.name, raw bytes)) and numpy scalars
as ExtType 3 (flax.serialization; flax itself is not in this image, so the encoding is restated here and pinned by
round trips and by the fixture tests/golden/ckpt_bridge.npz, which make_golden.py produced by letting the
REFERENCE's own restore_model_state_from_jaxnerf load a file written by this module).

Flat layout (include/plenoctree_b200.h): [MLP_0 | MLP_1], each Dense_0..Dense_9 as kernel [in,out] row-major, bias.
This module is host-side file plumbing (numpy only); nothing here touches the GPU.
"""
import glob
import os
import re

import msgpack
import numpy as np

from ..layouts import K_of, layer_dims, posenc_width

_EXT_NDARRAY, _EXT_NATIVE_COMPLEX, _EXT_NPSCALAR = 1, 2, 3


# ---- flat <-> nested parameter dicts -------------------------------------------------------------------------
# `posenc` = (min_deg_point, max_deg_point, legacy_posenc_order) of the model, None = the default (0, 10, False): its
# width W = 3 + 6 (max - min) sets the shapes Dense_0 [W, 256] and Dense_5 [256 + W, 256].
def _dims(sh_deg, posenc):
    return layer_dims(K_of(sh_deg), posenc_width(posenc))


def _posenc_of(model):
    """the model's encoder; objects without one (duck-typed models) have the default"""
    return getattr(model, "posenc", None)


def param_count(sh_deg, posenc=None):
    return sum(i * o + o for i, o in _dims(sh_deg, posenc))


def flat_to_flax_params(flat, sh_deg, posenc=None):
    """flat [num_mlps * P] -> {"MLP_0": {"Dense_i": {"kernel": [in,out], "bias": [out]}}, "MLP_1": ...}
    (the pytree under ["optimizer"]["target"]["params"], nerf_sh/nerf/model_utils.py:60-93)."""
    flat = np.asarray(flat, dtype=np.float32).reshape(-1)
    P = param_count(sh_deg, posenc)
    if flat.size % P != 0 or flat.size // P not in (1, 2):
        raise ValueError(f"expected {P} or {2 * P} parameters, got {flat.size}")
    out = {}
    for m in range(flat.size // P):
        off = m * P
        mlp = {}
        for i, (cin, cout) in enumerate(_dims(sh_deg, posenc)):
            k = flat[off:off + cin * cout].reshape(cin, cout).copy()
            off += cin * cout
            b = flat[off:off + cout].copy()
            off += cout
            mlp[f"Dense_{i}"] = {"kernel": k, "bias": b}
        out[f"MLP_{m}"] = mlp
    return out


def flax_params_to_flat(params, sh_deg, posenc=None):
    parts = []
    m = 0
    while f"MLP_{m}" in params:
        mlp = params[f"MLP_{m}"]
        for i, (cin, cout) in enumerate(_dims(sh_deg, posenc)):
            d = mlp[f"Dense_{i}"]
            k = np.asarray(d["kernel"], dtype=np.float32)
            b = np.asarray(d["bias"], dtype=np.float32)
            if k.shape != (cin, cout) or b.shape != (cout,):
                hint = ("wrong min_deg_point / max_deg_point? Dense_0 has 3 + 6 (max_deg_point - min_deg_point) rows"
                        if i in (0, 5) and k.shape[1:] == (cout,) else "wrong sh_deg?")
                raise ValueError(f"MLP_{m}/Dense_{i}: expected kernel {(cin, cout)}, got {k.shape} ({hint})")
            parts += [k.reshape(-1), b]
        m += 1
    if m == 0:
        raise ValueError("no MLP_0 in the parameter tree")
    return np.concatenate(parts).astype(np.float32)


_TORCH_NAMES = [f"input_layers.{i}" for i in range(8)] + ["sigma_layer", "rgb_layer"]


def flat_to_torch_state_dict(flat, sh_deg, posenc=None):
    """-> {"MLP_0.input_layers.0.weight": [out,in], ...} as numpy arrays: the state_dict of the reference's torch
    twin (octree/nerf/models.py:116-209, octree/nerf/model_utils.py:36-95), nn.Linear weight = kernel.T."""
    out = {}
    for mname, mlp in flat_to_flax_params(flat, sh_deg, posenc).items():
        for i, tname in enumerate(_TORCH_NAMES):
            out[f"{mname}.{tname}.weight"] = np.ascontiguousarray(mlp[f"Dense_{i}"]["kernel"].T)
            out[f"{mname}.{tname}.bias"] = mlp[f"Dense_{i}"]["bias"]
    return out


def torch_state_dict_to_flat(sd, sh_deg, posenc=None):
    params = {}
    m = 0
    while f"MLP_{m}.input_layers.0.weight" in sd:
        mlp = {}
        for i, tname in enumerate(_TORCH_NAMES):
            w = np.asarray(sd[f"MLP_{m}.{tname}.weight"], dtype=np.float32)
            mlp[f"Dense_{i}"] = {"kernel": w.T, "bias": np.asarray(sd[f"MLP_{m}.{tname}.bias"], dtype=np.float32)}
        params[f"MLP_{m}"] = mlp
        m += 1
    return flax_params_to_flat(params, sh_deg, posenc)


# ---- flax.serialization msgpack encoding -------------------------------------------------------------------------
def _ndarray_to_bytes(arr):
    arr = np.asarray(arr)
    if arr.dtype.hasobject:
        raise ValueError("object arrays cannot be serialised")
    return msgpack.packb((list(arr.shape), arr.dtype.name, arr.tobytes("C")), use_bin_type=True)


def _ext_pack(x):
    if isinstance(x, np.ndarray):
        return msgpack.ExtType(_EXT_NDARRAY, _ndarray_to_bytes(x))
    if isinstance(x, np.generic):
        return msgpack.ExtType(_EXT_NPSCALAR, _ndarray_to_bytes(np.asarray(x)))
    if isinstance(x, complex):
        return msgpack.ExtType(_EXT_NATIVE_COMPLEX, msgpack.packb((x.real, x.imag)))
    return x


def _ext_unpack(code, data):
    if code == _EXT_NDARRAY:
        shape, dtype_name, buf = msgpack.unpackb(data, raw=True)
        return np.frombuffer(buf, dtype=np.dtype(dtype_name.decode() if isinstance(dtype_name, bytes) else dtype_name)
                             ).reshape([int(s) for s in shape]).copy()
    if code == _EXT_NPSCALAR:
        shape, dtype_name, buf = msgpack.unpackb(data, raw=True)
        return np.frombuffer(buf, dtype=np.dtype(dtype_name.decode() if isinstance(dtype_name, bytes) else dtype_name))[0]
    if code == _EXT_NATIVE_COMPLEX:
        re_, im_ = msgpack.unpackb(data)
        return complex(re_, im_)
    return msgpack.ExtType(code, data)


def msgpack_serialize(pytree):
    """flax.serialization.msgpack_serialize: nested dicts of numpy arrays / scalars -> bytes."""
    return msgpack.packb(pytree, default=_ext_pack, strict_types=True, use_bin_type=True)


def msgpack_restore(data):
    """flax.serialization.msgpack_restore."""
    return msgpack.unpackb(data, ext_hook=_ext_unpack, raw=False, strict_map_key=False)


# ---- TrainState <-> flax state dict ---------------------------------------------------------------------------
def train_state_dict(params_flat, m_flat, v_flat, step, sh_deg, posenc=None):
    """to_state_dict(utils.TrainState(optimizer=flax.optim.Adam(...).create(variables))):
    {"optimizer": {"target": {"params": ...}, "state": {"step": int32, "param_states": {"params": <same tree with
    {"grad_ema", "grad_sq_ema"} leaves>}}}}  (nerf_sh/nerf/models.py:44-48, flax.optim.Adam._AdamParamState)."""
    tgt = flat_to_flax_params(params_flat, sh_deg, posenc)
    gm = flat_to_flax_params(m_flat, sh_deg, posenc)
    gv = flat_to_flax_params(v_flat, sh_deg, posenc)
    ps = {}
    for mname in tgt:
        ps[mname] = {}
        for dname in tgt[mname]:
            ps[mname][dname] = {w: {"grad_ema": gm[mname][dname][w], "grad_sq_ema": gv[mname][dname][w]}
                                for w in ("kernel", "bias")}
    return {"optimizer": {"target": {"params": tgt},
                          "state": {"step": np.int32(step), "param_states": {"params": ps}}}}


def state_dict_to_flat(sd, sh_deg, posenc=None):
    """-> (params, m, v, step); m / v are None when the file holds no optimiser state."""
    opt = sd["optimizer"]
    params = flax_params_to_flat(opt["target"]["params"], sh_deg, posenc)
    m = v = None
    step = 0
    if "state" in opt and opt["state"] is not None:
        step = int(opt["state"].get("step", 0))
        ps = opt["state"].get("param_states", {}).get("params")
        if ps:
            gm = {mn: {dn: {w: ps[mn][dn][w]["grad_ema"] for w in ("kernel", "bias")} for dn in ps[mn]} for mn in ps}
            gv = {mn: {dn: {w: ps[mn][dn][w]["grad_sq_ema"] for w in ("kernel", "bias")} for dn in ps[mn]} for mn in ps}
            m, v = flax_params_to_flat(gm, sh_deg, posenc), flax_params_to_flat(gv, sh_deg, posenc)
    return params, m, v, step


# ---- files -------------------------------------------------------------------------------------------------------
def _natural_key(path):
    return [int(t) if t.isdigit() else t for t in re.split(r"(\d+)", os.path.basename(path))]


def latest_checkpoint(train_dir, prefix="checkpoint_"):
    """flax.training.checkpoints.latest_checkpoint: natural sort of <prefix>*."""
    paths = [p for p in glob.glob(os.path.join(train_dir, prefix + "*")) if not p.endswith(".tmp")]
    return sorted(paths, key=_natural_key)[-1] if paths else None


def save_checkpoint(train_dir, model, state, step=None, keep=100, prefix="checkpoint_"):
    """checkpoints.save_checkpoint(train_dir, state, int(step), keep=100)  (nerf_sh/train.py:237-242,306-310)."""
    step = int(state.step if step is None else step)
    os.makedirs(train_dir, exist_ok=True)
    sd = train_state_dict(model.params.detach().cpu().numpy(), state.m.detach().cpu().numpy(),
                          state.v.detach().cpu().numpy(), state.step, model.sh_deg, _posenc_of(model))
    path = os.path.join(train_dir, f"{prefix}{step}")
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        f.write(msgpack_serialize(sd))
    os.replace(tmp, path)
    old = sorted([p for p in glob.glob(os.path.join(train_dir, prefix + "*")) if not p.endswith(".tmp")],
                 key=_natural_key)
    for p in old[:-keep] if keep > 0 else []:
        os.remove(p)
    return path


def restore_flax_state_dict(train_dir_or_file, prefix="checkpoint_"):
    """checkpoints.restore_checkpoint(train_dir, target=None): the raw nested dict of the newest checkpoint."""
    path = train_dir_or_file
    if not os.path.exists(path):
        return None
    if os.path.isdir(path):
        path = latest_checkpoint(path, prefix)
        if path is None:
            return None
    with open(path, "rb") as f:
        return msgpack_restore(f.read())


def restore_checkpoint(train_dir, model, state=None):
    """checkpoints.restore_checkpoint(FLAGS.train_dir, state)  (nerf_sh/nerf/models.py:46-48; nerf_sh/eval.py):
    loads parameters (and, when `state` is given and the file has them, Adam moments and the step counter).
    Returns the restored step, or None when the directory holds no checkpoint (the reference then keeps the
    freshly initialised state)."""
    sd = restore_flax_state_dict(train_dir)
    if sd is None:
        return None
    params, m, v, step = state_dict_to_flat(sd, model.sh_deg, _posenc_of(model))
    model.set_params(params)
    if state is not None:
        import torch
        if m is not None:
            state.m.copy_(torch.from_numpy(m).to(state.m.device))
            state.v.copy_(torch.from_numpy(v).to(state.v.device))
        state.step = step
    return step


def save_torch_ckpt(path, model):
    """torch `*.ckpt` = {"model": state_dict} of the reference's torch twin (octree/nerf/models.py:52-63)."""
    import torch
    sd = {k: torch.from_numpy(np.ascontiguousarray(v))
          for k, v in flat_to_torch_state_dict(model.params.detach().cpu().numpy(), model.sh_deg,
                                                     _posenc_of(model)).items()}
    torch.save({"model": sd}, path)


def restore_model_state(train_dir, model):
    """models.restore_model_state (octree/nerf/models.py:52-63): newest *.ckpt of train_dir."""
    import torch
    paths = sorted(glob.glob(os.path.join(train_dir, "*.ckpt")))
    if not paths:
        return None
    ckpt = torch.load(paths[-1], map_location="cpu")
    sd = {k: v.numpy() for k, v in ckpt["model"].items()}
    model.set_params(torch_state_dict_to_flat(sd, model.sh_deg, _posenc_of(model)))
    return paths[-1]


def restore_model_state_from_jaxnerf(train_dir, model):
    """models.restore_model_state_from_jaxnerf (octree/nerf/models.py:66-113): parameters only."""
    sd = restore_flax_state_dict(train_dir)
    if sd is None:
        return None
    model.set_params(flax_params_to_flat(sd["optimizer"]["target"]["params"], model.sh_deg, _posenc_of(model)))
    return True


# ---- vanilla NeRF (use_viewdirs) parameters: octree.extraction's SH projection input -------------------------------
# Dense_0..7 trunk (point posenc width W), Dense_8 raw sigma [256, 1], Dense_9 bottleneck [256, 256] (no activation),
# Dense_10 condition layer [256 + 3 + 6 deg_view, 128] (rows [bottleneck | posenc(viewdir, 0, deg_view)]), Dense_11 rgb
# [128, 3] (octree/nerf/model_utils.py:112-158; the rgb layer is 3 wide whatever sh_deg is, models.py:296-305).  A
# vanilla parameter set is {"MLP_0": [(kernel [in, out], bias [out]) x 12], "MLP_1": ...} of fp32 numpy arrays.
_VANILLA_TORCH_NAMES = ([f"input_layers.{i}" for i in range(8)]
                        + ["sigma_layer", "bottleneck_layer", "condition_layers.0", "rgb_layer"])


def vanilla_layer_dims(posenc=None, deg_view=4):
    """(in, out) of Dense_0..Dense_11 of a vanilla NeRF MLP (net_depth_condition 1, net_width_condition 128)."""
    return (layer_dims(1, posenc_width(posenc))[:8]
            + [(256, 1), (256, 256), (256 + 3 + 6 * int(deg_view), 128), (128, 3)])


def _vanilla_check(mlps, posenc, deg_view):
    dims = vanilla_layer_dims(posenc, deg_view)
    if "MLP_0" not in mlps:
        raise ValueError("no MLP_0 in the parameter tree")
    for mname, layers in mlps.items():
        for i, ((k, b), (cin, cout)) in enumerate(zip(layers, dims)):
            if k.shape != (cin, cout) or b.shape != (cout,):
                hint = ("wrong min_deg_point / max_deg_point? Dense_0 has 3 + 6 (max_deg_point - min_deg_point) rows"
                        if i in (0, 5) else
                        "wrong deg_view? Dense_10 has 256 + 3 + 6 deg_view rows" if i == 10 else
                        "not a vanilla NeRF (net_depth_condition 1, net_width_condition 128, 3 rgb channels)?")
                raise ValueError(f"{mname}/Dense_{i}: expected kernel {(cin, cout)} and bias ({cout},), got "
                                 f"{k.shape} and {b.shape} ({hint})")
    return mlps


def vanilla_from_flax_params(params, posenc=None, deg_view=4):
    """["optimizer"]["target"]["params"] of a jaxnerf checkpoint -> vanilla parameter set (Dense_0..11 in order, as
    restore_model_state_from_jaxnerf maps them: octree/nerf/models.py:66-113)."""
    mlps = {}
    m = 0
    while f"MLP_{m}" in params:
        src = params[f"MLP_{m}"]
        layers = []
        for i in range(12):
            if f"Dense_{i}" not in src:
                raise ValueError(f"MLP_{m}/Dense_{i} is missing (a vanilla NeRF has Dense_0..Dense_11)")
            d = src[f"Dense_{i}"]
            layers.append((np.asarray(d["kernel"], dtype=np.float32), np.asarray(d["bias"], dtype=np.float32)))
        if "Dense_12" in src:
            raise ValueError(f"MLP_{m}/Dense_12: net_depth_condition 1 expected (Dense_0..Dense_11)")
        mlps[f"MLP_{m}"] = layers
        m += 1
    return _vanilla_check(mlps, posenc, deg_view)


def vanilla_to_flax_params(mlps):
    return {mname: {f"Dense_{i}": {"kernel": k, "bias": b} for i, (k, b) in enumerate(layers)}
            for mname, layers in mlps.items()}


def vanilla_from_torch_state_dict(sd, posenc=None, deg_view=4):
    """state_dict of the reference's torch NerfModel(use_viewdirs=True) (octree/nerf/models.py:52-63) -> vanilla
    parameter set; nn.Linear weight = kernel.T."""
    mlps = {}
    m = 0
    while f"MLP_{m}.input_layers.0.weight" in sd:
        layers = []
        for tname in _VANILLA_TORCH_NAMES:
            key = f"MLP_{m}.{tname}.weight"
            if key not in sd:
                raise ValueError(f"{key} is missing (a vanilla NeRF state_dict has {', '.join(_VANILLA_TORCH_NAMES)})")
            layers.append((np.asarray(sd[key], dtype=np.float32).T.copy(),
                           np.asarray(sd[f"MLP_{m}.{tname}.bias"], dtype=np.float32)))
        mlps[f"MLP_{m}"] = layers
        m += 1
    return _vanilla_check(mlps, posenc, deg_view)


def vanilla_to_torch_state_dict(mlps):
    return {f"{mname}.{tname}.{w}": (np.ascontiguousarray(k.T) if w == "weight" else b)
            for mname, layers in mlps.items() for tname, (k, b) in zip(_VANILLA_TORCH_NAMES, layers)
            for w in ("weight", "bias")}


def restore_vanilla(train_dir, is_jaxnerf_ckpt, posenc=None, deg_view=4):
    """the vanilla parameter set of train_dir: the newest flax checkpoint_<step> (is_jaxnerf_ckpt) or *.ckpt, as
    restore_model_state_from_jaxnerf / restore_model_state read them; None when there is none."""
    if is_jaxnerf_ckpt:
        sd = restore_flax_state_dict(train_dir)
        return None if sd is None else vanilla_from_flax_params(sd["optimizer"]["target"]["params"], posenc, deg_view)
    import torch
    paths = sorted(glob.glob(os.path.join(train_dir, "*.ckpt")))
    if not paths:
        return None
    ckpt = torch.load(paths[-1], map_location="cpu")
    return vanilla_from_torch_state_dict({k: v.numpy() for k, v in ckpt["model"].items()}, posenc, deg_view)

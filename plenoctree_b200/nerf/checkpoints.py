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


# ---- one MLP stack per on-disk format ----------------------------------------------------------------------------
# The format-neutral form of a checkpoint's parameters is {"MLP_0": [(kernel [in, out], bias [out]) per layer], ...}
# of fp32 numpy arrays; each family (NeRF-SH here, vanilla NeRF below) is a layer count and shape list of it.
def _mlp_names(present):
    """MLP_0, MLP_1, ... for as long as present(name) holds"""
    m = 0
    while present(f"MLP_{m}"):
        yield f"MLP_{m}"
        m += 1


def _from_flax(params, n_layers):
    """{"MLP_m": {"Dense_i": {"kernel", "bias"}}} (Dense_0..Dense_{n_layers - 1}) -> the neutral form"""
    return {mname: [(np.asarray(params[mname][f"Dense_{i}"]["kernel"], dtype=np.float32),
                     np.asarray(params[mname][f"Dense_{i}"]["bias"], dtype=np.float32)) for i in range(n_layers)]
            for mname in _mlp_names(params.__contains__)}


def _to_flax(mlps):
    return {mname: {f"Dense_{i}": {"kernel": k, "bias": b} for i, (k, b) in enumerate(layers)}
            for mname, layers in mlps.items()}


def _from_torch(sd, names):
    """{"MLP_m.<name>.weight" [out, in], ".bias"} of the reference's torch twin -> the neutral form (kernel =
    nn.Linear weight.T), one layer per entry of `names`"""
    return {mname: [(np.asarray(sd[f"{mname}.{t}.weight"], dtype=np.float32).T.copy(),
                     np.asarray(sd[f"{mname}.{t}.bias"], dtype=np.float32)) for t in names]
            for mname in _mlp_names(lambda mname: f"{mname}.input_layers.0.weight" in sd)}


def _to_torch(mlps, names):
    return {f"{mname}.{t}.{w}": (np.ascontiguousarray(k.T) if w == "weight" else b)
            for mname, layers in mlps.items() for t, (k, b) in zip(names, layers) for w in ("weight", "bias")}


def _check_shapes(mlps, dims, refusal):
    """refuses a parameter set without MLP_0 or with a layer that is not its (in, out) of `dims`;
    refusal(mlp name, layer, (in, out), kernel, bias) is the family's message, naming the flag that sets the shape"""
    if "MLP_0" not in mlps:
        raise ValueError("no MLP_0 in the parameter tree")
    for mname, layers in mlps.items():
        for i, ((k, b), want) in enumerate(zip(layers, dims)):
            if k.shape != want or b.shape != want[1:]:
                raise ValueError(refusal(mname, i, want, k, b))
    return mlps


_POSENC_HINT = "wrong min_deg_point / max_deg_point? Dense_0 has 3 + 6 (max_deg_point - min_deg_point) rows"


def _sh_refusal(mname, i, want, k, b):
    hint = _POSENC_HINT if i in (0, 5) and k.shape[1:] == want[1:] else "wrong sh_deg?"
    return f"{mname}/Dense_{i}: expected kernel {want}, got {k.shape} ({hint})"


# ---- NeRF-SH: flat [MLP_0 | MLP_1] <-> the neutral form -----------------------------------------------------------
def _split(flat, sh_deg, posenc):
    flat = np.asarray(flat, dtype=np.float32).reshape(-1)
    P = param_count(sh_deg, posenc)
    if flat.size % P != 0 or flat.size // P not in (1, 2):
        raise ValueError(f"expected {P} or {2 * P} parameters, got {flat.size}")
    mlps, off = {}, 0
    for m in range(flat.size // P):
        layers = []
        for cin, cout in _dims(sh_deg, posenc):
            layers.append((flat[off:off + cin * cout].reshape(cin, cout).copy(),
                           flat[off + cin * cout:off + cin * cout + cout].copy()))
            off += cin * cout + cout
        mlps[f"MLP_{m}"] = layers
    return mlps


def _join(mlps, sh_deg, posenc):
    mlps = _check_shapes(mlps, _dims(sh_deg, posenc), _sh_refusal)
    return np.concatenate([a.reshape(-1) for layers in mlps.values() for k, b in layers for a in (k, b)]
                          ).astype(np.float32)


def flat_to_flax_params(flat, sh_deg, posenc=None):
    """flat [num_mlps * P] -> {"MLP_0": {"Dense_i": {"kernel": [in,out], "bias": [out]}}, "MLP_1": ...}
    (the pytree under ["optimizer"]["target"]["params"], nerf_sh/nerf/model_utils.py:60-93)."""
    return _to_flax(_split(flat, sh_deg, posenc))


def flax_params_to_flat(params, sh_deg, posenc=None):
    return _join(_from_flax(params, len(_TORCH_NAMES)), sh_deg, posenc)


_TORCH_NAMES = [f"input_layers.{i}" for i in range(8)] + ["sigma_layer", "rgb_layer"]


def flat_to_torch_state_dict(flat, sh_deg, posenc=None):
    """-> {"MLP_0.input_layers.0.weight": [out,in], ...} as numpy arrays: the state_dict of the reference's torch
    twin (octree/nerf/models.py:116-209, octree/nerf/model_utils.py:36-95), nn.Linear weight = kernel.T."""
    return _to_torch(_split(flat, sh_deg, posenc), _TORCH_NAMES)


def torch_state_dict_to_flat(sd, sh_deg, posenc=None):
    return _join(_from_torch(sd, _TORCH_NAMES), sh_deg, posenc)


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


def _newest_torch_ckpt(train_dir):
    """(the "model" state_dict as numpy arrays, path) of the newest *.ckpt of train_dir; (None, None) when none"""
    import torch
    paths = sorted(glob.glob(os.path.join(train_dir, "*.ckpt")))
    if not paths:
        return None, None
    ckpt = torch.load(paths[-1], map_location="cpu")
    return {k: v.numpy() for k, v in ckpt["model"].items()}, paths[-1]


def restore_model_state(train_dir, model):
    """models.restore_model_state (octree/nerf/models.py:52-63): newest *.ckpt of train_dir."""
    sd, path = _newest_torch_ckpt(train_dir)
    if sd is None:
        return None
    model.set_params(torch_state_dict_to_flat(sd, model.sh_deg, _posenc_of(model)))
    return path


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
# vanilla parameter set is the neutral form itself, 12 layers an MLP.
_VANILLA_TORCH_NAMES = ([f"input_layers.{i}" for i in range(8)]
                        + ["sigma_layer", "bottleneck_layer", "condition_layers.0", "rgb_layer"])


def vanilla_layer_dims(posenc=None, deg_view=4):
    """(in, out) of Dense_0..Dense_11 of a vanilla NeRF MLP (net_depth_condition 1, net_width_condition 128)."""
    return (layer_dims(1, posenc_width(posenc))[:8]
            + [(256, 1), (256, 256), (256 + 3 + 6 * int(deg_view), 128), (128, 3)])


def _vanilla_refusal(mname, i, want, k, b):
    hint = (_POSENC_HINT if i in (0, 5) else
            "wrong deg_view? Dense_10 has 256 + 3 + 6 deg_view rows" if i == 10 else
            "not a vanilla NeRF (net_depth_condition 1, net_width_condition 128, 3 rgb channels)?")
    return (f"{mname}/Dense_{i}: expected kernel {want} and bias ({want[1]},), got {k.shape} and {b.shape} "
            f"({hint})")


def vanilla_from_flax_params(params, posenc=None, deg_view=4):
    """["optimizer"]["target"]["params"] of a jaxnerf checkpoint -> vanilla parameter set (Dense_0..11 in order, as
    restore_model_state_from_jaxnerf maps them: octree/nerf/models.py:66-113)."""
    for mname in _mlp_names(params.__contains__):
        for i in range(12):
            if f"Dense_{i}" not in params[mname]:
                raise ValueError(f"{mname}/Dense_{i} is missing (a vanilla NeRF has Dense_0..Dense_11)")
        if "Dense_12" in params[mname]:
            raise ValueError(f"{mname}/Dense_12: net_depth_condition 1 expected (Dense_0..Dense_11)")
    return _check_shapes(_from_flax(params, 12), vanilla_layer_dims(posenc, deg_view), _vanilla_refusal)


vanilla_to_flax_params = _to_flax


def vanilla_from_torch_state_dict(sd, posenc=None, deg_view=4):
    """state_dict of the reference's torch NerfModel(use_viewdirs=True) (octree/nerf/models.py:52-63) -> vanilla
    parameter set; nn.Linear weight = kernel.T."""
    for mname in _mlp_names(lambda mname: f"{mname}.input_layers.0.weight" in sd):
        for tname in _VANILLA_TORCH_NAMES:
            if f"{mname}.{tname}.weight" not in sd:
                raise ValueError(f"{mname}.{tname}.weight is missing (a vanilla NeRF state_dict has "
                                 f"{', '.join(_VANILLA_TORCH_NAMES)})")
    return _check_shapes(_from_torch(sd, _VANILLA_TORCH_NAMES), vanilla_layer_dims(posenc, deg_view),
                         _vanilla_refusal)


def vanilla_to_torch_state_dict(mlps):
    return _to_torch(mlps, _VANILLA_TORCH_NAMES)


def restore_vanilla_and_step(train_dir, is_jaxnerf_ckpt, posenc=None, deg_view=4):
    """(the vanilla parameter set of train_dir, its step): the newest flax checkpoint_<step> (is_jaxnerf_ckpt) or
    *.ckpt, as restore_model_state_from_jaxnerf / restore_model_state read them; the step is the flax file's (0 for
    a torch file).  (None, None) when there is none."""
    if is_jaxnerf_ckpt:
        sd = restore_flax_state_dict(train_dir)
        if sd is None:
            return None, None
        step = int((sd["optimizer"].get("state") or {}).get("step", 0))
        return vanilla_from_flax_params(sd["optimizer"]["target"]["params"], posenc, deg_view), step
    sd, _ = _newest_torch_ckpt(train_dir)
    return (None, None) if sd is None else (vanilla_from_torch_state_dict(sd, posenc, deg_view), 0)


def restore_vanilla(train_dir, is_jaxnerf_ckpt, posenc=None, deg_view=4):
    """the vanilla parameter set of restore_vanilla_and_step; None when there is none."""
    return restore_vanilla_and_step(train_dir, is_jaxnerf_ckpt, posenc, deg_view)[0]

"""Models with every NeRF-SH flag (encoder, activations, SM count, L2 discard): flag helpers, fp64 activations and
encoder features, canaries."""
import types

import numpy as np
import pytest
import torch

from oracle import net_activation_oracle as NA, posenc_oracle as PO
from plenoctree_b200 import _lib, layouts as L


SP_BAR = 4.0            # softplus in the heads epilogue, in units of u * softplus64(x)
SP_FLOOR = 2.0 ** -148  # absolute: expf's denormal outputs below x = -87


def softplus64(x):
    x = torch.as_tensor(x).double()
    return x.clamp_min(0) + torch.log1p(torch.exp(-x.abs()))


def _scope_args(**kw):
    base = dict(use_viewdirs=False, sg_dim=-1, dataset="blender", net_depth=8, net_width=256, skip_layer=4,
                min_deg_point=0, max_deg_point=10, net_activation="relu", rgb_activation="sigmoid",
                sigma_activation="relu", legacy_posenc_order=False, render_path=False, spherify=False)
    base.update(kw)
    return types.SimpleNamespace(**base)


def _ref_features(x, pe):
    """fp64 sines of the kernel's fp32 arguments: [M, W - 3] in the encoder's column order"""
    cols = []
    half_pi = torch.tensor(np.float32(np.pi / 2), device=x.device)
    for kind, j, c in PO.feature_index(pe)[3:]:
        xb = x[:, c] * float(2 ** j)                                 # exact fp32 product
        cols.append(torch.sin((xb if kind == "sin" else xb + half_pi).double()))
    return torch.stack(cols, 1) if cols else torch.zeros(x.shape[0], 0, dtype=torch.float64, device=x.device)


def _act64(act, z):
    return NA.activation(act)(z)


def _set_flags(**kw):
    from plenoctree_b200.nerf import flags as F
    F.define_flags()
    if not F.FLAGS.is_parsed():
        F.FLAGS.mark_as_parsed()
    for k, v in kw.items():
        setattr(F.FLAGS, k, v)
    return F.FLAGS


def _device_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _set_sms(monkeypatch, n):
    """make the library split its work for n SMs ("device": POB_SM_COUNT unset) until the test ends"""
    from plenoctree_b200._lib import lib
    dev = _device_sms()
    if n == "device":
        monkeypatch.delenv("POB_SM_COUNT", raising=False)
        n = dev
    else:
        if n > dev:
            pytest.skip(f"{n} SMs: the device has {dev}")
        monkeypatch.setenv("POB_SM_COUNT", str(n))
    assert lib.pob_sm_count() == n
    return n


def _alt_pe(pe):
    """an encoder of the same width that differs from pe: the other feature order, or (one degree) shifted degrees
    where both orders coincide; None for W = 3 (no sines)"""
    mn, mx, legacy = pe
    if mn == mx:
        return None
    if mx - mn == 1:
        return (mn - 1, mx - 1, legacy) if mn > 0 else (mn + 1, mx + 1, legacy)
    return (mn, mx, not legacy)


RAYS, NC, NF, NSP = 4096, 64, 128, 10000     # the production SH16 step (bench.py)
FILL = 0x5A


def _model(sh_deg, nf, nsp, near=2.0, far=6.0, R=RAYS):
    from plenoctree_b200.nerf.models import NerfModel
    model = NerfModel(sh_deg=sh_deg, num_coarse_samples=NC, num_fine_samples=nf, near=near, far=far,
                      white_bkgd=True, max_rays=R, sparsity_npoints=nsp)
    model.init_params(20200823)
    return model


def _batch(R, seed):
    from plenoctree_b200.nerf.models import Rays
    from plenoctree_b200.nerf.utils import random_rays_np
    o, d, v, px = random_rays_np(R, seed)
    b = torch.from_numpy(np.concatenate([o, d, v, px], axis=1)).cuda()
    return {"rays": Rays(b[:, 0:3], b[:, 3:6], b[:, 6:9]), "pixels": b[:, 9:12]}, b


def _call(model, state, batch, keep, precision=_lib.PREC_FP16, **kw):
    """loss_and_grad from a workspace filled with FILL; returns (grads, stats_raw, workspace bytes)"""
    from plenoctree_b200.nerf import train as T
    ws = model.workspace(True, precision)
    ws.fill_(FILL)
    T.loss_and_grad(model, state, batch, precision=precision, keep_saved_tiles=keep, **kw)
    torch.cuda.synchronize()
    return state.grads.clone(), state.stats_raw.clone(), ws.clone()


def _saved_grad_ranges(model, R, sparsity_on):
    """[start, end) byte ranges of the DZ and DO images the call writes"""
    views = L.train_workspace_views(model.cfg, R, sparsity_on)
    out = []
    for v in views["levels"]:
        for name in ("DZ", "DO"):
            off, shape = v[name]
            out.append((off, off + int(np.prod(shape))))
    return out


def _equal_outside(w0, w1, ranges):
    start = 0
    for a, b in sorted(ranges) + [(w0.numel(), w0.numel())]:
        if not torch.equal(w0[start:a], w1[start:a]):
            return False
        start = b
    return True


CANARY = 0x7FBADBAD         # a NaN bit pattern behind every output


def _canary(shape, tail=1024):
    """(int32 buffer of the canary, float32 view of its first prod(shape) words)"""
    n = int(np.prod(shape))
    buf = torch.full((n + tail,), CANARY, dtype=torch.int32, device="cuda")
    return buf, buf[:n].view(torch.float32).view(shape)


def _points(n, seed):
    rs = np.random.RandomState(seed)
    return torch.from_numpy(rs.uniform(-1.2, 1.2, size=(n, 3)).astype(np.float32)).cuda()


def _run_points(nerf, pts):
    """pob_sh_proj_points on a 0xFF workspace and canary outputs -> (ws, a, sigma, a_buf, sigma_buf)"""
    from plenoctree_b200._lib import check, lib, posenc_ref, ptr, stream_ptr
    m = pts.shape[0]
    ws = torch.full((int(lib.pob_sh_proj_points_workspace_bytes(m)),), 0xFF, dtype=torch.uint8, device="cuda")
    ab, a = _canary((m, 128))
    sb, s = _canary((m,))
    check(lib.pob_sh_proj_points(ptr(nerf.sigma_blob), posenc_ref(nerf._pe), ptr(pts), m, ptr(nerf.head_w),
                                 ptr(nerf.head_b), ptr(ws), ptr(a), ptr(s), stream_ptr()))
    torch.cuda.synchronize()
    return ws, a, s, ab, sb

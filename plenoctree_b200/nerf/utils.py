"""Host utilities mirrored from the reference for the hot path's callers (numpy only, no math kernels).

    Rays namedtuple          nerf_sh/nerf/utils.py:53
    pose_spherical           nerf_sh/nerf/utils.py:656-685
    generate_rays            nerf_sh/nerf/utils.py:545-589
    learning_rate_decay      nerf_sh/nerf/utils.py:483-515   (in train.py)
"""
import numpy as np

from .rays import Rays, generate_rays, pose_spherical, random_rays_np  # noqa: F401  (numpy only)


def render_image(model, rays, normalize_disp=False, chunk=8192, precision=None):
    """utils.render_image (nerf_sh/nerf/utils.py:331-381): render all the pixels of an image (test mode,
    randomized=False) in chunks of `chunk` rays; with torch.distributed initialised every rank renders a
    contiguous slice of each chunk (reference: shard over devices + all_gather, utils.py:357-371,701-706).

    rays: Rays of [H, W, 3] arrays.  Returns rgb [H,W,3], disp [H,W,1], acc [H,W,1] (torch CUDA tensors)."""
    import torch
    import torch.distributed as dist
    from .models import Rays, _cuda_f32

    height, width = rays.origins.shape[:2]
    num_rays = height * width
    flat = Rays(*[_cuda_f32(np.ascontiguousarray(r).reshape(num_rays, -1) if isinstance(r, np.ndarray)
                            else r.reshape(num_rays, -1), "rays") for r in rays])
    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank() if world > 1 else 0
    chunk = min(chunk, model.max_rays * world)
    out = []
    for i in range(0, num_rays, chunk):
        n = min(chunk, num_rays - i)
        per = (n + world - 1) // world
        lo, hi = min(n, rank * per), min(n, (rank + 1) * per)
        part = torch.zeros((per, 5), dtype=torch.float32, device=model.device)
        if hi > lo:
            sl = Rays(*[r[i + lo:i + hi] for r in flat])
            rgb, disp, acc = model(sl, randomized=False, precision=precision)[-1]
            part[:hi - lo, :3], part[:hi - lo, 3], part[:hi - lo, 4] = rgb, disp, acc
        if world > 1:
            full = torch.empty((world * per, 5), dtype=torch.float32, device=model.device)
            dist.all_gather_into_tensor(full, part)
            part = full
        out.append(part[:n])
    res = torch.cat(out, 0)
    rgb, disp, acc = res[:, :3], res[:, 3:4], res[:, 4:5]
    if normalize_disp:   # utils.py:376-378
        disp = (disp - disp.min()) / (disp.max() - disp.min())
    return rgb.reshape(height, width, 3), disp.reshape(height, width, 1), acc.reshape(height, width, 1)


def eval_points(model, points, chunk=720720, to_cpu=False, coarse=False, precision=None):
    """utils.eval_points (nerf_sh/nerf/utils.py:282-328): raw SH coefficients and sigma of arbitrary points,
    evaluated chunk by chunk.  Returns (raw_rgb [M,3K], raw_sigma [M,1])."""
    import torch
    from .models import _cuda_f32

    points = _cuda_f32(points, "points", 3)
    rgbs, sigmas = [], []
    for i in range(0, points.shape[0], chunk):
        rgb, sigma = model.eval_points_raw(points[i:i + chunk], coarse=coarse, precision=precision)
        rgbs.append(rgb.cpu() if to_cpu else rgb)
        sigmas.append(sigma.cpu() if to_cpu else sigma)
    return torch.cat(rgbs, 0), torch.cat(sigmas, 0)


def compute_psnr(mse):
    """utils.compute_psnr (nerf_sh/nerf/utils.py:384-393)."""
    return -10.0 * np.log(mse) / np.log(10.0)


def compute_ssim(img0, img1, max_val=1.0, filter_size=11, filter_sigma=1.5, k1=0.01, k2=0.03, return_map=False,
                 padding="valid"):
    """utils.compute_ssim: mean SSIM of two [H,W,C] images with the separable 11-tap Gaussian window and clipped
    (co)variances.  The reference has two border conventions: the JAX side convolves "valid"
    (nerf_sh/nerf/utils.py:396-466, used by nerf_sh.train / eval), its torch twin zero-pads to "same"
    (octree/nerf/utils.py:322-400, used by octree evaluation; golden-pinned in tests/golden/ssim.npz)."""
    import torch
    import torch.nn.functional as F
    a = torch.as_tensor(img0, dtype=torch.float32)
    b = torch.as_tensor(img1, dtype=torch.float32).to(a.device)
    hw = filter_size // 2
    shift = (2 * hw - filter_size + 1) / 2
    f_i = ((torch.arange(filter_size, dtype=torch.float32, device=a.device) - hw + shift) / filter_sigma) ** 2
    filt = torch.exp(-0.5 * f_i)
    filt = filt / filt.sum()

    def blur(z):                                  # [H,W,C] -> valid separable blur
        z = z.permute(2, 0, 1)[:, None]           # [C,1,H,W]
        ph = filter_size // 2 if padding == "same" else 0
        z = F.conv2d(z, filt[None, None, None, :], padding=[0, ph])
        z = F.conv2d(z, filt[None, None, :, None], padding=[ph, 0])
        return z[:, 0].permute(1, 2, 0)

    mu0, mu1 = blur(a), blur(b)
    mu00, mu11, mu01 = mu0 * mu0, mu1 * mu1, mu0 * mu1
    sigma00 = torch.clamp(blur(a * a) - mu00, min=0.0)
    sigma11 = torch.clamp(blur(b * b) - mu11, min=0.0)
    sigma01 = blur(a * b) - mu01
    sigma01 = torch.sign(sigma01) * torch.minimum(torch.sqrt(sigma00 * sigma11), torch.abs(sigma01))
    c1, c2 = (k1 * max_val) ** 2, (k2 * max_val) ** 2
    ssim_map = ((2 * mu01 + c1) * (2 * sigma01 + c2)) / ((mu00 + mu11 + c1) * (sigma00 + sigma11 + c2))
    return ssim_map if return_map else ssim_map.mean()


def save_img(img, pth):
    """utils.save_img (nerf_sh/nerf/utils.py:469-480): float image in [0,1] ([H,W,3] or [H,W]) -> PNG."""
    from PIL import Image
    arr = img.detach().cpu().numpy() if hasattr(img, "detach") else np.asarray(img)
    Image.fromarray((np.clip(arr, 0.0, 1.0) * 255.0).astype(np.uint8)).save(pth, "PNG")


def write_video(path, frames, fps):
    """frames [n,h,w,3] float in [0,1] -> mp4 (OpenCV's mp4v writer stands in for imageio.mimwrite, which this image
    does not carry); returns False when no encoder is available."""
    try:
        import cv2
    except ImportError:
        return False
    h, w = frames.shape[1:3]
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), float(fps), (w, h))
    if not vw.isOpened():
        return False
    for f in frames:
        vw.write(np.ascontiguousarray((np.clip(f, 0.0, 1.0) * 255).astype(np.uint8)[..., ::-1]))     # RGB -> BGR
    vw.release()
    return True

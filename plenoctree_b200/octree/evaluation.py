"""`python -m plenoctree_b200.octree.evaluation` and `eval_octree` (octree/evaluation.py:75-123,
octree/nerf/utils.py:448-498): render every test view of a PlenOctree, PSNR / SSIM against the ground truth
LPIPS is added when its downloaded weights can be found (nerf/lpips.py), else reported as nan.  `--write_disp DIR`
writes each view's disparity map as `disp_{i:04d}.png`, as nerf_sh.eval does for the NeRF.  `--input` may also be a
compressed tree written by octree.compression (quantised or --noquant), rendered as stored.  Forward-facing scenes
('llff' in --config, not --spherify) are rendered in NDC (renderer.scene_ndc).  There `--write_disp` writes acc / depth
with depth a distance along the unit NDC direction, so its maps differ from nerf_sh.eval's for the same model, whose
depth is the parameter t along the un-normalised NDC direction: by that direction's length per pixel, about 2 near the
image centre."""
import os

import numpy as np
import torch

from ..nerf.utils import compute_psnr, compute_ssim, save_img, write_video
from .n3tree import load_tree
from .renderer import VolumeRenderer, disparity, scene_ndc


def eval_octree(t, dataset, args, want_frames=False, lpips_fn=None, metrics=None, disp_fn=None):
    """utils.eval_octree (octree/nerf/utils.py:448-498): -> (avg_psnr, avg_ssim[, frames]).  With `lpips_fn`
    (nerf/lpips.py::load_lpips) the mean LPIPS(gt, render) is left in `metrics["lpips"]`.  With `disp_fn`, each view's
    disparity [H,W,1] (renderer.disparity of the same render's depth and acc) is passed to disp_fn(idx, disp)."""
    w, h, focal = dataset.w, dataset.h, dataset.focal
    ndc = scene_ndc(args, w, h, focal)
    r = VolumeRenderer(t, step_size=args.renderer_step_size, **({} if ndc is None else {"ndc": ndc}))
    avg_psnr = avg_ssim = avg_lpips = 0.0
    frames = []
    with torch.no_grad():
        for idx in range(dataset.size):
            c2w = dataset.camtoworlds[idx]
            im_gt = torch.from_numpy(dataset.images[idx]).float().to(t.device)
            if disp_fn is None:
                im = r.render_persp(c2w, width=w, height=h, fx=focal, fast=not args.no_early_stop)
            else:
                im, depth, acc = r.render_persp(c2w, width=w, height=h, fx=focal, fast=not args.no_early_stop,
                                                return_depth=True)
                disp_fn(idx, disparity(depth, acc))
            im = im.clamp_(0.0, 1.0)
            mse = float(((im - im_gt) ** 2).mean())
            avg_psnr += float(compute_psnr(mse))
            avg_ssim += float(compute_ssim(im, im_gt, max_val=1.0, padding="same"))   # octree/nerf/utils.py twin
            if lpips_fn is not None:
                avg_lpips += lpips_fn(im_gt.permute(2, 0, 1).contiguous(), im.permute(2, 0, 1).contiguous())
            if want_frames:
                frames.append((im.cpu().numpy() * 255).astype(np.uint8))
    n = max(dataset.size, 1)
    if metrics is not None:
        metrics["lpips"] = avg_lpips / n if lpips_fn is not None else float("nan")
    return (avg_psnr / n, avg_ssim / n, frames) if want_frames else (avg_psnr / n, avg_ssim / n)


def _define_cli_flags():
    from ..nerf import flags as F
    F.define_flags(octree=True)
    F.define({"input": ("string", "./tree.npz", "Input octree npz"),
              "write_vid": ("string", None, "If specified, writes rendered video to given path (*.mp4)"),
              "write_images": ("string", None, "If specified, writes rendered images to this directory"),
              "write_disp": ("string", None, "If specified, writes disparity maps (disp_XXXX.png) to this directory")})
    return F


def _cli_main(argv):
    main(argv)          # absl exits with main's return value; the command line exits 0 on success


def main(unused_argv):
    from ..nerf import datasets
    F = _define_cli_flags()
    FLAGS = F.FLAGS
    F.update_flags(FLAGS)
    dev = torch.device("cuda")
    dataset = datasets.get_dataset("test", FLAGS, device=dev)
    t = load_tree(FLAGS.input, map_location=dev)      # tree.npz, or a compressed one (octree.compression)
    from ..nerf.lpips import load_lpips
    extra = {}
    disp_fn = None
    if FLAGS.write_disp:
        os.makedirs(FLAGS.write_disp, exist_ok=True)

        def disp_fn(i, disp):    # nerf_sh.eval: save_img(pred_disp[..., 0]), i.e. disparity clipped to [0, 1]
            save_img(disp[..., 0], os.path.join(FLAGS.write_disp, f"disp_{i:04d}.png"))
    psnr, ssim, frames = eval_octree(t, dataset, FLAGS, want_frames=True, lpips_fn=load_lpips(dev), metrics=extra,
                                     disp_fn=disp_fn)
    print("Average PSNR", psnr, "SSIM", ssim, "LPIPS", extra["lpips"])
    if FLAGS.write_vid and frames:
        # evaluation.py:88-90: imageio.mimwrite at its default 10 fps
        print("Writing to", FLAGS.write_vid)
        if not write_video(FLAGS.write_vid, np.stack(frames).astype(np.float32) / 255.0, 10):
            print("* No mp4 encoder available: frames only")
    if FLAGS.write_images:
        os.makedirs(FLAGS.write_images, exist_ok=True)
        for i, fr in enumerate(frames):
            save_img(fr.astype(np.float32) / 255.0, os.path.join(FLAGS.write_images, f"{i:04d}.png"))
    return psnr, ssim


if __name__ == "__main__":
    from absl import app
    _define_cli_flags()       # before app.run parses the command line
    app.run(_cli_main)

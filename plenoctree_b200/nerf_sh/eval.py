"""`python -m plenoctree_b200.nerf_sh.eval` — the reference's `nerf_sh.eval` CLI (nerf_sh/eval.py:45-133): restore the
newest checkpoint of train_dir, render every test image deterministically (randomized=False), write
`test_preds/{idx:03d}.png`, `disp_{idx:03d}.png`, and the PSNR / SSIM summaries (psnr.txt, ssim.txt,
psnrs_<step>.txt, ssims_<step>.txt — the block the reference keeps commented out at eval.py:99-127).  With
use_viewdirs (nerf_sh/config/misc/og_nerf) the model is a vanilla NeRF (nerf/vanilla.py), restored from a flax
checkpoint_<step> or a torch *.ckpt."""
import os

import numpy as np
import torch
from absl import app

from ..nerf import datasets, flags as F, models, utils

FLAGS = F.FLAGS
F.define_flags()


def main(unused_argv):
    F.update_flags(FLAGS)
    F.check_flags(FLAGS)
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    model, step = models.load_for_inference(FLAGS, dev, max_rays=min(FLAGS.chunk, 8192))
    dataset = datasets.get_dataset("test", FLAGS, device=dev)
    out_dir = os.path.join(FLAGS.train_dir, "path_renders" if FLAGS.render_path else "test_preds")   # eval.py:63-65
    if FLAGS.save_output:
        os.makedirs(out_dir, exist_ok=True)
    psnrs, ssims = [], []
    for idx in range(dataset.size):
        batch = dataset.next_test()
        if idx % FLAGS.approx_eval_skip != 0:
            continue
        pred_color, pred_disp, pred_acc = utils.render_image(model, batch["rays"], chunk=FLAGS.chunk)
        if FLAGS.render_path:                          # generated camera path (llff): frames only, no ground truth
            if FLAGS.save_output:
                utils.save_img(pred_color, os.path.join(out_dir, f"{idx:03d}.png"))
                utils.save_img(pred_disp[..., 0], os.path.join(out_dir, f"disp_{idx:03d}.png"))
            continue
        gt = torch.from_numpy(batch["pixels"]).to(pred_color.device)
        psnr = float(utils.compute_psnr(float(((pred_color - gt) ** 2).mean())))
        ssim = float(utils.compute_ssim(pred_color, gt, max_val=1.0))
        print(f"Evaluating {idx + 1}/{dataset.size}: PSNR = {psnr:.4f}, SSIM = {ssim:.4f}", flush=True)
        psnrs.append(psnr)
        ssims.append(ssim)
        if FLAGS.save_output:
            utils.save_img(pred_color, os.path.join(out_dir, f"{idx:03d}.png"))
            utils.save_img(pred_disp[..., 0], os.path.join(out_dir, f"disp_{idx:03d}.png"))
    if FLAGS.render_path:
        return None, None
    if FLAGS.save_output:
        for name, val in (("psnr.txt", np.mean(psnrs)), ("ssim.txt", np.mean(ssims))):
            with open(os.path.join(out_dir, name), "w") as f:
                f.write(f"{val}")
        with open(os.path.join(out_dir, f"psnrs_{step}.txt"), "w") as f:
            f.write(" ".join(str(v) for v in psnrs))
        with open(os.path.join(out_dir, f"ssims_{step}.txt"), "w") as f:
            f.write(" ".join(str(v) for v in ssims))
    print(f"Average PSNR {np.mean(psnrs):.4f} SSIM {np.mean(ssims):.4f}")
    return float(np.mean(psnrs)), float(np.mean(ssims))


if __name__ == "__main__":
    app.run(main)

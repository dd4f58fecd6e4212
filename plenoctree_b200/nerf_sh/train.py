"""`python -m plenoctree_b200.nerf_sh.train` — the reference's `nerf_sh.train` CLI (nerf_sh/train.py:124-314) over the
CUDA library: same flags / YAML configs / train_dir layout (flax-format `checkpoint_<step>`, tensorboard scalars,
`render/` test renders).  One process per GPU: launch with torchrun for data parallelism (batch_size is global and
split over ranks like the reference splits it over devices)."""
import functools
import gc
import os
import time

import numpy as np
import torch
import torch.distributed as dist
from absl import app, flags

from .._lib import PREC_FP16, PREC_FP16X3
from ..nerf import checkpoints, datasets, flags as F, models, train as T, utils

FLAGS = F.FLAGS
F.define_flags()
# not a reference flag: fp16x3 trains with error-compensated operands (fp32-class gradients, DESIGN.md section 3)
if "train_precision" not in FLAGS:
    flags.DEFINE_enum("train_precision", "fp16", ["fp16", "fp16x3"],
                      "tensor-core operands of the training step: fp16, or the hi + lo split fp16x3.")
_TRAIN_PRECISION = {"fp16": PREC_FP16, "fp16x3": PREC_FP16X3}


from .._dist import dist_init as _dist_init  # noqa: E402


def main(unused_argv):
    rank, world, dev = _dist_init()
    F.update_flags(FLAGS)
    F.check_flags(FLAGS, world=world)
    F.check_model_scope(FLAGS)
    torch.manual_seed(20200823 + rank)
    os.makedirs(FLAGS.train_dir, exist_ok=True)
    render_dir = os.path.join(FLAGS.train_dir, "render")
    os.makedirs(render_dir, exist_ok=True)
    h0print = print if rank == 0 else (lambda *a, **k: None)

    h0print("* Load train data")
    dataset = datasets.get_dataset("train", FLAGS, device=dev, rank=rank, world=world)
    h0print("* Load test data")
    test_dataset = datasets.get_dataset("test", FLAGS, device=dev)
    h0print("* Load model")
    per_rank = FLAGS.batch_size // world
    margs = type("A", (), dict(sh_deg=FLAGS.sh_deg, sigma_activation=FLAGS.sigma_activation,
                               net_activation=FLAGS.net_activation,
                               min_deg_point=FLAGS.min_deg_point, max_deg_point=FLAGS.max_deg_point,
                               legacy_posenc_order=FLAGS.legacy_posenc_order,
                               num_coarse_samples=FLAGS.num_coarse_samples,
                               num_fine_samples=FLAGS.num_fine_samples, near=FLAGS.near, far=FLAGS.far,
                               white_bkgd=FLAGS.white_bkgd, lindisp=FLAGS.lindisp,
                               batch_size=per_rank,   # workspace capacity; test renders chunk by it
                               sparsity_npoints=FLAGS.sparsity_npoints if FLAGS.sparsity_weight > 0 else 0,
                               train_dir=FLAGS.train_dir))
    model, state = models.get_model_state(margs, device=dev, restore=True)
    model.noise_std = FLAGS.noise_std
    learning_rate_fn = functools.partial(T.learning_rate_decay, lr_init=FLAGS.lr_init, lr_final=FLAGS.lr_final,
                                         max_steps=FLAGS.max_steps, lr_delay_steps=FLAGS.lr_delay_steps,
                                         lr_delay_mult=FLAGS.lr_delay_mult)
    init_step = state.step + 1                       # resume at the step of the last checkpoint (train.py:176)
    writer = None
    if rank == 0:
        try:
            from torch.utils.tensorboard import SummaryWriter
            writer = SummaryWriter(FLAGS.train_dir)
        except Exception:
            writer = None
    gc.disable()                                      # train.py:188
    stats_trace = []
    t_loop_start = time.time()
    for step in range(init_step, FLAGS.max_steps + 1):
        batch = dataset.next_train()
        lr = learning_rate_fn(step)
        want_stats = rank == 0 and (step % FLAGS.print_every == 0 or step == FLAGS.max_steps)
        stats = T.train_step(model, state, batch, lr, sparsity_weight=FLAGS.sparsity_weight,
                             sparsity_length=FLAGS.sparsity_length, sparsity_radius=FLAGS.sparsity_radius,
                             weight_decay_mult=FLAGS.weight_decay_mult, randomized=FLAGS.randomized,
                             sync_stats=want_stats, precision=_TRAIN_PRECISION[FLAGS.train_precision])
        if step % FLAGS.gc_every == 0:
            gc.collect()
        if rank == 0 and stats is not None:
            stats_trace.append(stats)
            steps_per_sec = (FLAGS.print_every if step % FLAGS.print_every == 0 else 1) / (time.time() - t_loop_start)
            t_loop_start = time.time()
            rays_per_sec = FLAGS.batch_size * steps_per_sec
            if writer:
                for k, v in (("train_loss", stats.loss), ("train_psnr", stats.psnr), ("train_loss_coarse", stats.loss_c),
                             ("train_psnr_coarse", stats.psnr_c), ("weight_l2", stats.weight_l2),
                             ("learning_rate", lr), ("train_steps_per_sec", steps_per_sec),
                             ("train_rays_per_sec", rays_per_sec)):
                    writer.add_scalar(k, v, step)
                if FLAGS.sparsity_weight > 0.0:
                    writer.add_scalar("train_sparse_loss", stats.loss_sp, step)
            precision = int(np.ceil(np.log10(FLAGS.max_steps))) + 1
            print(("{:" + "{:d}".format(precision) + "d}").format(step) + f"/{FLAGS.max_steps:d}: "
                  + f"i_loss={stats.loss:0.4f}, psnr={stats.psnr:0.2f}, weight_l2={stats.weight_l2:0.2e}, "
                  + f"lr={lr:0.2e}, {rays_per_sec:0.0f} rays/sec", flush=True)
        if rank == 0 and (step % FLAGS.save_every == 0 or step == FLAGS.max_steps):
            print("* Saving")
            checkpoints.save_checkpoint(FLAGS.train_dir, model, state, int(step), keep=200)
        if FLAGS.render_every > 0 and step % FLAGS.render_every == 0:
            test_case = test_dataset.next_test()
            pred_color, pred_disp, pred_acc = utils.render_image(model, test_case["rays"], chunk=FLAGS.chunk)
            if rank == 0:
                gt = torch.from_numpy(test_case["pixels"]).to(pred_color.device)
                psnr = utils.compute_psnr(float(((pred_color - gt) ** 2).mean()))
                ssim = float(utils.compute_ssim(pred_color, gt, max_val=1.0))
                print(f"* Rendering: test psnr {psnr:.4f} ssim {ssim:.4f}", flush=True)
                if writer:
                    writer.add_scalar("test_psnr", psnr, step)
                    writer.add_scalar("test_ssim", ssim, step)
                utils.save_img(pred_color, os.path.join(render_dir, f"{step:07d}.png"))
    if writer:
        writer.close()
    gc.enable()
    if world > 1:
        dist.barrier()
    return model, state


if __name__ == "__main__":
    app.run(main)

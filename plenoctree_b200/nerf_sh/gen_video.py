"""`python -m plenoctree_b200.nerf_sh.gen_video` — the reference's `nerf_sh.gen_video` CLI (nerf_sh/gen_video.py:52-176):
restore the newest checkpoint of train_dir, render `num_views` frames from a circle of `pose_spherical` cameras at
the given elevation / radius / up axis through `render_image` (randomized=False), write
`<train_dir>/video/e<elev*10>/frames/NNNN.png` and `video.mp4` (OpenCV's mp4v writer stands in for imageio, which
this image does not carry; without OpenCV the frames alone are written).  Under torchrun every rank renders its slice
of each frame and rank 0 writes the files."""
import os

import numpy as np
from absl import app, flags

from .. import _dist
from ..nerf import flags as F, models, utils
from ..nerf.models import Rays
from ..nerf.rays import generate_rays, pose_spherical
from ..nerf.utils import write_video

FLAGS = F.FLAGS
F.define_flags()
F.define({       # nerf_sh/gen_video.py:52-106
    "elevation": ("float", -30.0, "Elevation angle (negative is above)"),
    "num_views": ("integer", 40, "The number of views to generate."),
    "height": ("integer", 800, "The size of images to generate."),
    "width": ("integer", 800, "The size of images to generate."),
    "camera_angle_x": ("float", 0.7, "The camera angle in rad in x direction (used to get focal length)."),
    "intrin": ("string", None, "Intrinsics file. If set, overrides camera_angle_x"),
    "radius": ("float", 4.0, "Radius to origin of camera path."),
    "fps": ("integer", 20, "FPS of generated video"),
    "up_axis": ("integer", 1, "up axis for camera views; 1-6: Z up/Z down/Y up/Y down/X up/X down"),
    "write_poses": ("string", None, "Specify to write poses to given file (4N x 4), does not write poses else"),
})
if "A" not in FLAGS:
    flags.DEFINE_alias("A", "camera_angle_x")


def orbit_poses(num_views, elevation, radius, up_axis):
    """[num_views,4,4] cameras on a circle around the up axis (gen_video.py:113-119; up_axis is 1-based)."""
    angles = np.linspace(-180, 180, num_views + 1)[:-1]
    return np.stack([pose_spherical(a, elevation, radius, up_axis - 1) for a in angles], 0)


def main(unused_argv):
    F.update_flags(FLAGS)
    F.check_flags(FLAGS, require_data=False)
    rank, world, dev = _dist.dist_init()
    model, _ = models.load_for_inference(FLAGS, dev, max_rays=min(FLAGS.chunk, 8192))
    render_poses = orbit_poses(FLAGS.num_views, FLAGS.elevation, float(FLAGS.radius), FLAGS.up_axis)
    if FLAGS.write_poses and rank == 0:
        np.savetxt(FLAGS.write_poses, render_poses.reshape(-1, 4))
        print("Saved poses to", FLAGS.write_poses)
    focal = 0.5 * FLAGS.width / np.tan(0.5 * FLAGS.camera_angle_x)
    if FLAGS.intrin is not None:
        K = np.loadtxt(FLAGS.intrin)
        focal = (K[0, 0] + K[1, 1]) * 0.5
    video_dir = os.path.join(FLAGS.train_dir, "video", "e{:03}".format(int(-FLAGS.elevation * 10)))
    frames_dir = os.path.join(video_dir, "frames")
    if rank == 0:
        os.makedirs(frames_dir, exist_ok=True)
        print(" Saving to", video_dir)
    frames = []
    for i in range(FLAGS.num_views):
        rays = generate_rays(FLAGS.width, FLAGS.height, focal, render_poses[i:i + 1])      # one frame at a time
        pred_color, _, _ = utils.render_image(model, Rays(*[r[0] for r in rays]), chunk=FLAGS.chunk,
                                              normalize_disp=FLAGS.dataset == "llff")
        if rank == 0:
            utils.save_img(pred_color, os.path.join(frames_dir, f"{i:04}.png"))
            frames.append(pred_color.detach().cpu().numpy())
            print(f"** View {i + 1}/{FLAGS.num_views}", flush=True)
    if rank == 0:
        vid_path = os.path.join(video_dir, "video.mp4")
        if write_video(vid_path, np.stack(frames), FLAGS.fps):
            print("* Wrote video", vid_path)
        else:
            print("* No mp4 encoder available: frames only")
    _dist.dist_finish()
    return video_dir


if __name__ == "__main__":
    app.run(main)

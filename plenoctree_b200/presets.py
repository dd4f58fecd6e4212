"""Built-in stand-ins for the reference's shipped configuration files, so that the README command lines
(`--config nerf_sh/config/blender`, `python -m octree.task_manager octree/config/syn_sh16.json ...`) work in a
checkout that does not carry those files: when the named file does not exist, its base name selects a preset.
A file on disk always wins.  Values: nerf_sh/config/{blender,tt,misc/proj,misc/og_nerf}.yaml,
octree/config/{syn_sh16,tt_sh25}.json.
"""
import os

_NERF_SH_COMMON = dict(image_batching=False, factor=0, num_coarse_samples=64, num_fine_samples=128,
                       use_viewdirs=False, white_bkgd=True, batch_size=1024, randomized=True, max_steps=2000000)

NERF_SH = {
    # NeRF-synthetic, SH16
    "blender": dict(_NERF_SH_COMMON, dataset="blender", sh_deg=3),
    # Tanks and Temples (NSVF layout), SH25, wider sparsity prior
    "tt": dict(_NERF_SH_COMMON, dataset="nsvf", sh_deg=4, near=0.0, far=4.0, sparsity_radius=5.0, sparsity_length=0.2),
    # misc/proj: a vanilla NeRF (use_viewdirs) projected to an SH25 tree by octree.extraction
    "proj": dict(_NERF_SH_COMMON, dataset="blender", use_viewdirs=True, sh_deg=4),
    # misc/og_nerf: the original NeRF (use_viewdirs, plain RGB head), evaluated by nerf_sh.eval / gen_video
    "og_nerf": dict(_NERF_SH_COMMON, dataset="blender", use_viewdirs=True, sparsity_weight=0.0),
}


def nerf_sh_preset(config):
    """flags of `--config <path>` when <path>.yaml is absent and basename(<path>) names a preset, else None."""
    return NERF_SH.get(os.path.basename(str(config)))


def _flags(**kw):
    out = []
    for k, v in kw.items():
        out += [f"--{k}"] if v is True else [f"--{k}", str(v)]
    return out


def _syn_task(scene, radius="1.4", **extra):
    extr = _flags(autoscale=True, **extra, scale_alpha_thresh="0.1", radius=radius, samples_per_cell=256,
                  no_early_stop=True, renderer_step_size="1e-5")
    return {"octree_name": "", "train_dir": scene, "data_dir": scene, "config": "nerf_sh/config/blender",
            "extr_flags": extr,
            "opt_flags": _flags(num_epochs=80, sgd=True, lr="1e7", no_early_stop=True, renderer_step_size="1e-5"),
            "eval_flags": _flags(renderer_step_size="1e-5")}


def _tt_task(scene, bbox_scale="1.0"):
    return {"octree_name": "", "train_dir": scene, "data_dir": scene, "config": "nerf_sh/config/tt",
            "extr_flags": _flags(autoscale=True, scale_alpha_thresh="0.1", bbox_from_data=True, data_bbox_scale="1.2",
                                 bbox_scale=bbox_scale, samples_per_cell=256, chunk=8192, no_early_stop=True,
                                 renderer_step_size="1e-5"),
            "opt_flags": _flags(num_epochs=40, sgd=True, lr="1.5e6", renderer_step_size="1e-5", split_train=True,
                                split_holdout_prop="0.1"),
            "eval_flags": _flags(renderer_step_size="1e-5")}


def octree_tasks_preset(path):
    """task-file contents for octree.task_manager when `path` is absent and its base name is a preset, else None."""
    name = os.path.splitext(os.path.basename(str(path)))[0]
    if name == "syn_sh16":
        return {"data_root": "./data/NeRF/nerf_synthetic/", "train_root": "./data/Plenoctree/checkpoints/syn_sh16/",
                "scenes": ["chair", "drums", "ficus", "hotdog", "lego", "ship"], "scene_tasks": [_syn_task("{%}")],
                "tasks": [_syn_task("materials", bbox_scale="1.1"), _syn_task("mic", radius="1.6")]}
    if name == "tt_sh25":
        return {"data_root": "./data/TanksAndTemple", "train_root": "./data/Plenoctree/checkpoints/tt_sh25/",
                "scenes": ["Barn", "Caterpillar", "Family", "Truck"], "scene_tasks": [_tt_task("{%}")],
                "tasks": [_tt_task("Ignatius", bbox_scale="1.25")]}
    return None

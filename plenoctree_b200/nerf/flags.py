"""The reference's command-line flags (nerf_sh/nerf/utils.py:60-253, octree/nerf/utils.py:60-253) as absl flags with
the same names and defaults, and `update_flags` (utils.py:233-244): a YAML file `<config>.yaml` overrides them, so the
reference's own config files (nerf_sh/config/blender.yaml, tt.yaml) drive this package unchanged.

Flags that select features outside the scope of this path are accepted (so existing command lines keep parsing) and
rejected by `check_model_scope` (every CLI's check) when set to an unsupported value."""
import os

import yaml
from absl import flags

FLAGS = flags.FLAGS

# name -> (kind, default, help)
_COMMON = {
    "train_dir": ("string", None, "where to store ckpts and logs"),
    "data_dir": ("string", None, "input data directory."),
    "config": ("string", None, "using config files to set hyperparameters."),
    "dataset": ("string", "blender", "The type of dataset feed to nerf."),
    "image_batching": ("bool", False, "sample rays in a batch from different images."),
    "white_bkgd": ("bool", True, "using white color as default background."),
    "batch_size": ("integer", 1024, "the number of rays in a mini-batch (for training)."),
    "factor": ("integer", 4, "the downsample factor of images, 0 for no downsample."),
    "spherify": ("bool", False, "set for spherical 360 scenes."),
    "render_path": ("bool", False, "render generated path if set true."),
    "llffhold": ("integer", 8, "will take every 1/N images as LLFF test set."),
    "model": ("string", "nerf", "name of model to use."),
    "near": ("float", 2.0, "near clip of volumetric rendering."),
    "far": ("float", 6.0, "far clip of volumentric rendering."),
    "net_depth": ("integer", 8, "depth of the first part of MLP."),
    "net_width": ("integer", 256, "width of the first part of MLP."),
    "net_depth_condition": ("integer", 1, "depth of the second part of MLP."),
    "net_width_condition": ("integer", 128, "width of the second part of MLP."),
    "weight_decay_mult": ("float", 0.0, "The multiplier on weight decay"),
    "skip_layer": ("integer", 4, "add a skip connection to the output vector of every skip_layer layers."),
    "num_rgb_channels": ("integer", 3, "the number of RGB channels."),
    "num_sigma_channels": ("integer", 1, "the number of density channels."),
    "randomized": ("bool", True, "use randomized stratified sampling."),
    "min_deg_point": ("integer", 0, "Minimum degree of positional encoding for points."),
    "max_deg_point": ("integer", 10, "Maximum degree of positional encoding for points."),
    "deg_view": ("integer", 4, "Degree of positional encoding for viewdirs."),
    "num_coarse_samples": ("integer", 64, "the number of samples on each ray for the coarse model."),
    "num_fine_samples": ("integer", 128, "the number of samples on each ray for the fine model."),
    "use_viewdirs": ("bool", True, "use view directions as a condition."),
    "sh_deg": ("integer", -1, "set to use SH output up to given degree, -1 = disable."),
    "sg_dim": ("integer", -1, "set to use spherical gaussians (SG). -1 = disable"),
    "noise_std": ("float", None, "std dev of noise added to regularize sigma output."),
    "lindisp": ("bool", False, "sampling linearly in disparity rather than depth."),
    "net_activation": ("string", "relu", "activation function used within the MLP."),
    "rgb_activation": ("string", "sigmoid", "activation function used to produce RGB."),
    "sigma_activation": ("string", "relu", "activation function used to produce density."),
    "legacy_posenc_order": ("bool", False, "revert the positional encoding feature order to an older version."),
    "lr_init": ("float", 5e-4, "The initial learning rate."),
    "lr_final": ("float", 5e-6, "The final learning rate."),
    "lr_delay_steps": ("integer", 0, "steps at the beginning of training to reduce the learning rate"),
    "lr_delay_mult": ("float", 1.0, "A multiplier on the learning rate when the step is < lr_delay_steps"),
    "max_steps": ("integer", 1000000, "the number of optimization steps."),
    "save_every": ("integer", 10000, "the number of steps to save a checkpoint."),
    "print_every": ("integer", 1000, "the number of steps between reports to tensorboard."),
    "render_every": ("integer", 20000, "the number of steps to render a test image."),
    "gc_every": ("integer", 5000, "the number of steps to run python garbage collection."),
    "sparsity_weight": ("float", 1e-3, "Sparsity loss weight"),
    "sparsity_length": ("float", 0.05, "Sparsity loss 'length' for alpha calculation"),
    "sparsity_radius": ("float", 1.5, "Sparsity loss point sampling box 1/2 side length"),
    "sparsity_npoints": ("integer", 10000, "Number of samples for sparsity loss"),
    "eval_once": ("bool", True, "evaluate the model only once if true."),
    "save_output": ("bool", True, "save predicted images to disk if True."),
    "chunk": ("integer", 8192, "the size of chunks for evaluation inferences."),
    "approx_eval_skip": ("integer", 1, "Evaluates only every x images"),
    # octree side (octree/nerf/utils.py:210-225)
    "renderer_step_size": ("float", 1e-4, "step size epsilon in volume render."),
    "no_early_stop": ("bool", False, "If set, does not use early stopping in the octree renderer."),
}

_DEFINERS = {"string": flags.DEFINE_string, "bool": flags.DEFINE_bool, "integer": flags.DEFINE_integer,
             "float": flags.DEFINE_float}


def define(table):
    for name, (kind, default, helptxt) in table.items():
        if name not in FLAGS:
            _DEFINERS[kind](name, default, helptxt)


# defaults that differ on the octree side of the reference (octree/nerf/utils.py:44-219 vs nerf_sh/nerf/utils.py:60-253)
_OCTREE_DEFAULTS = {"chunk": 81920, "gc_every": 10000, "print_every": 500, "render_every": 10000, "save_every": 5000,
                    "net_activation": "ReLU", "rgb_activation": "Sigmoid", "sigma_activation": "ReLU"}


def define_flags(octree=False):
    """nerf_sh side by default; octree=True applies the octree side's defaults (octree.extraction / optimization /
    evaluation are separate programs in the reference, each with its own copy of define_flags)."""
    define(_COMMON)
    if octree:
        for name, value in _OCTREE_DEFAULTS.items():
            FLAGS.set_default(name, value)


def update_flags(args):
    """utils.update_flags (nerf_sh/nerf/utils.py:233-244): `<config>.yaml` overrides existing flags only."""
    if getattr(args, "config", None) is None:
        return
    pth = os.path.expanduser(args.config + ".yaml")
    if not os.path.exists(pth):
        from ..presets import nerf_sh_preset          # the reference's shipped configs, by base name
        configs = nerf_sh_preset(args.config)
        if configs is None:
            raise FileNotFoundError(pth)
    else:
        with open(pth, "r") as fin:
            configs = yaml.load(fin, Loader=yaml.FullLoader)
    known = set(args) if hasattr(args, "__iter__") else set(dir(args))
    invalid = sorted(set(configs.keys()) - known)
    if invalid:
        raise ValueError(f"Invalid args {invalid} in {pth}.")
    for k, v in configs.items():
        setattr(args, k, v)


def check_flags(args, require_data=True, world=1):
    """utils.check_flags (nerf_sh/nerf/utils.py:247-253)."""
    if args.train_dir is None:
        raise ValueError("train_dir must be set. None set now.")
    if require_data and args.data_dir is None:
        raise ValueError("data_dir must be set. None set now.")
    if args.batch_size % world != 0:
        raise ValueError("Batch size must be divisible by the number of devices.")


SIGMA_ACTIVATIONS = {"relu": 0, "softplus": 1}   # _lib.SIGMA_RELU / SIGMA_SOFTPLUS


def sigma_activation_code(name):
    """flag sigma_activation -> POB_SIGMA_* code.  The nerf_sh side names flax's nn.relu / nn.softplus, the octree
    side torch's nn.ReLU / nn.Softplus (octree/nerf/utils.py:136), so the name is matched case-insensitively."""
    code = SIGMA_ACTIVATIONS.get(str(name).lower())
    if code is None:
        raise NotImplementedError(f"sigma_activation {name!r}: relu or softplus expected")
    return code


# flag net_activation: the trunk activations the kernels build (_lib.NET_*), by their flax (nn.elu) and torch
# (nn.ELU) names.  Each is 1-Lipschitz with a derivative that is a function of its output, so the training step forms
# it from the saved activations.  gelu / swish / silu need the pre-activation, which the step does not save.
NET_ACTIVATIONS = {"relu": 0, "elu": 1, "softplus": 2, "tanh": 3}
_NET_NEEDS_PREACTIVATION = ("gelu", "swish", "silu")


def net_activation_code(name):
    """flag net_activation -> POB_NET_* code, matched case-insensitively like sigma_activation_code (the octree
    side's default is torch's "ReLU")."""
    key = str(name).lower()
    code = NET_ACTIVATIONS.get(key)
    if code is not None:
        return code
    if key in _NET_NEEDS_PREACTIVATION:
        raise NotImplementedError(
            f"net_activation {name!r}: its derivative needs the pre-activation, which the training step does not "
            "save (the data gradient forms f'(h) from the saved activations h); relu, elu, softplus or tanh expected")
    raise NotImplementedError(f"net_activation {name!r} is not built: relu, elu, softplus or tanh expected")


POSENC_MAX_DEG = 10


def check_posenc(min_deg_point, max_deg_point):
    """flags min_deg_point / max_deg_point (either legacy_posenc_order) that the kernels take: 0 <= min <= max <= 10.
    The W = 3 + 6 (max - min) features must fit the 64-column posenc tile beside its constant-one bias column
    (W <= 63), and the top scale 2^(max - 1) must stay inside the posenc sine's accurate range."""
    mn, mx = int(min_deg_point), int(max_deg_point)
    if not 0 <= mn <= mx <= POSENC_MAX_DEG:
        raise NotImplementedError(
            f"posenc degrees min_deg_point={mn}, max_deg_point={mx}: 0 <= min_deg_point <= max_deg_point <= 10 "
            f"expected (the width 3 + 6 (max - min) = {3 + 6 * (mx - mn)} must fit the 64-column posenc tile with its "
            "bias column, and scales above 2^9 leave the posenc sine's range)")


MAX_RAY_SAMPLES = 1024


def check_samples(num_coarse_samples, num_fine_samples):
    """flags num_coarse_samples / num_fine_samples that the per-ray kernels take: 3 <= Nc and Nc + Nf <= 1024.  A ray
    is one warp up to 256 samples and four warps (one 128-thread block, 8 samples per lane) up to 1024; resampling
    needs at least one interior coarse weight."""
    nc, nf = int(num_coarse_samples), int(num_fine_samples)
    bound = f"3 <= num_coarse_samples and num_coarse_samples + num_fine_samples <= {MAX_RAY_SAMPLES}"
    if nc < 3 or nf < 0:
        raise ValueError(f"num_coarse_samples={nc}, num_fine_samples={nf}: {bound} and num_fine_samples >= 0 expected "
                         "(resampling draws from the coarse weights between the first and the last sample)")
    if nc + nf > MAX_RAY_SAMPLES:
        raise NotImplementedError(
            f"num_coarse_samples={nc}, num_fine_samples={nf}: {bound} expected (the per-ray kernels hold at most "
            f"{MAX_RAY_SAMPLES} samples of a ray, 8 per thread of one 128-thread block)")


def check_scope(args):
    """features of the reference the relu-trunk path does not cover: fail loudly instead of training something else.
    A model with another trunk activation is checked by check_model_scope, which every CLI calls."""
    if args.use_viewdirs:
        raise NotImplementedError("use_viewdirs (vanilla NeRF colour head) is outside the NeRF-SH path")
    if args.sg_dim > 0:
        raise NotImplementedError("spherical gaussians (sg_dim) are outside the NeRF-SH path")
    if args.dataset not in ("blender", "llff", "nsvf"):
        raise NotImplementedError(f"dataset {args.dataset!r}: blender, llff or nsvf expected")
    if (args.net_depth, args.net_width, args.skip_layer) != (8, 256, 4):
        raise NotImplementedError("the fused kernel is built for the 8x256 trunk with the skip after layer 4")
    check_posenc(args.min_deg_point, args.max_deg_point)
    check_samples(getattr(args, "num_coarse_samples", 64), getattr(args, "num_fine_samples", 128))
    if (str(args.net_activation).lower(), str(args.rgb_activation).lower()) != ("relu", "sigmoid"):
        raise NotImplementedError("activations other than relu (trunk) / sigmoid (rgb)")
    sigma_activation_code(args.sigma_activation)
    if (args.render_path or args.spherify) and args.dataset != "llff":
        raise ValueError("render_path / spherify apply to the llff dataset only")        # datasets.py:194-195,496-497


class _Trunk:
    """`args` with its net_activation replaced (absl FlagValues cannot be copied field by field)"""

    def __init__(self, args, net_activation):
        self._args, self.net_activation = args, net_activation

    def __getattr__(self, name):
        return getattr(self._args, name)


def check_model_scope(args):
    """check_scope for a model with any trunk activation the kernels build: net_activation relu, elu, softplus or
    tanh in any case (net_activation_code, which refuses the others and says why), every other flag as check_scope
    has it."""
    net_activation_code(args.net_activation)
    check_scope(_Trunk(args, "relu"))


class _Override:
    """`args` with some flags replaced (absl FlagValues cannot be copied field by field)"""

    def __init__(self, args, **values):
        self._args, self._values = args, values

    def __getattr__(self, name):
        return self._values[name] if name in self._values else getattr(self._args, name)


MAX_DEG_VIEW = 32


def check_projection_scope(args):
    """octree.extraction of a vanilla NeRF (use_viewdirs): the SH projection of its view branch
    (octree/extraction.py:217-241,362-394).  Accepts sh_deg 1-4, the reference's condition branch
    (net_depth_condition 1, net_width_condition 128), a relu trunk and condition layer, 0 <= deg_view <= 32, and every
    point-posenc, sample, dataset and density flag check_scope accepts.  Training, rendering and evaluating a vanilla
    NeRF stay refused by check_scope."""
    sh_deg = int(args.sh_deg)
    if not 1 <= sh_deg <= 4:
        raise NotImplementedError(
            f"sh_deg={sh_deg}: projecting a vanilla NeRF needs an SH tree, 1 <= sh_deg <= 4 (with sh_deg 0 or less the "
            "reference writes projected coefficients into an RGBA tree, and sh_deg -1 fails its order >= 0 assert)")
    if (int(args.net_depth_condition), int(args.net_width_condition)) != (1, 128):
        raise NotImplementedError(
            f"net_depth_condition={args.net_depth_condition}, net_width_condition={args.net_width_condition}: the "
            "projection kernel is built for one 128-wide condition layer (1, 128)")
    if not 0 <= int(args.deg_view) <= MAX_DEG_VIEW:
        raise NotImplementedError(
            f"deg_view={args.deg_view}: 0 <= deg_view <= {MAX_DEG_VIEW} expected (scales above 2^31 of a unit "
            "direction are below the resolution of an fp32 sine's argument)")
    check_scope(_Override(args, use_viewdirs=False))

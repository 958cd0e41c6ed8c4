"""The reference's command-line parameters (arguments/__init__.py, arguments_games/__init__.py) and its cfg_args file.

Every parameter group adds its flags in declaration order, `--name` plus `-n` (the first letter) for the ones the reference
marks as shorthand; booleans are store_true flags.  The order matters: cfg_args is the repr of an argparse Namespace, whose
keys follow the order the parser declared them in."""
from __future__ import annotations

import ast
import os
from argparse import ArgumentParser, Namespace

# (name, default, shorthand)
MODEL_PARAMS = (("sh_degree", 3, False), ("source_path", "", True), ("model_path", "", True), ("images", "images", True),
                ("resolution", -1, True), ("white_background", False, True), ("data_device", "cuda", False), ("eval", False, False))
PIPELINE_PARAMS = (("convert_SHs_python", False, False), ("compute_cov3D_python", False, False), ("debug", False, False),
                   ("antialiasing", False, False))
# OptimizationParams (gs, gs_flat)
OPT_PARAMS_FREE = (("iterations", 30_000), ("position_lr_init", 0.00016), ("position_lr_final", 0.0000016),
                   ("position_lr_delay_mult", 0.01), ("position_lr_max_steps", 30_000), ("feature_lr", 0.0025), ("opacity_lr", 0.05),
                   ("scaling_lr", 0.005), ("rotation_lr", 0.001), ("percent_dense", 0.01), ("lambda_dssim", 0.2),
                   ("densification_interval", 100), ("opacity_reset_interval", 3000), ("densify_from_iter", 500),
                   ("densify_until_iter", 15_000), ("densify_grad_threshold", 0.0002), ("random_background", False))
# OptimizationParamsMesh (gs_mesh)
OPT_PARAMS_MESH = (("iterations", 30_000), ("vertices_lr", 0.0), ("alpha_lr", 0.001), ("feature_lr", 0.0025), ("opacity_lr", 0.05),
                   ("scaling_lr", 0.005), ("rotation_lr", 0.001), ("random_background", False), ("use_mesh", True),
                   ("lambda_dssim", 0.2))
# OptimizationParamsFlame (gs_flame)
OPT_PARAMS_FLAME = (("iterations", 30_000), ("alpha_lr", 0.001), ("feature_lr", 0.0025), ("opacity_lr", 0.05), ("scaling_lr", 0.005),
                    ("rotation_lr", 0.001), ("flame_shape_lr", 0.01), ("flame_exp_lr", 0.001), ("flame_pose_lr", 0.001),
                    ("flame_neck_pose_lr", 0.001), ("flame_trans_lr", 0.001), ("vertices_enlargement_lr", 0.0002),
                    ("random_background", False), ("use_mesh", True), ("lambda_dssim", 0.2))

# what train.py's ModelParams.extract keeps (the group's own keys plus the three train.py sets on it) -> cfg_args
MODEL_KEYS = tuple(n for n, _, _ in MODEL_PARAMS) + ("num_splats", "meshes", "gs_type")


def add_group(parser: ArgumentParser, title: str, params, fill_none: bool = False) -> None:
    """ParamGroup.__init__: one flag per parameter; fill_none gives every flag the default None (render.py's sentinel)."""
    group = parser.add_argument_group(title)
    for p in params:
        name, default = p[0], p[1]
        short = len(p) > 2 and p[2]
        flags = ["--" + name] + (["-" + name[0]] if short else [])
        value = None if fill_none else default
        if type(default) is bool:
            group.add_argument(*flags, default=value, action="store_true")
        else:
            group.add_argument(*flags, default=value, type=type(default))


def cfg_args_string(args: Namespace) -> str:
    """What prepare_output_and_logger writes to cfg_args: the Namespace of the model parameters, source_path absolute."""
    d = {k: v for k, v in vars(args).items() if k in MODEL_KEYS}
    d["source_path"] = os.path.abspath(d["source_path"])
    return str(Namespace(**d))


def parse_cfg_args(text: str) -> Namespace:
    """A cfg_args file back into a Namespace, without eval: the text must be one Namespace(...) call whose keyword values are
    Python literals (a `**{...}` literal dict too, as Namespace's repr writes keys that are not identifiers)."""
    try:
        node = ast.parse(text.strip(), mode="eval").body
    except SyntaxError as e:
        raise ValueError(f"cfg_args is not a Namespace(...) expression: {e}") from None
    if not (isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == "Namespace" and not node.args):
        raise ValueError("cfg_args must hold a single Namespace(...) call with keyword arguments")
    out = {}
    for kw in node.keywords:
        value = ast.literal_eval(kw.value)
        if kw.arg is None:
            if not isinstance(value, dict):
                raise ValueError("cfg_args: ** must expand a literal dict")
            out.update(value)
        else:
            out[kw.arg] = value
    return Namespace(**out)


def combined_args(parser: ArgumentParser, argv) -> Namespace:
    """get_combined_args (arguments/__init__.py:93-113) on `argv`: the model directory's cfg_args, overridden by every
    command-line value that is not None."""
    cmdline = parser.parse_args(argv)
    cfg = Namespace()
    if cmdline.model_path is not None:
        path = os.path.join(cmdline.model_path, "cfg_args")
        if os.path.exists(path):
            with open(path) as f:
                cfg = parse_cfg_args(f.read())
    merged = vars(cfg).copy()
    for k, v in vars(cmdline).items():
        if v is not None:
            merged[k] = v
    return Namespace(**merged)

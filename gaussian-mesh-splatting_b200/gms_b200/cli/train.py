"""python -m gms_b200.cli.train -s <scene> [-m <output>] [--gs_type gs_mesh|gs_multi_mesh|gs_flame|gs_flat|gs] ...: the
reference's train.py on the native trainers.

Flags, defaults and the output directory are the reference's (cfg_args, cameras.json, input.ply -- input_<i>.ply per mesh
for gs_multi_mesh --, point_cloud/iteration_N/point_cloud.ply [+ model_params.pt or flame_params.pt], chkpnt<N>.pth).
gs_multi_mesh trains on a COLMAP scene with --meshes a b ... (sparse/0/<name>.obj) and one --num_splats per mesh
(MultiMeshGaussianModel, MeshTrainer); gs_flame on a NeRF-synthetic scene with the FLAME model file --flame_model
(NativeFlame, FlameTrainer).  One iteration, in train.py's order
(train.py:61-157):

    [--viewer: the remote viewer's requests] -> SH degree up every 1000 -> the view from the Scene's view order ->
    background (torch.rand(3) on the device under --random_background) -> the one-call training frame -> training_report at --test_iterations -> Scene.save at
    --save_iterations -> densify / opacity reset (gs, gs_flat) -> Adam on every iteration but the last -> checkpoint at
    --checkpoint_iterations.

The report and the save run inside the trainer's `before_update` callback, so they see the parameters after N-1 updates,
as the reference's do.  The loop itself never synchronises with the host: the loss reaches the progress display's moving
average through pinned host slots and CUDA events that are polled, not waited on.

Remote viewer, opt-in with --viewer (train.py:65-79 with network_gui.init, which the reference leaves commented out):
--ip / --port are bound before the output folder is written (--port 0 binds a free port, printed and held in
Training.viewer.address; an address that cannot be bound is an error naming it), and the listener and any connection are
closed when run() returns or raises.  At the very top of every iteration a waiting SIBR viewer is accepted (one at a
time) and its requests are answered (network_gui.serve_iteration) until one says `train` and (the iteration is not the
last, or not `keep_alive`): a viewer that sends `train: false` pauses the run, and `keep_alive` holds the last iteration.
A frame shows the parameters after N-1 updates at iteration N-1's active SH degree, with the fixed background (also
under --random_background) and the request's scaling modifier; the verify string is the absolute source path.  A paused
iteration draws no view, no background and no random number, so pausing does not change the run; iter_time and the loss
display do not include viewer time.  A frame is cli.view's (view.Frames) on the trainer's live model: gs_mesh and
gs_multi_mesh expanded from the raw parameters Adam updates in place; gs and gs_flat at the current Gaussian count (a
renderer sized before a densification is replaced); gs_flame at its current FLAME parameters, one FLAME forward and one
expansion per frame, drawn as cli.view draws a checkpoint saved at that moment.  Each frame costs one host
synchronisation; a run with --viewer and no viewer connected synchronises no more than one without it.  Without
--viewer no socket is opened.

TensorBoard, as prepare_output_and_logger / training_report (train.py:174-223): when torch.utils.tensorboard imports, a
SummaryWriter(model_path) gets every iteration's train_loss_patches/l1_loss, train_loss_patches/total_loss and iter_time
(ms), and at each --test_iterations entry the first five renders of each split (and their ground truth at the first listed
test iteration), the split's loss_viewpoint - l1_loss / - psnr, scene/opacity_histogram and total_points; else it prints
"Tensorboard not available: not logging progress".  The three per-iteration values travel through the same pinned slots
(loss and L1, elements 0 and 1 of the frame's loss vector) with a pair of timing events per slot, and are written, as ONE
event per iteration, once the slot's events have completed.  TensorBoard's writer spends its host time per event (a
protobuf, a checksum in Python, a file append), so one event for the three values costs a third of three add_scalar calls.

Views may differ in size, as the reference's cameras each carry their own (a COLMAP scene with several cameras, or source
images of different sizes before -r rescales them): the trainer's one frame is sized for the largest training width and
height and runs every view at the view's own size, training_report scores each size through its own renderer (the split
means average the per-view values in float64) and its TensorBoard images are each at their view's size.

Deliberate differences:
  * chkpnt<N>.pth holds (state, N) with the library's own state (the trainer's state_dict(), the view-order stream and the
    background generator), not the reference's capture() tuple; a resumed run continues the uninterrupted run's sequence of
    views and backgrounds, where the reference re-shuffles.
  * --seed (default 0) seeds what safe_state seeds: the view shuffle and order, the initial model and the backgrounds.
  * gs_multi_mesh without --meshes, or with a --num_splats count other than the --meshes count, is refused (the reference's
    zip would drop the unmatched meshes); so are gs_multi_mesh on a NeRF-synthetic scene and gs_flame on a COLMAP scene, on
    which the reference crashes, and gs_flame without its model file.
  * flame_params.pt carries the FLAME buffers as NativeFlame.to_point_cloud()'s dict, not the reference's pickled
    FLAMEPointCloud: cli.render and cli.render_flame rebuild the model from the checkpoint alone.
  * TensorBoard: the per-iteration scalars are written when their slot is consumed, as one event per iteration holding
    all three (the reference writes one event per tag), so the order of events across tags in the file differs from the
    reference's (per tag, steps increase as there).  iter_time brackets the frame's launches, which on one GPU include
    the SH Adam step the frame fuses into the preprocess backward (and for gs_flame the FLAME forward and backward); the
    reference's window holds render, loss and backward only.  The writer is closed when run() returns or raises.
  * Not built, refused by name: --antialiasing, --debug, --debug_from, --detect_anomaly,
    --convert_SHs_python, --compute_cov3D_python, --save_xyz, --data_device other than cuda.  --ip / --port are only read
    under --viewer (the reference does not start its viewer at all)."""
from __future__ import annotations

import collections
import json
import os
import random
import shutil
import sys
import uuid
from argparse import ArgumentParser, Namespace
from types import SimpleNamespace
from typing import List

import numpy as np
import torch

from .. import _lib, dataset, expansion, io_ply, network_gui
from ..model import FlameGaussianModel, FreeGaussianModel, MeshGaussianModel, MultiMeshGaussianModel
from ..scenes import MeshGaussianParams
from ..trainer import FlameOptimizationParams, FlameTrainer, FreeOptimizationParams, FreeTrainer, MeshTrainer
from . import options

GS_TYPES = ("gs_mesh", "gs_multi_mesh", "gs_flame", "gs_flat", "gs")
FREE_TYPES = ("gs", "gs_flat")
MESH_TYPES = ("gs_mesh", "gs_multi_mesh")       # MeshTrainer: OptimizationParamsMesh, SH degree up in the loop
# flags of the reference that the native training frames do not implement: (name, default)
REFUSED = (("debug_from", -1), ("detect_anomaly", False), ("save_xyz", False), ("convert_SHs_python", False),
           ("compute_cov3D_python", False), ("debug", False), ("antialiasing", False))


def build_parser(gs_type: str) -> ArgumentParser:
    """train.py's parser for `gs_type`, in its declaration order, plus --seed."""
    p = ArgumentParser(description="Training script parameters")
    p.add_argument("--ip", type=str, default="127.0.0.1")
    p.add_argument("--port", type=int, default=6009)
    p.add_argument("--gs_type", type=str, default="gs_mesh")
    p.add_argument("--num_splats", nargs="+", type=int, default=[2])
    p.add_argument("--meshes", nargs="+", type=str, default=[])
    p.add_argument("--debug_from", type=int, default=-1)
    p.add_argument("--detect_anomaly", action="store_true", default=False)
    p.add_argument("--test_iterations", nargs="+", type=int, default=[7_000, 20_000, 30_000, 60_000, 90_000])
    p.add_argument("--save_iterations", nargs="+", type=int, default=[7_000, 20_000, 30_000, 60_000, 90_000])
    p.add_argument("--quiet", action="store_true")
    p.add_argument("--checkpoint_iterations", nargs="+", type=int, default=[])
    p.add_argument("--start_checkpoint", type=str, default=None)
    p.add_argument("--save_xyz", action="store_true")
    options.add_group(p, "Loading Parameters", options.MODEL_PARAMS)
    opt = options.OPT_PARAMS_MESH if gs_type in MESH_TYPES else options.OPT_PARAMS_FLAME if gs_type == "gs_flame" else options.OPT_PARAMS_FREE
    options.add_group(p, "Optimization Parameters", opt)
    options.add_group(p, "Pipeline Parameters", options.PIPELINE_PARAMS)
    p.add_argument("--seed", type=int, default=0, help="seeds the view shuffle and order, the initial model and the backgrounds")
    p.add_argument("--flame_model", type=str, default=dataset.DEFAULT_FLAME_MODEL,
                   help="gs_flame: FLAME's model file (FlameConfig's path, relative to the working directory)")
    p.add_argument("--viewer", action="store_true", default=False,
                   help="serve the SIBR remote viewer on --ip / --port while training (train.py's network_gui loop)")
    return p


def scene_kind(source_path: str):
    """"colmap" (sparse/), "blender" (transforms_train.json) or None, as Scene.__init__ tells them apart."""
    if os.path.exists(os.path.join(source_path, "sparse")):
        return "colmap"
    if os.path.exists(os.path.join(source_path, "transforms_train.json")):
        return "blender"
    return None


def parse_args(argv) -> Namespace:
    """train.py's argument handling: --gs_type first (it picks the optimisation group), then everything; --iterations is
    appended to --save_iterations.  Unsupported types and flags exit with an error that names them."""
    argv = list(argv)
    pre = ArgumentParser(add_help=False)
    pre.add_argument("--gs_type", type=str, default="gs_mesh")
    gs_type = pre.parse_known_args(argv)[0].gs_type
    parser = build_parser(gs_type if gs_type in GS_TYPES else "gs_mesh")
    if gs_type not in GS_TYPES:
        parser.error(f"--gs_type {gs_type} is not supported (supported: {', '.join(GS_TYPES)})")
    args = parser.parse_args(argv)
    for name, default in REFUSED:
        if getattr(args, name) != default:
            parser.error(f"--{name} is not supported by the native training frames")
    if args.data_device != "cuda":
        parser.error(f"--data_device {args.data_device} is not supported: images stay resident on the GPU (--data_device cuda)")
    if gs_type == "gs_multi_mesh":
        if not args.meshes:
            parser.error("--gs_type gs_multi_mesh needs --meshes (the names of sparse/0/<name>.obj) and one --num_splats per mesh")
        if len(args.num_splats) != len(args.meshes):
            parser.error(f"--gs_type gs_multi_mesh needs one --num_splats per --meshes entry; got {len(args.num_splats)} "
                         f"--num_splats for {len(args.meshes)} --meshes")
    if gs_type == "gs_flame" and not os.path.isfile(args.flame_model):
        parser.error(f"--gs_type gs_flame needs FLAME's model file: --flame_model {args.flame_model} does not exist")
    kind = scene_kind(args.source_path)
    need = {"gs_multi_mesh": "colmap", "gs_flame": "blender"}.get(gs_type)
    if need is not None and kind is not None and kind != need:
        parser.error(f"--gs_type {gs_type} trains on {'COLMAP' if need == 'colmap' else 'NeRF-synthetic'} scenes; "
                     f"--source_path {args.source_path} is a {'COLMAP' if kind == 'colmap' else 'NeRF-synthetic'} scene")
    args.save_iterations.append(args.iterations)
    return args


def set_default_model_path(args: Namespace) -> None:
    """prepare_output_and_logger's default -m: ./output/ + the first ten characters of $OAR_JOB_ID or a random UUID."""
    if not args.model_path:
        unique = os.getenv("OAR_JOB_ID") or str(uuid.uuid4())
        args.model_path = os.path.join("./output/", unique[0:10])


def iteration_events(it: int, args: Namespace) -> List[str]:
    """What train.py does at iteration `it` besides the frame, in its order: "report", "save", "densify", "reset", "step",
    "checkpoint"."""
    ev = []
    if it in args.test_iterations:
        ev.append("report")
    if it in args.save_iterations:
        ev.append("save")
    if args.gs_type in FREE_TYPES:
        _, densify, reset = FreeTrainer.schedule(SimpleNamespace(opt=free_params(args), white_background=args.white_background), it)
        ev += ["densify"] * densify + ["reset"] * reset
    if it < args.iterations:
        ev.append("step")
    if it in args.checkpoint_iterations:
        ev.append("checkpoint")
    return ev


def free_params(args: Namespace) -> FreeOptimizationParams:
    return FreeOptimizationParams(**{k: getattr(args, k) for k in FreeOptimizationParams.__dataclass_fields__ if k != "min_opacity"})


def flame_params(args: Namespace) -> FlameOptimizationParams:
    return FlameOptimizationParams(**{k: getattr(args, k) for k in FlameOptimizationParams.__dataclass_fields__})


class ViewOrder:
    """train.py's viewpoint_stack.pop(randint(0, len - 1)) on the Random stream that shuffled the scene (Scene.view_order),
    drawn one view at a time, with a state a checkpoint can hold."""

    def __init__(self, scene: dataset.Scene):
        self.rng = random.Random()
        self.rng.setstate(scene._rng_state)
        self.n = len(scene.train_cameras)
        self.stack = []

    def next(self) -> int:
        if not self.stack:
            self.stack = list(range(self.n))
        return self.stack.pop(self.rng.randint(0, len(self.stack) - 1))

    def state_dict(self) -> dict:
        version, internal, gauss = self.rng.getstate()
        return {"rng": [version, list(internal), gauss], "stack": list(self.stack)}

    def load_state_dict(self, state: dict) -> None:
        version, internal, gauss = state["rng"]
        self.rng.setstate((int(version), tuple(int(x) for x in internal), gauss))
        self.stack = [int(x) for x in state["stack"]]


def unshuffled_views(scene: dataset.Scene, seed: int):
    """(train, test) ViewInfos in file order: read_scene shuffled both lists with random.Random(seed), train first; the same
    draws on index lists give the permutations to undo."""
    rng = random.Random(seed)
    out = []
    for views in (scene.train_views, scene.test_views):
        perm = list(range(len(views)))
        rng.shuffle(perm)
        orig = [None] * len(views)
        for i, p in enumerate(perm):
            orig[p] = views[i]
        out.append(orig)
    return out[0], out[1]


def camera_json(idx: int, v: dataset.ViewInfo) -> dict:
    """camera_to_JSON (utils/camera_utils.py): the camera-to-world position and rotation, the file's size, focal lengths."""
    Rt = np.zeros((4, 4))
    Rt[:3, :3] = v.R.transpose()
    Rt[:3, 3] = v.T
    Rt[3, 3] = 1.0
    C2W = np.linalg.inv(Rt)
    return {"id": idx, "img_name": v.name, "width": v.width, "height": v.height, "position": C2W[:3, 3].tolist(),
            "rotation": [x.tolist() for x in C2W[:3, :3]], "fy": dataset.fov2focal(v.FovY, v.height),
            "fx": dataset.fov2focal(v.FovX, v.width)}


def write_cameras_json(path: str, scene: dataset.Scene, seed: int) -> None:
    train, test = unshuffled_views(scene, seed)
    with open(path, "w") as f:
        json.dump([camera_json(i, v) for i, v in enumerate(test + train)], f)


def write_input_ply(path: str, scene: dataset.Scene, source_path: str, gs_type: str, seed: int) -> None:
    """Scene.__init__'s input.ply: a byte copy of the dataset's own cloud file where it has one, else the cloud the
    reference's reader would have stored (the random NeRF-synthetic cloud, the converted COLMAP points, the gs_mesh cloud).
    gs_multi_mesh writes input_<i>.ply per mesh next to `path` instead; gs_flame's cloud needs the model (Training.prepare)."""
    if gs_type == "gs_multi_mesh":
        for i, cloud in enumerate(scene.mesh_clouds):
            io_ply.save_point_cloud(os.path.join(os.path.dirname(path), f"input_{i}.ply"), *cloud)
        return
    if gs_type == "gs_mesh":
        io_ply.save_point_cloud(path, *dataset.mesh_input_cloud(scene.mesh, seed))
        return
    for src in (os.path.join(source_path, "points3d.ply"), os.path.join(source_path, "sparse", "0", "points3D.ply")):
        if os.path.exists(src):
            shutil.copyfile(src, path)
            return
    points, colors, _ = scene.point_cloud
    io_ply.save_point_cloud(path, points, np.round(colors * 255.0))      # colors are bytes / 255: the round trip is exact


def open_summary_writer(model_path: str, log):
    """prepare_output_and_logger's writer: SummaryWriter(model_path) when torch.utils.tensorboard imports, else None after
    the reference's message through `log`."""
    try:
        from torch.utils.tensorboard import SummaryWriter
    except ImportError:
        log("Tensorboard not available: not logging progress")
        return None
    return SummaryWriter(model_path)


def add_scalars_event(writer, step: int, pairs) -> None:
    """What add_scalar writes for each (tag, value) of `pairs` (a simple_value summary), in ONE event at `step`: one record,
    one checksum pass and one file append in TensorBoard's writer instead of one per tag."""
    from tensorboard.compat.proto.summary_pb2 import Summary
    writer.file_writer.add_summary(Summary(value=[Summary.Value(tag=t, simple_value=float(v)) for t, v in pairs]), step)


def training_size(scene: dataset.Scene):
    """(largest width, largest height) of the training views: the one frame of a run is sized for it and runs every
    training view at the view's own size."""
    cams = scene.train_cameras
    return max(int(c.image_width) for c in cams), max(int(c.image_height) for c in cams)


def report_configs(scene: dataset.Scene):
    """training_report's validation configs: (name, cameras, resident images, image names) of the test views and of train
    views 5, 10, ..., 25 taken mod n."""
    n = len(scene.train_cameras)
    idx = [i % n for i in range(5, 30, 5)]
    names = scene.train_names
    return (("test", scene.test_cameras, scene.test_images, scene.test_names),
            ("train", [scene.train_cameras[i] for i in idx], [scene.train_images[i] for i in idx], [names[i] for i in idx]))


def _mesh_params(p: MeshGaussianParams, sh_degree: int) -> MeshGaussianParams:
    """create_from_pcd's features for max_sh_degree `sh_degree` (the loader builds degree 3: the rest is zero anyway)."""
    M = (int(sh_degree) + 1) ** 2
    rest = torch.zeros(p._features_dc.shape[0], M - 1, 3)
    return MeshGaussianParams(p.vertices, p.faces, p._alpha, p._scale, p._features_dc, rest, p._opacity)


class LiveFlame:
    """What FlameRenderer draws of a FlameCheckpoint, at a gs_flame training model's current parameters.  refresh() does on
    the device what save_flame_model does before it writes: the driver at the current FLAME tensors into model.vertices,
    then the expansion's activated weights and raw scaling / rotation rows at that pose.  A frame drawn after it is the
    frame cli.view draws from a checkpoint saved at that moment.  (The next FlameTrainer.step runs the driver again before
    it reads model.vertices.)"""

    def __init__(self, model):
        self.model, self.faces, self._vertices_enlargement = model, model.faces, model._vertices_enlargement
        self.vertices = self.alpha = self._scaling = self._rotation = None

    @property
    def active_sh_degree(self) -> int:
        return self.model.active_sh_degree

    @property
    def P(self) -> int:
        return self.model.P

    @property
    def _features(self) -> torch.Tensor:
        return self.model._features.detach()

    @property
    def _opacity(self) -> torch.Tensor:
        return self.model._opacity.detach()

    def refresh(self) -> None:
        m = self.model
        self.vertices = m.refresh_vertices()
        _, self._scaling, self._rotation, self.alpha, _ = expansion.expand(
            self.vertices, m.faces, m._alpha.detach(), m._scales.detach(), m.eps_s0, activated=False,
            alpha_activation=_lib.ALPHA_SOFTMAX)


class _Progress:
    def __init__(self, first: int, last: int, quiet: bool):
        self.bar = None
        if not quiet:
            try:
                from tqdm import tqdm
                self.bar = tqdm(range(first, last), desc="Training progress")
            except ImportError:
                pass

    def show(self, ema: float) -> None:
        if self.bar is not None:
            self.bar.set_postfix({"Loss": f"{ema:.{7}f}"})
            self.bar.update(10)

    def close(self) -> None:
        if self.bar is not None:
            self.bar.close()


class Training:
    """One train.py run: prepare() builds the output directory, the TensorBoard writer, scene, model and trainer (and
    restores --start_checkpoint); run() iterates.  Attributes the tests read: trainer, model, scene, order (ViewOrder), ema
    (per consumed iteration: (iteration, loss, moving average)), reports ((iteration, split, L1, PSNR)), events (per
    iteration: iteration_events), tb_writer (None without TensorBoard; closed once run() ends), viewer
    (network_gui.TrainingViewer under --viewer, else None; closed once run() ends)."""

    LOSS_SLOTS = 64

    def __init__(self, args: Namespace, device="cuda", scene: dataset.Scene = None):
        """scene: the load_scene result for these arguments, when the caller already has it (loaded on `device`)."""
        self.args, self.dev = args, torch.device(device)
        self.ema, self.reports, self.events = [], [], []
        self.first_iter = 0
        self.scene = scene
        self.tb_writer = None
        self.viewer = None

    def log(self, msg: str) -> None:
        if not self.args.quiet:
            print(msg)

    # ---- set-up (prepare_output_and_logger, Scene.__init__, training_setup, restore)
    def prepare(self) -> "Training":
        a = self.args
        set_default_model_path(a)
        if getattr(a, "viewer", False):         # network_gui.init comes before training() in train.py
            self.viewer = network_gui.TrainingViewer(a.ip, a.port, os.path.abspath(a.source_path).encode("utf-8"), log=self.log)
            ip, port = self.viewer.address
            self.log(f"Serving the remote viewer on {ip}:{port}")
        try:
            self.log(f"Output folder: {a.model_path}")
            os.makedirs(a.model_path, exist_ok=True)
            with open(os.path.join(a.model_path, "cfg_args"), "w") as f:
                f.write(options.cfg_args_string(a))
            self.tb_writer = open_summary_writer(a.model_path, self.log)
            self._setup()
            if self.viewer is not None:
                self.viewer.draw = self.viewer_frames()
            return self
        except BaseException:
            self.close_writer()
            self.close_viewer()
            raise

    def _setup(self) -> "Training":
        a = self.args
        if self.scene is None:
            self.scene = dataset.load_scene(a.source_path, a.gs_type, a.white_background, a.eval, a.resolution, a.images,
                                            a.num_splats if a.gs_type == "gs_multi_mesh" else a.num_splats[0], a.seed,
                                            device=self.dev, meshes=a.meshes, flame_model=a.flame_model)
        sc = self.scene
        if a.gs_type != "gs_flame":
            write_input_ply(os.path.join(a.model_path, "input.ply"), sc, a.source_path, a.gs_type, a.seed)
        write_cameras_json(os.path.join(a.model_path, "cameras.json"), sc, a.seed)
        max_size = training_size(sc)
        self.bg = torch.tensor([1.0, 1.0, 1.0] if a.white_background else [0.0, 0.0, 0.0], dtype=torch.float32, device=self.dev)
        self.bg_gen = torch.Generator(device=self.dev).manual_seed(a.seed) if a.random_background else None
        if a.gs_type in MESH_TYPES:
            if a.gs_type == "gs_mesh":
                self.model = MeshGaussianModel.from_params(_mesh_params(sc.mesh, a.sh_degree), self.dev, sh_degree=a.sh_degree,
                                                           active_sh_degree=0, packed_features=True)
            else:
                self.model = MultiMeshGaussianModel.from_mesh_params([_mesh_params(p, a.sh_degree) for p in sc.meshes], self.dev,
                                                                     sh_degree=a.sh_degree, active_sh_degree=0, packed_features=True)
            tr = self.trainer = MeshTrainer(self.model, self.bg, a.lambda_dssim, native=True, max_size=max_size)
            lrs = {"vertices": a.vertices_lr, "alpha": a.alpha_lr, "opacity": a.opacity_lr, "scaling": a.scaling_lr}
            for g in tr.opt.groups:         # OptimizationParamsMesh's learning rates (mesh_model_groups' f_rest = f_dc / 20)
                if g["name"] == "features":
                    g["lr0"], g["lr1"] = a.feature_lr, a.feature_lr / 20.0
                else:
                    g["lr"] = lrs[g["name"]]
        elif a.gs_type == "gs_flame":
            from ..flame import NativeFlame
            self.driver = NativeFlame.from_model_file(a.flame_model, device=self.dev)
            self.model = FlameGaussianModel.create(self.driver, sc.flame.faces, K=dataset.FLAME_K, sh_degree=a.sh_degree, seed=a.seed,
                                                   device=self.dev)
            io_ply.save_point_cloud(os.path.join(a.model_path, "input.ply"), *dataset.flame_input_cloud(self.model, sc.flame))
            self.trainer = FlameTrainer(self.model, self.bg, flame_params(a), max_size=max_size)
        else:
            points, colors, _ = sc.point_cloud
            self.model = FreeGaussianModel.from_point_cloud(points, colors, a.gs_type, a.sh_degree, self.dev)
            gen = torch.Generator(device=self.dev).manual_seed(a.seed)
            self.trainer = FreeTrainer(self.model, self.bg, sc.cameras_extent, free_params(a), white_background=a.white_background,
                                       generator=gen, max_size=max_size)
        self.order = ViewOrder(sc)
        if a.start_checkpoint:
            state, self.first_iter = torch.load(a.start_checkpoint, map_location="cpu", weights_only=True)
            self.load_state_dict(state)
        return self

    def state_dict(self) -> dict:
        return {"gs_type": self.args.gs_type, "trainer": self.trainer.state_dict(), "view_order": self.order.state_dict(),
                "bg_generator": self.bg_gen.get_state() if self.bg_gen is not None else None}

    def load_state_dict(self, state: dict) -> None:
        if state.get("gs_type") != self.args.gs_type:
            raise ValueError(f"--start_checkpoint holds a {state.get('gs_type')} run, not {self.args.gs_type}")
        self.trainer.load_state_dict(state["trainer"])
        self.order.load_state_dict(state["view_order"])
        if self.bg_gen is not None and state["bg_generator"] is not None:
            self.bg_gen.set_state(state["bg_generator"])

    def close_writer(self) -> None:
        if self.tb_writer is not None:
            self.tb_writer.close()

    def close_viewer(self) -> None:
        if self.viewer is not None:
            self.viewer.close()

    def viewer_frames(self):
        """cli.view's Frames on the trainer's live model, with the fixed background."""
        from ..render import FlameRenderer, NativeFreeRenderer, NativeRenderer
        from .view import Frames
        if self.args.gs_type in MESH_TYPES:
            return Frames(self.model, NativeRenderer, self.bg)
        if self.args.gs_type == "gs_flame":
            live = LiveFlame(self.model)
            return Frames(live, FlameRenderer, self.bg, refresh=live.refresh)
        return Frames(self.model, NativeFreeRenderer, self.bg)

    # ---- what happens at an iteration besides the frame
    def report(self, it: int) -> None:
        """training_report at a test iteration: the test views and train views 5, 10, ..., 25 (mod n) with the fixed
        background; mean L1 and mean per-channel PSNR, as the reference prints them.  With TensorBoard, also its images,
        split scalars, opacity histogram and point count."""
        w = self.tb_writer
        for name, cams, gts, names in report_configs(self.scene):
            if cams:
                r = self.trainer.evaluate(cams, gts)
                l1, psnr = float(r.mean[0]), float(r.mean[3])
                self.reports.append((it, name, l1, psnr))
                self.log(f"\n[ITER {it}] Evaluating {name}: L1 {l1} PSNR {psnr}")
                if w is not None:
                    self._report_images(it, name, cams[:5], gts[:5], names[:5])
                    w.add_scalar(f"{name}/loss_viewpoint - l1_loss", l1, it)
                    w.add_scalar(f"{name}/loss_viewpoint - psnr", psnr, it)
        if w is not None:
            opacity = self.model.get_opacity.detach().cpu()
            w.add_histogram("scene/opacity_histogram", opacity, it)
            w.add_scalar("total_points", int(opacity.shape[0]), it)

    def _report_images(self, it: int, name: str, cams, gts, names) -> None:
        """The renders (and, at the first listed test iteration, the ground truth) of up to five views as the float tensors
        the reference hands add_images: TensorBoard's own (x * 255) truncation then gives the reference's PNGs.  The renders
        come from the renderers evaluate() just built for these views (one per image size, each image at its view's size),
        so none can overflow its capacity."""
        w, r = self.tb_writer, self.trainer.renderer
        for cam, gt, image_name in zip(cams, gts, names):
            image = torch.clamp(r.render(cam, self.trainer.bg)[0], 0.0, 1.0)
            w.add_images(f"{name}_view_{image_name}/render", image[None].cpu(), global_step=it)
            if it == self.args.test_iterations[0]:
                gt_image = torch.clamp(gt.cpu().permute(2, 0, 1).float() / 255.0, 0.0, 1.0)
                w.add_images(f"{name}_view_{image_name}/ground_truth", gt_image[None], global_step=it)

    def log_iteration(self, it: int, loss: float, l1: float, ms: float) -> None:
        """training_report's per-iteration scalars, in one event."""
        add_scalars_event(self.tb_writer, it, (("train_loss_patches/l1_loss", l1), ("train_loss_patches/total_loss", loss),
                                               ("iter_time", ms)))

    def save(self, it: int) -> None:
        self.log(f"\n[ITER {it}] Saving Gaussians")
        path = os.path.join(self.args.model_path, "point_cloud", f"iteration_{it}", "point_cloud.ply")
        if self.args.gs_type == "gs_mesh":
            io_ply.save_mesh_model(path, self.model)
        elif self.args.gs_type == "gs_multi_mesh":
            io_ply.save_multi_mesh_model(path, self.model)
        elif self.args.gs_type == "gs_flame":
            io_ply.save_flame_model(path, self.model, point_cloud=self.driver.to_point_cloud())
        else:
            self.model.save(path)

    def checkpoint(self, it: int) -> None:
        self.log(f"\n[ITER {it}] Saving Checkpoint")
        torch.save((self.state_dict(), it), os.path.join(self.args.model_path, f"chkpnt{it}.pth"))

    # ---- the loss, L1 and frame time, read without synchronising
    def _slot_events(self, i: int):
        """The events slot i's values wait for: the loss copy's, and with TensorBoard the frame's end."""
        return (self._loss_ready[i],) + ((self._timing[i][1],) if self._timing else ())

    def _consume(self, block: bool = False) -> None:
        while self._pending and (block or all(e.query() for e in self._slot_events(self._pending[0][1]))):
            it, i = self._pending.popleft()
            for e in self._slot_events(i):
                e.synchronize()
            loss = float(self._slots_np[i, 0])
            self._ema = 0.4 * loss + 0.6 * self._ema
            self.ema.append((it, loss, self._ema))
            if self._timing:
                self.log_iteration(it, loss, float(self._slots_np[i, 1]), self._timing[i][0].elapsed_time(self._timing[i][1]))
            if it % 10 == 0:
                self._progress.show(self._ema)

    def run(self) -> "Training":
        try:
            self._loop()
        finally:
            self.close_writer()
            self.close_viewer()
        self.log("\nTraining complete.")
        return self

    def _loop(self) -> None:
        a, sc, dev = self.args, self.scene, self.dev
        slots = torch.zeros(self.LOSS_SLOTS, 2, dtype=torch.float32).pin_memory()     # per slot: loss, L1
        self._slots_np = slots.numpy()
        self._loss_ready = [torch.cuda.Event() for _ in range(self.LOSS_SLOTS)]
        # train.py's iter_start / iter_end per slot; read only once the end event has completed
        self._timing = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                        for _ in range(self.LOSS_SLOTS)] if self.tb_writer is not None else None
        self._pending, self._ema = collections.deque(), 0.0
        self._progress = _Progress(self.first_iter, a.iterations, a.quiet)
        mesh = a.gs_type in MESH_TYPES
        stream = torch.cuda.current_stream(dev)
        for it in range(self.first_iter + 1, a.iterations + 1):
            if self.viewer is not None:
                with torch.no_grad():
                    self.viewer.poll(it, a.iterations)
            ev = iteration_events(it, a)
            self.events.append((it, ev))
            if mesh and it % 1000 == 0:
                self.model.oneupSHdegree()
            v = self.order.next()
            bg = torch.rand(3, device=dev, generator=self.bg_gen) if self.bg_gen is not None else None
            hooks = [f for name, f in (("report", self.report), ("save", self.save)) if name in ev]
            # the last iteration takes no Adam step: never let the frame fuse one in
            before = (lambda: [f(it) for f in hooks]) if hooks or "step" not in ev else None
            if len(self._pending) == self.LOSS_SLOTS:
                for e in self._slot_events(self._pending[0][1]):
                    e.synchronize()
                self._consume()
            slot = it % self.LOSS_SLOTS
            start, end = self._timing[slot] if self._timing else (None, None)
            if start is not None:
                start.record(stream)
            if mesh:
                self.trainer.optimizer_step = "step" in ev
                self.trainer.step(sc.train_cameras[v], sc.train_images[v], loss_host=slots[slot], loss_ready=self._loss_ready[slot],
                                  bg=bg, before_update=before, frame_end=end)
            else:
                self.trainer.step(sc.train_cameras[v], sc.train_images[v], bg=bg, before_update=before, frame_end=end)
                slots[slot].copy_(self.trainer.loss_vector[:2], non_blocking=True)
                self._loss_ready[slot].record(stream)
            self._pending.append((it, slot))
            self._consume()
            if "checkpoint" in ev:
                self.checkpoint(it)
        self._consume(block=True)
        self._progress.close()


def main(argv=None) -> Training:
    args = parse_args(sys.argv[1:] if argv is None else argv)
    if not torch.cuda.is_available():
        raise RuntimeError("gms_b200.cli.train needs a CUDA device")
    try:
        run = Training(args).prepare()
    except network_gui.AddressError as e:
        sys.exit(f"gms_b200.cli.train: error: {e}")
    return run.run()


if __name__ == "__main__":
    main()

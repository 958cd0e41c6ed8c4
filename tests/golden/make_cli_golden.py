"""Generate cli.npz: what the reference's train.py writes into its output directory before training, from its own code.

    python tests/golden/make_cli_golden.py        (needs /root/reference and PIL)

Importing make_dataset_golden installs its stubs (plyfile in memory, trimesh, CUDA allocations on the CPU, empty
simple-knn / smplx / rasterizer modules); here plyfile's write also leaves a file on disk, because Scene.__init__ copies
the cloud file byte for byte into input.ply.  Then:
- cfg_args: for each command line of CFG_ARGV, train.py's parser (its own arguments, then ModelParams, the optimisation
  group of --gs_type and PipelineParams, the reference's classes), parse_known_args / parse_args as its __main__ does, and
  prepare_output_and_logger(lp.extract(args)).  The source and output paths are stored as <SRC> and <OUT>; OAR_JOB_ID fixes
  the name of the default output directory.
- cameras.json and input.ply: Scene.__init__ with a stub model (create_from_pcd does nothing) on every case of
  dataset_cases.CASES, after safe_state's seeds.  Stored: cameras.json's text, and for input.ply the vertex rows storePly
  built (every field's SHA-256, its first 256 rows, the row count)."""
import hashlib
import os
import random
import shutil
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_dataset_golden as mdg  # noqa: E402  (installs the stubs)
import dataset_cases  # noqa: E402

from argparse import ArgumentParser  # noqa: E402

_write = mdg._PlyData.write


def _write_to_disk(self, path):
    _write(self, path)
    with open(path, "wb") as f:          # Scene.__init__ copies the file; its content is read back from mdg._PLY_FILES
        f.write(b"placeholder")


mdg._PlyData.write = _write_to_disk

from arguments import ModelParams, PipelineParams  # noqa: E402
from games import optimizationParamTypeCallbacks  # noqa: E402
from scene import Scene  # noqa: E402
import train as ref_train  # noqa: E402

ROWS = 256
JOB_ID = "0123456789abcdef"
CFG_ARGV = [
    ["-s", "<SRC>", "-m", "<OUT>"],
    ["-s", "<SRC>", "-m", "<OUT>", "--gs_type", "gs_flat", "-w", "--eval", "-r", "2", "-i", "imgs", "--sh_degree", "2",
     "--iterations", "50", "--num_splats", "3", "4"],
    ["--gs_type", "gs", "--source_path", "<SRC>", "--resolution", "4", "--white_background", "--test_iterations", "-1"],
    ["-s", "<SRC>", "-m", "<OUT>", "--gs_type", "gs_mesh", "--meshes", "a.obj", "b.obj", "--data_device", "cuda"],
]


def reference_cfg_args(argv, src, out) -> str:
    """train.py's __main__ up to training(), then prepare_output_and_logger."""
    argv = [src if a == "<SRC>" else out if a == "<OUT>" else a for a in argv]
    parser = ArgumentParser(description="Training script parameters")
    parser.add_argument('--ip', type=str, default="127.0.0.1")
    parser.add_argument('--port', type=int, default=6009)
    parser.add_argument('--gs_type', type=str, default="gs_mesh")
    parser.add_argument("--num_splats", nargs="+", type=int, default=[2])
    parser.add_argument("--meshes", nargs="+", type=str, default=[])
    parser.add_argument('--debug_from', type=int, default=-1)
    parser.add_argument('--detect_anomaly', action='store_true', default=False)
    parser.add_argument("--test_iterations", nargs="+", type=int, default=[7_000, 20_000, 30_000, 60_000, 90_000])
    parser.add_argument("--save_iterations", nargs="+", type=int, default=[7_000, 20_000, 30_000, 60_000, 90_000])
    parser.add_argument("--quiet", action="store_true")
    parser.add_argument("--checkpoint_iterations", nargs="+", type=int, default=[])
    parser.add_argument("--start_checkpoint", type=str, default=None)
    parser.add_argument("--save_xyz", action='store_true')
    lp = ModelParams(parser)
    args, _ = parser.parse_known_args(argv)
    lp.num_splats, lp.meshes, lp.gs_type = args.num_splats, args.meshes, args.gs_type
    optimizationParamTypeCallbacks[args.gs_type](parser)
    PipelineParams(parser)
    args = parser.parse_args(argv)
    dataset = lp.extract(args)
    cwd = os.getcwd()
    os.chdir(out)                        # the default ./output/<id> lands under `out`
    try:
        ref_train.prepare_output_and_logger(dataset)
        with open(os.path.join(dataset.model_path, "cfg_args")) as f:
            text = f.read()
    finally:
        os.chdir(cwd)
    return text.replace(os.path.abspath(src), "<SRC>").replace(out, "<OUT>")


class _StubModel:
    def create_from_pcd(self, *a, **k):
        pass


def run_case(src: str, out: str, kw: dict, res: dict, key: str) -> None:
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    mdg._PLY_FILES.clear()
    os.makedirs(out, exist_ok=True)
    args = types.SimpleNamespace(model_path=out, source_path=src, gs_type=kw["gs_type"], images="images", eval=kw["eval"],
                                 white_background=kw.get("white_background", False), num_splats=[kw.get("num_splats", 2)],
                                 resolution=kw["resolution"], data_device="cpu", meshes=[])
    Scene(args, _StubModel())
    with open(os.path.join(out, "cameras.json")) as f:
        res[f"{key}/cameras_json"] = np.array(f.read())
    ply = next(p for p in mdg._PLY_FILES if os.path.dirname(p) in (src, os.path.join(src, "sparse/0")))
    el = mdg._PLY_FILES[ply]
    res[f"{key}/ply_n"] = np.array(el.shape[0], np.int64)
    for name in el.dtype.names:
        a = np.ascontiguousarray(el[name])
        res[f"{key}/ply_{name}"] = a[:ROWS].copy()
        res[f"{key}/ply_{name}_sha256"] = np.array(hashlib.sha256(a.tobytes()).hexdigest())


def main():
    res = {}
    os.environ["OAR_JOB_ID"] = JOB_ID
    with tempfile.TemporaryDirectory() as d:
        dirs = dataset_cases.write_all(os.path.join(d, "src"))
        for i, argv in enumerate(CFG_ARGV):
            out = os.path.join(d, "cfg", str(i))
            os.makedirs(out)
            res[f"cfg/{i}/argv"] = np.array("\x1f".join(argv))
            res[f"cfg/{i}/text"] = np.array(reference_cfg_args(argv, dirs["blender_a"], out))
        for key, (ds, kw) in dataset_cases.CASES.items():
            work = os.path.join(d, "work", key)
            shutil.copytree(dirs[ds], work)
            run_case(work, os.path.join(d, "out", key), kw, res, key)
    np.savez_compressed(os.path.join(HERE, "cli.npz"), **res)
    print(f"{len(res)} arrays, {os.path.getsize(os.path.join(HERE, 'cli.npz'))} bytes")


if __name__ == "__main__":
    main()

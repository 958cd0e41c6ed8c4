"""cli.train's gs_multi_mesh and gs_flame end to end on the GPU: the FLAME reader's mesh and input.ply against the
reference's (tests/golden/train_mesh_types.npz); on small generated scenes, agreement with the bare MeshTrainer /
FlameTrainer loop, resume from --start_checkpoint, no host synchronisation in the loop, and the saved iteration through
cli.render and cli.metrics."""
import json
import os

import numpy as np
import pytest
import torch

import dataset_cases
import mesh_types_cases as cases
from gms_b200 import dataset, io_image, io_ply
from gms_b200.cli import metrics as cli_metrics
from gms_b200.cli import render as cli_render
from gms_b200.cli import train as cli_train
from gms_b200.flame import NativeFlame
from gms_b200.model import FlameGaussianModel, MultiMeshGaussianModel
from gms_b200.render import NativeRenderer
from gms_b200.trainer import FlameTrainer, MeshTrainer
from test_gpu_dataset import _write_rendered_blender

pytestmark = pytest.mark.gpu

N = 30
COMMON = ["--eval", "--iterations", str(N), "--test_iterations", "10", "--save_iterations", "10", "20",
          "--checkpoint_iterations", "15", "--quiet"]
MULTI_ARGV = ["--gs_type", "gs_multi_mesh", "--meshes", "a", "b", "--num_splats", "2", "3"] + COMMON
FLAME_ARGV = ["--gs_type", "gs_flame", "--flame_model", cases.FLAME_MODEL] + COMMON
HOOKS = {10, 20, 30}            # report / save / last iterations: the CLI passes a before_update there
SYNC_OK = {1, 10, 20, 30}
MULTI_NAMES = ("vertices", "_alpha", "_scale", "_features", "_opacity")
FLAME_NAMES = FlameGaussianModel.FLAME_NAMES + ("_alpha", "_scales", "_features", "_opacity")


def _params(model, names):
    return {n: getattr(model, n).detach().clone() for n in names}


def _within_spread(got, ref, other, what):
    """max |got - ref| <= 10 x max |other - ref| + 1e-7 per tensor, `other` a second run of the bare loop (the frames sum
    with float atomics, so two runs of one loop differ)."""
    for n in ref:
        assert got[n].shape == ref[n].shape, f"{what}: {n}"
        d_got, d_other = float((got[n] - ref[n]).abs().max()), float((other[n] - ref[n]).abs().max())
        print(f"[{what}] {n}: max |got - ref| {d_got:.3e}, run-to-run {d_other:.3e}")
        assert d_got <= 10 * d_other + 1e-7, f"{what}: {n} {d_got:.3e} against the run-to-run {d_other:.3e}"


def _write_colmap_from_blender(blender_root, root):
    """The same views as a COLMAP scene: PINHOLE cameras, RGB PNGs, world->camera rotations as quaternions, and the two
    meshes a.obj / b.obj under sparse/0/."""
    import struct
    from scipy.spatial.transform import Rotation
    sparse = os.path.join(root, "sparse", "0")
    os.makedirs(sparse)
    os.makedirs(os.path.join(root, "images"))
    views = []
    for split in ("train", "test"):
        views += dataset.read_transforms(blender_root, f"transforms_{split}.json")
    W, H = dataset.image_size(views[0].path)
    f = dataset.fov2focal(views[0].FovX, W)
    with open(os.path.join(sparse, "cameras.bin"), "wb") as fh:
        fh.write(struct.pack("<Q", 1) + struct.pack("<iiQQ", 1, 1, W, H) + struct.pack("<dddd", f, f, W / 2, H / 2))
    with open(os.path.join(sparse, "images.bin"), "wb") as fh:
        fh.write(struct.pack("<Q", len(views)))
        for k, v in enumerate(views):
            name = f"view_{k:02d}.png"
            rgb = dataset.decode_image(v.path, "RGBA")[:, :, :3]
            dataset_cases.write_png(os.path.join(root, "images", name), np.ascontiguousarray(rgb))
            x, y, z, w = Rotation.from_matrix(v.R.T).as_quat()
            fh.write(struct.pack("<idddddddi", k + 1, w, x, y, z, *v.T, 1) + name.encode() + b"\x00" + struct.pack("<Q", 0))
    with open(os.path.join(sparse, "points3D.bin"), "wb") as fh:
        fh.write(struct.pack("<Q", 0))
    from gms_b200 import scenes
    v, fc = scenes.icosphere(1, 0.45)
    cases.write_obj(os.path.join(sparse, "a.obj"), v, fc)
    v, fc = scenes.icosphere(0, 0.25)
    cases.write_obj(os.path.join(sparse, "b.obj"), v + np.array([0.3, 0.1, -0.2]), fc)
    return root


@pytest.fixture(scope="module")
def roots(tmp_path_factory):
    base = tmp_path_factory.mktemp("mesh_types")
    blender = str(base / "blender")
    _write_rendered_blender(blender)
    return {"gs_flame": blender, "gs_multi_mesh": _write_colmap_from_blender(blender, str(base / "colmap"))}


def _argv(gs_type):
    return MULTI_ARGV if gs_type == "gs_multi_mesh" else FLAME_ARGV


def _names(gs_type):
    return MULTI_NAMES if gs_type == "gs_multi_mesh" else FLAME_NAMES


def _cli(root, out, argv, cls=cli_train.Training):
    return cls(cli_train.parse_args(["-s", root, "-m", out] + argv)).prepare().run()


def _bare(gs_type, root):
    """The bare loop: load_scene's view order, the trainer built from the library API, a before_update where the CLI
    passes one.  -> the final parameters."""
    bg = torch.zeros(3, device="cuda")
    if gs_type == "gs_multi_mesh":
        sc = dataset.load_scene(root, gs_type, eval=True, num_splats=[2, 3], meshes=["a", "b"])
        m = MultiMeshGaussianModel.from_mesh_params(sc.meshes, "cuda", active_sh_degree=0, packed_features=True)
        tr = MeshTrainer(m, bg, native=True)
    else:
        sc = dataset.load_scene(root, gs_type, eval=True, flame_model=cases.FLAME_MODEL)
        m = FlameGaussianModel.create(NativeFlame.from_model_file(cases.FLAME_MODEL), sc.flame.faces, K=dataset.FLAME_K)
        tr = FlameTrainer(m, bg, cli_train.flame_params(cli_train.parse_args(["-s", root] + FLAME_ARGV)))
    for it, v in enumerate(sc.view_order(N), 1):
        if gs_type == "gs_multi_mesh":
            tr.optimizer_step = it < N
        tr.step(sc.train_cameras[v], sc.train_images[v], before_update=(lambda: None) if it in HOOKS else None)
    return _params(m, _names(gs_type))


@pytest.fixture(scope="module")
def runs(roots, tmp_path_factory):
    out = {}
    for t in ("gs_multi_mesh", "gs_flame"):
        d = str(tmp_path_factory.mktemp(t))
        out[t] = (d, _cli(roots[t], d, _argv(t)), _bare(t, roots[t]), _bare(t, roots[t]))
    return out


# ------------------------------------------------------------------------------------------------ the FLAME reader

def test_flame_reader_mesh_and_input_ply_match_reference(golden_dir, tmp_path):
    g = np.load(os.path.join(golden_dir, "train_mesh_types.npz"))
    src = cases.write_flame(str(tmp_path / "src"))
    run = cli_train.Training(cli_train.parse_args(["-s", src, "-m", str(tmp_path / "out"), "--gs_type", "gs_flame",
                                                   "--flame_model", cases.FLAME_MODEL, "--quiet"])).prepare()
    ref_v = torch.from_numpy(g["flame/vertices"]).double()
    d = float((run.model.vertices.double().cpu() - ref_v).abs().max())
    print(f"[flame reader] vertices: max |native - reference| {d:.3e}")
    assert d <= 1e-5 * float(ref_v.abs().max())
    assert torch.equal(run.model._alpha.cpu(), torch.from_numpy(g["flame/alpha"]))
    el, _ = io_ply.read_ply_vertices(str(tmp_path / "out" / "input.ply"))
    for c in ("red", "green", "blue"):
        assert np.array_equal(el[c], g[f"flame/ply_{c}"]), c
    xyz = np.stack([el[c] for c in "xyz"], 1).astype(np.float64)
    ref = np.stack([g[f"flame/ply_{c}"] for c in "xyz"], 1).astype(np.float64)
    assert xyz.shape == ref.shape and np.abs(xyz - ref).max() <= 1e-5 * np.abs(ref).max()
    assert not os.path.exists(os.path.join(src, "points3d.ply"))


# ------------------------------------------------------------------------------------------------ training

@pytest.mark.parametrize("gs_type", ["gs_multi_mesh", "gs_flame"])
def test_trains_end_to_end_and_agrees_with_the_bare_loop(runs, gs_type):
    out, run, a, b = runs[gs_type]
    inputs = ["input_0.ply", "input_1.ply"] if gs_type == "gs_multi_mesh" else ["input.ply"]
    for f in ["cfg_args", "cameras.json", "chkpnt15.pth"] + inputs:
        assert os.path.exists(os.path.join(out, f)), f
    assert (gs_type == "gs_multi_mesh") != os.path.exists(os.path.join(out, "input.ply"))
    side = "model_params.pt" if gs_type == "gs_multi_mesh" else "flame_params.pt"
    for it in (10, 20, 30):
        for f in ("point_cloud.ply", side):
            assert os.path.exists(os.path.join(out, "point_cloud", f"iteration_{it}", f)), (it, f)
    assert [e for _, e in run.events] == [cli_train.iteration_events(it, run.args) for it in range(1, N + 1)]
    assert [it for it, _, _ in run.ema] == list(range(1, N + 1)) and all(np.isfinite(l) for _, l, _ in run.ema)
    assert [(it, s) for it, s, _, _ in run.reports] == [(10, "test"), (10, "train")]
    _within_spread(_params(run.model, _names(gs_type)), a, b, f"{gs_type} CLI vs bare loop")


@pytest.mark.parametrize("gs_type", ["gs_multi_mesh", "gs_flame"])
def test_resume_restores_state_bit_for_bit(roots, runs, gs_type, tmp_path):
    out, _, a, b = runs[gs_type]
    ck = os.path.join(out, "chkpnt15.pth")
    state, k = torch.load(ck, map_location="cpu", weights_only=True)
    assert k == 15
    run = cli_train.Training(cli_train.parse_args(["-s", roots[gs_type], "-m", str(tmp_path), "--start_checkpoint", ck]
                                                  + _argv(gs_type))).prepare()
    now = run.trainer.state_dict()
    for key in ("p", "m", "v"):
        assert torch.equal(now["adam"][key].cpu(), state["trainer"]["adam"][key]), key
    assert now["adam"]["steps"] == state["trainer"]["adam"]["steps"]
    assert now["active_sh_degree"] == state["trainer"]["active_sh_degree"]
    if gs_type == "gs_flame":
        assert now["iteration"] == state["trainer"]["iteration"] == 15
    assert run.first_iter == 15 and run.order.state_dict() == state["view_order"]
    run.run()
    assert [it for it, _ in run.events] == list(range(16, N + 1))
    _within_spread(_params(run.model, _names(gs_type)), a, b, f"{gs_type} resumed CLI vs bare loop")


@pytest.mark.parametrize("gs_type", ["gs_multi_mesh", "gs_flame"])
def test_loop_never_synchronises(roots, gs_type, tmp_path):
    """Every iteration but the first, the report iterations and the save iterations runs under sync debug mode "error"."""

    class Strict(cli_train.Training):
        def _relaxed(self, fn, *a, **k):
            torch.cuda.set_sync_debug_mode(0)
            try:
                return fn(*a, **k)
            finally:
                torch.cuda.set_sync_debug_mode("error")

        def report(self, it):
            assert it in SYNC_OK
            self._relaxed(super().report, it)

        def save(self, it):
            assert it in SYNC_OK
            self._relaxed(super().save, it)

        def checkpoint(self, it):
            self._relaxed(super().checkpoint, it)

        def _consume(self, block=False):
            return self._relaxed(super()._consume, block) if block else super()._consume(block)

    run = Strict(cli_train.parse_args(["-s", roots[gs_type], "-m", str(tmp_path)] + _argv(gs_type))).prepare()
    step = run.trainer.step

    def first_relaxed(*a, **k):
        return run._relaxed(step, *a, **k) if run._first else step(*a, **k)

    run._first = True
    run.trainer.step = lambda *a, **k: (first_relaxed(*a, **k), setattr(run, "_first", False))[0]
    torch.cuda.set_sync_debug_mode("error")
    try:
        run.run()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(run.ema) == N


# ------------------------------------------------------------------------------------------------ render and metrics

@pytest.mark.parametrize("gs_type", ["gs_multi_mesh", "gs_flame"])
def test_saved_iteration_renders_and_scores(roots, runs, gs_type):
    out, run, _, _ = runs[gs_type]
    cli_render.main(["-m", out, "--gs_type", gs_type, "--skip_train", "--quiet"])
    sc = dataset.load_scene(roots[gs_type], "gs_flat", eval=True, shuffle=False)
    bg = torch.zeros(3, device="cuda")
    if gs_type == "gs_flame":
        run.model.refresh_vertices()          # the pose of the saved parameters
    r = NativeRenderer(run.model, sc.test_cameras[0].image_width, sc.test_cameras[0].image_height)
    worst = 0.0
    for i, c in enumerate(sc.test_cameras):
        want = r.render(c, bg)[0]
        with open(os.path.join(out, "test", f"ours_{N}", f"renders_{gs_type}", f"{i:05d}.png"), "rb") as f:
            got = io_image.decode_png(f.read())
        if gs_type == "gs_multi_mesh":
            assert np.array_equal(got, io_image.quantize(want).cpu().numpy().reshape(got.shape)), f"view {i}"
        else:
            d = float(np.abs(got.astype(np.float64) / 255.0 - want.permute(1, 2, 0).double().cpu().numpy()).max())
            worst = max(worst, d)
            assert d <= 0.5 / 255 + 1e-3, f"view {i}: {d:.3e}"
    print(f"[{gs_type}] cli.render against the trained model: worst {worst:.3e}")
    res = cli_metrics.main(["-m", out, "--gs_type", gs_type, "--quiet"])[out]
    with open(os.path.join(out, f"results_{gs_type}.json")) as f:
        assert json.load(f) == res["results"]
    for key in ("SSIM", "PSNR"):
        assert np.isfinite(res["results"][f"ours_{N}"][key])
        assert len(res["per_view"][f"ours_{N}"][key]) == len(sc.test_cameras)

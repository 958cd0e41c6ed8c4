"""cli.train's gs_multi_mesh and gs_flame host side against the reference's own readers and train.py
(tests/golden/train_mesh_types.npz, written by make_train_mesh_types_golden.py): the COLMAP-mesh and FLAME scene readers'
cameras and random initialisation, the input clouds, cfg_args, the per-iteration schedule, the optimisation flags and the
refusals."""
import os

import numpy as np
import pytest

import mesh_types_cases as cases
from gms_b200 import dataset, io_ply
from gms_b200.cli import options
from gms_b200.cli import train as cli_train
from test_cli_host import restated_train_py


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "train_mesh_types.npz"))


@pytest.fixture(scope="module")
def scenes_dir(tmp_path_factory):
    root = tmp_path_factory.mktemp("mesh_types_src")
    return {"multi": cases.write_multi(str(root / "multi")), "flame": cases.write_flame(str(root / "flame"))}


def _read(key, src):
    if key == "multi":
        return dataset.read_scene(src, "gs_multi_mesh", eval=cases.MULTI_EVAL, num_splats=cases.NUM_SPLATS, meshes=cases.MESHES)
    return dataset.read_scene(src, "gs_flame", eval=cases.FLAME_EVAL, flame_model=cases.FLAME_MODEL)


@pytest.mark.parametrize("key", ["multi", "flame"])
def test_cameras_names_and_extent_equal_reference(golden, scenes_dir, key):
    sc = _read(key, scenes_dir[key])
    assert sc.cameras_extent == float(golden[f"{key}/extent"])
    for split, views, cams in (("train", sc.train_views, sc.train_cameras), ("test", sc.test_views, sc.test_cameras)):
        assert [v.name for v in views] == list(golden[f"{key}/{split}/names"]), f"{key} {split} names"
        assert np.array_equal(np.array([v.R for v in views]).reshape(-1, 3, 3), golden[f"{key}/{split}/R"])
        assert np.array_equal(np.array([v.T for v in views]).reshape(-1, 3), golden[f"{key}/{split}/T"])
        assert np.array_equal(np.array([[v.FovX, v.FovY] for v in views]).reshape(-1, 2), golden[f"{key}/{split}/fov"])
        assert np.array_equal(np.array([[c.image_width, c.image_height] for c in cams]).reshape(-1, 2), golden[f"{key}/{split}/size"])
    if key == "flame":
        assert not sc.test_views and len(sc.train_views) == 5        # no --eval: the test views join training


def test_colmap_mesh_reader_equals_reference(golden, scenes_dir, tmp_path):
    sc = _read("multi", scenes_dir["multi"])
    assert len(sc.meshes) == len(sc.mesh_clouds) == 2
    for i, (p, K) in enumerate(zip(sc.meshes, cases.NUM_SPLATS)):
        ref_alpha, ref_colors = golden[f"multi/mesh{i}/alpha"], golden[f"multi/mesh{i}/colors"]
        assert p._alpha.shape[1] == K and np.array_equal(p._alpha.numpy(), ref_alpha), f"mesh {i}: _alpha"
        assert np.array_equal(sc.mesh_clouds[i][1], ref_colors * 255), f"mesh {i}: colours"
        # create_from_pcd: DC = RGB2SH(float32 colours), rest 0, scale 1, opacity inverse_sigmoid(0.1)
        fdc = (np.float32(ref_colors) - np.float32(0.5)) / np.float32(dataset.SH_C0)
        assert np.array_equal(p._features_dc.numpy().reshape(-1, 3), fdc.astype(np.float32))
        assert not p._features_rest.any() and (p._scale == 1).all()
        assert np.allclose(p._opacity.numpy(), np.log(0.1 / 0.9), rtol=0, atol=1e-7)
    # Scene.__init__'s input_<i>.ply: the reference's points3d_<i>.ply byte for byte, and no input.ply
    cli_train.write_input_ply(str(tmp_path / "input.ply"), sc, scenes_dir["multi"], "gs_multi_mesh", seed=0)
    assert sorted(os.listdir(tmp_path)) == ["input_0.ply", "input_1.ply"]
    for i in range(2):
        assert (tmp_path / f"input_{i}.ply").read_bytes() == golden[f"multi/mesh{i}/ply"].tobytes(), f"input_{i}.ply"
    # nothing was written into the source directory
    assert not [f for f in os.listdir(scenes_dir["multi"]) if f.endswith(".ply")]


def test_flame_reader_draws_equal_reference(golden, scenes_dir):
    sc = _read("flame", scenes_dir["flame"])
    f = sc.flame
    assert f.model_path == cases.FLAME_MODEL
    assert np.array_equal(f.faces.numpy(), golden["flame/faces"])
    assert f.alpha.shape[1] == dataset.FLAME_K and np.array_equal(f.alpha.numpy(), golden["flame/alpha"])
    assert np.array_equal(f.colors, golden["flame/colors"])
    # points3d.ply's colour bytes (storePly's u1 cast); its coordinates need the FLAME mesh, checked on the GPU
    assert np.array_equal(np.stack([golden[f"flame/ply_{c}"] for c in ("red", "green", "blue")], 1), (f.colors * 255).astype(np.uint8))
    assert not [x for x in os.listdir(scenes_dir["flame"]) if x.endswith(".ply")]


@pytest.mark.parametrize("key", ["multi", "flame"])
def test_cfg_args_equal_reference(golden, scenes_dir, tmp_path, monkeypatch, key):
    monkeypatch.setenv("OAR_JOB_ID", "0123456789abcdef")
    monkeypatch.chdir(tmp_path)
    src, out = scenes_dir[key], str(tmp_path / "out")
    argv = [src if a == "<SRC>" else out if a == "<OUT>" else a for a in str(golden[f"cfg/{key}/argv"]).split("\x1f")]
    args = cli_train.parse_args(argv + (["--flame_model", cases.FLAME_MODEL] if key == "flame" else []))
    cli_train.set_default_model_path(args)
    text = options.cfg_args_string(args).replace(os.path.abspath(src), "<SRC>").replace(out, "<OUT>")
    assert text == str(golden[f"cfg/{key}/text"])


SCHEDULES = [
    ["--gs_type", "gs_multi_mesh", "--meshes", "a", "b", "--num_splats", "2", "3", "--iterations", "30", "--test_iterations",
     "10", "30", "--save_iterations", "20", "--checkpoint_iterations", "15", "30"],
    ["--gs_type", "gs_flame", "--flame_model", cases.FLAME_MODEL, "--iterations", "25", "--test_iterations", "-1",
     "--save_iterations", "5", "--checkpoint_iterations", "24"],
    ["--gs_type", "gs_flame", "--flame_model", cases.FLAME_MODEL, "--iterations", "1"],
]


@pytest.mark.parametrize("argv", SCHEDULES, ids=[f"s{i}" for i in range(len(SCHEDULES))])
def test_schedule_matches_train_py(argv):
    args = cli_train.parse_args(["-s", "scene"] + argv)
    got = [cli_train.iteration_events(it, args) for it in range(1, args.iterations + 1)]
    assert got == restated_train_py(args)


def test_flame_optimisation_flags_are_the_reference_group():
    # OptimizationParamsFlame (arguments_games/__init__.py:32-49), in declaration order
    ref = [("iterations", 30_000), ("alpha_lr", 0.001), ("feature_lr", 0.0025), ("opacity_lr", 0.05), ("scaling_lr", 0.005),
           ("rotation_lr", 0.001), ("flame_shape_lr", 0.01), ("flame_exp_lr", 0.001), ("flame_pose_lr", 0.001),
           ("flame_neck_pose_lr", 0.001), ("flame_trans_lr", 0.001), ("vertices_enlargement_lr", 0.0002),
           ("random_background", False), ("use_mesh", True), ("lambda_dssim", 0.2)]
    assert list(options.OPT_PARAMS_FLAME) == ref
    p = cli_train.build_parser("gs_flame")
    group = next(g for g in p._action_groups if g.title == "Optimization Parameters")
    assert [a.dest for a in group._group_actions] == [n for n, _ in ref]
    a = cli_train.parse_args(["-s", "scene", "--gs_type", "gs_flame", "--flame_model", cases.FLAME_MODEL, "--flame_exp_lr", "0.5"])
    o = cli_train.flame_params(a)
    assert (o.flame_exp_lr, o.flame_shape_lr, o.vertices_enlargement_lr, o.iterations) == (0.5, 0.01, 0.0002, 30_000)
    m = cli_train.parse_args(["-s", "scene", "--gs_type", "gs_multi_mesh", "--meshes", "a", "--num_splats", "4"])
    assert (m.vertices_lr, m.alpha_lr, m.num_splats, m.meshes) == (0.0, 0.001, [4], ["a"])
    assert not hasattr(m, "flame_shape_lr")


@pytest.mark.parametrize("argv,flags", [
    (["--gs_type", "gs_multi_mesh"], ["--gs_type", "--meshes"]),
    (["--gs_type", "gs_multi_mesh", "--meshes", "a", "b"], ["--gs_type", "--num_splats", "--meshes"]),
    (["--gs_type", "gs_multi_mesh", "--meshes", "a", "--num_splats", "1", "2"], ["--gs_type", "--num_splats", "--meshes"]),
    (["--gs_type", "gs_flame", "--flame_model", "/nonexistent/flame2023.pkl"], ["--gs_type", "--flame_model"]),
    (["--gs_type", "gs_flame"], ["--gs_type", "--flame_model"]),
])
def test_new_refusals_name_their_flags(argv, flags, capsys):
    with pytest.raises(SystemExit):
        cli_train.parse_args(["-s", "scene"] + argv)
    err = capsys.readouterr().err
    for f in flags:
        assert f in err


def test_scene_kind_refusals(scenes_dir, capsys):
    with pytest.raises(SystemExit):
        cli_train.parse_args(["-s", scenes_dir["flame"], "--gs_type", "gs_multi_mesh", "--meshes", "a", "--num_splats", "2"])
    assert "--gs_type gs_multi_mesh" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        cli_train.parse_args(["-s", scenes_dir["multi"], "--gs_type", "gs_flame", "--flame_model", cases.FLAME_MODEL])
    assert "--gs_type gs_flame" in capsys.readouterr().err
    with pytest.raises(ValueError, match="gs_mesh"):
        dataset.read_scene(scenes_dir["multi"], "gs_mesh")
    with pytest.raises(ValueError, match="gs_flame"):
        dataset.read_scene(scenes_dir["multi"], "gs_flame", flame_model=cases.FLAME_MODEL)
    with pytest.raises(ValueError, match="gs_multi_mesh"):
        dataset.read_scene(scenes_dir["flame"], "gs_multi_mesh", num_splats=[2], meshes=["a"])
    with pytest.raises(ValueError, match="--num_splats"):
        dataset.read_scene(scenes_dir["multi"], "gs_multi_mesh", num_splats=[2], meshes=["a", "b"])


def test_existing_readers_unchanged(scenes_dir):
    sc = dataset.read_scene(scenes_dir["multi"], "gs")
    assert sc.meshes is None and sc.mesh_clouds is None and sc.flame is None and sc.point_cloud is not None
    sc = dataset.read_scene(scenes_dir["flame"], "gs_mesh", num_splats=3)
    assert sc.mesh is not None and sc.mesh._alpha.shape[1] == 3 and sc.flame is None

"""The host side of the command-line programs for the reference's scripts/ (gms_b200.cli.render_time_animated and the
others): parsers against literal restatements of each script's, the cfg_args merge, output paths, the frame times and the
morph against the reference's own functions (tests/golden/scripts.npz, written by make_scripts_golden.py), and the OBJ
writers byte for byte against the reference's."""
import argparse
import os

import numpy as np
import pytest
import torch

from gms_b200 import io_obj, scenes
from gms_b200.cli import edit_pseudomesh, options, render, render_flame, render_from_mesh_to_mesh, render_from_object
from gms_b200.cli import render_multi_mesh, render_points_time_animated, render_time_animated, save_pseudomesh


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "scripts.npz"))


def _model_parser():
    """ModelParams(parser, sentinel=True); PipelineParams(parser)."""
    p = argparse.ArgumentParser(description="Testing script parameters")
    options.add_group(p, "Loading Parameters", options.MODEL_PARAMS, fill_none=True)
    options.add_group(p, "Pipeline Parameters", options.PIPELINE_PARAMS)
    return p


def ref_render_time_animated():
    parser = _model_parser()
    parser.add_argument("--iteration", default=-1, type=int)
    parser.add_argument('--gs_type', type=str, default="gs_mesh")
    parser.add_argument("--num_splats", nargs="+", type=int, default=[2])
    parser.add_argument("--skip_train", action="store_true")
    parser.add_argument("--skip_test", action="store_true")
    parser.add_argument("--quiet", action="store_true")
    return parser


def ref_render_points_time_animated():
    parser = _model_parser()
    parser.add_argument("--iteration", default=-1, type=int)
    parser.add_argument("--skip_train", action="store_true")
    parser.add_argument("--skip_test", action="store_true")
    parser.add_argument("--quiet", action="store_true")
    parser.add_argument('--gs_type', type=str, default="gs_points")
    parser.add_argument("--num_splats", type=int, default=2)
    return parser


def ref_render_from_object():
    parser = _model_parser()
    parser.add_argument("--iteration", default=-1, type=int)
    parser.add_argument("--skip_train", action="store_false")
    parser.add_argument("--skip_test", action="store_true")
    parser.add_argument("--quiet", action="store_true")
    parser.add_argument('--gs_type', type=str, default="gs_points")
    parser.add_argument("--scale", default=2, type=float)
    parser.add_argument("--object_path", default="", type=str)
    return parser


def ref_render_flame():
    parser = _model_parser()
    parser.add_argument("--iteration", default=-1, type=int)
    parser.add_argument('--gs_type', type=str, default="gs_flame")
    parser.add_argument("--num_splats", nargs="+", type=int, default=5)
    parser.add_argument("--skip_train", action="store_true")
    parser.add_argument("--skip_test", action="store_true")
    parser.add_argument("--animated", action="store_true")
    parser.add_argument("--quiet", action="store_true")
    return parser


def ref_render_multi_mesh():
    parser = _model_parser()
    parser.add_argument("--iteration", default=-1, type=int)
    parser.add_argument('--gs_type', type=str, default="gs")
    parser.add_argument("--skip_train", action="store_true")
    parser.add_argument("--skip_test", action="store_true")
    parser.add_argument("--quiet", action="store_true")
    parser.add_argument("--num_splats", nargs="+", type=int, default=[])
    parser.add_argument("--meshes", nargs="+", type=str, default=[])
    return parser


def ref_render_from_mesh_to_mesh():
    return ref_render_time_animated()          # the same declarations, line for line


def ref_save_pseudomesh():
    parser = argparse.ArgumentParser(description="Testing script parameters")
    parser.add_argument("--model_path", type=str)
    parser.add_argument("--iteration", default=-1, type=int)
    parser.add_argument("--sh_degree", default=3, type=int)
    parser.add_argument("--scale", default=2, type=int)
    parser.add_argument("--save_faces", action="store_true")
    parser.add_argument("--save_vertices", action="store_true")
    return parser


def ref_edit_pseudomesh():
    parser = argparse.ArgumentParser(description="Testing script parameters")
    parser.add_argument("--triangle_soup_path", type=str)
    parser.add_argument("--mesh_path", type=str)
    parser.add_argument("--edited_mesh_path", type=str)
    parser.add_argument("--save_dir", type=str)
    parser.add_argument("--scale", default=1, type=int)
    return parser


def _sig(parser):
    return [(tuple(a.option_strings), a.dest, a.default, a.type, a.nargs, a.const, type(a).__name__)
            for a in parser._actions if a.dest != "help"]


SEED = [(("--seed",), "seed", 0, int, None, None, "_StoreAction")]
TARGET = [(("--target_mesh",), "target_mesh", None, str, None, None, "_StoreAction")]
PROGRAMS = {   # program: (reference parser, what the program declares after the reference's flags)
    "render_time_animated": (render_time_animated, ref_render_time_animated, SEED),
    "render_points_time_animated": (render_points_time_animated, ref_render_points_time_animated, SEED),
    "render_from_object": (render_from_object, ref_render_from_object, SEED),
    "render_flame": (render_flame, ref_render_flame, SEED),
    "render_multi_mesh": (render_multi_mesh, ref_render_multi_mesh, SEED),
    "render_from_mesh_to_mesh": (render_from_mesh_to_mesh, ref_render_from_mesh_to_mesh, TARGET + SEED),
    "save_pseudomesh": (save_pseudomesh, ref_save_pseudomesh, []),
    "edit_pseudomesh": (edit_pseudomesh, ref_edit_pseudomesh, []),
}
MODEL_PROGRAMS = [k for k, v in PROGRAMS.items() if v[2]]


@pytest.mark.parametrize("prog", sorted(PROGRAMS))
def test_flags_defaults_and_order_equal_the_script(prog):
    mod, ref, extra = PROGRAMS[prog]
    assert _sig(mod.build_parser()) == _sig(ref()) + extra
    assert mod.build_parser().description == "Testing script parameters"


def test_target_mesh_is_required(capsys):
    with pytest.raises(SystemExit):
        render_from_mesh_to_mesh.build_parser().parse_args(["-m", "x"])
    assert "--target_mesh" in capsys.readouterr().err


def restated_get_combined_args(parser, argv, cfg_text):
    """arguments/__init__.py:93-113, with the cfg_args text parsed by options.parse_cfg_args instead of eval."""
    args_cmdline = parser.parse_args(argv)
    args_cfgfile = options.parse_cfg_args(cfg_text)
    merged_dict = vars(args_cfgfile).copy()
    for k, v in vars(args_cmdline).items():
        if v is not None:
            merged_dict[k] = v
    return argparse.Namespace(**merged_dict)


@pytest.mark.parametrize("prog", MODEL_PROGRAMS)
def test_cfg_args_merge_as_get_combined_args(prog, tmp_path):
    mod = PROGRAMS[prog][0]
    cfg = argparse.Namespace(sh_degree=2, source_path=str(tmp_path / "scene"), model_path=str(tmp_path), images="imgs",
                             resolution=4, white_background=True, data_device="cuda", eval=True, num_splats=[3],
                             meshes=["a.obj"], gs_type="gs_mesh")
    (tmp_path / "cfg_args").write_text(str(cfg))
    extra = ["--target_mesh", "t.obj"] if prog == "render_from_mesh_to_mesh" else []
    for argv in (["-m", str(tmp_path)], ["-m", str(tmp_path), "--sh_degree", "1", "-r", "2", "--skip_test", "--iteration", "7"]):
        got = render.combined_args(mod.build_parser(), argv + extra)
        want = restated_get_combined_args(mod.build_parser(), argv + extra, str(cfg))
        assert vars(got) == vars(want)
        assert got.source_path == str(tmp_path / "scene") and got.white_background is True and got.images == "imgs"
        assert got.gs_type == PROGRAMS[prog][1]().get_default("gs_type")       # the script's own default wins


def test_output_paths():
    m = "/out/model"
    assert render.split_dirs(m, "test", 7, render_time_animated.FRAMES) == \
        (os.path.join(m, "test", "ours_7", "time_animated"), os.path.join(m, "test", "ours_7", "gt"))
    assert render.split_dirs(m, "train", 3, render_points_time_animated.FRAMES)[0] == \
        os.path.join(m, "train", "ours_3", "time_animated_gs_points")
    assert render.split_dirs(m, "test", 7, render_multi_mesh.FRAMES)[0] == os.path.join(m, "test", "ours_7", "renders")
    assert render.split_dirs(m, "test", 7, render_from_mesh_to_mesh.FRAMES)[0] == \
        os.path.join(m, "test", "ours_7", "from_mesh_to_mesh_animated")
    assert render_flame.output_dirs(m, "test", 9, "gs_flame", False) == \
        (os.path.join(m, "test", "ours_9", "renders_gs_flame"), os.path.join(m, "test", "ours_9", "gt"), None)
    assert render_flame.output_dirs(m, "train", 9, "gs_flame", True) == \
        (os.path.join(m, "train", "ours_9", "flame_animated"), None,
         f'{os.path.join(m, "train", "ours_9", "flame_animated")}/9_flame_render_vertices.pt')
    assert save_pseudomesh.output_dir(m, 30) == os.path.join(m, "pseudomesh_info", "ours_30")
    for path, base in (("/a/b/ficus.obj", "ficus"), ("x/hot.dog.v2.obj", "hot"), ("plain", "plain"), (".hidden.obj", "")):
        assert render_from_object.output_name(path) == os.path.basename(path).split('.')[0] == base


def test_skip_train_is_inverted_for_render_from_object():
    sc = argparse.Namespace(train_cameras=["a"], train_images=["A"], test_cameras=["b"], test_images=["B"])
    p = render_from_object.build_parser()
    assert [s[0] for s in render.splits(p.parse_args([]), sc)] == ["test"]
    assert [s[0] for s in render.splits(p.parse_args(["--skip_train"]), sc)] == ["train", "test"]
    assert [s[0] for s in render.splits(p.parse_args(["--skip_train", "--skip_test"]), sc)] == ["train"]
    q = render_time_animated.build_parser()
    assert [s[0] for s in render.splits(q.parse_args([]), sc)] == ["train", "test"]
    assert [s[0] for s in render.splits(q.parse_args(["--skip_train"]), sc)] == ["test"]


# ------------------------------------------------------------------------------------------------ frames

def test_time_sweep_against_the_script(golden):
    """Frame idx of render_time_animated: transform_hotdog_fly(vertices, linspace(0, 10 pi, n)[idx])[faces]."""
    v, f, frames = (torch.from_numpy(golden[k]) for k in ("ta/vertices", "ta/faces", "ta/frames"))
    n = frames.shape[0]
    t = render_time_animated.sweep_times(n)
    assert t.dtype == torch.float32 and torch.equal(t, torch.linspace(0, 10 * torch.pi, n))
    for idx in range(n):
        assert torch.equal(scenes.transform_hotdog_fly(v, t[idx])[f], frames[idx]), idx


def test_points_frame_time_is_t43(golden):
    tri = torch.from_numpy(golden["pta/triangles"])
    for n in (44, 45):
        frames = torch.from_numpy(golden[f"pta/frames{n}"])
        assert frames.shape[0] == n
        t43 = render_points_time_animated.frame_time(n)
        assert torch.equal(t43, torch.linspace(0, 10 * torch.pi, n)[43])
        want = scenes.transform_hotdog(tri, t43)
        assert all(torch.equal(want, fr) for fr in frames)
    assert bool(golden["pta/raises43"])
    for n in (1, 43):
        with pytest.raises(ValueError, match="t\\[43\\]"):
            render_points_time_animated.frame_time(n)


def test_points_program_refuses_43_views(monkeypatch, tmp_path, capsys):
    sc = argparse.Namespace(train_cameras=[object()] * 43, train_images=[], test_cameras=[], test_images=[])
    monkeypatch.setattr(render, "device", lambda *a: torch.device("cpu"))
    monkeypatch.setattr(render, "checkpoint", lambda *a: (7, "unused.ply"))
    monkeypatch.setattr(render, "load_views", lambda *a: sc)
    with pytest.raises(SystemExit):
        render_points_time_animated.main(["-m", str(tmp_path), "-s", str(tmp_path), "--quiet"])
    err = capsys.readouterr().err
    assert "t[43]" in err and "has 43" in err and "train" in err


def test_morph_against_the_script(golden, golden_dir):
    v, f, frames = (torch.from_numpy(golden[k]) for k in ("ta/vertices", "ta/faces", "m2m/frames"))
    n = frames.shape[0]
    assert golden["m2m/view"].tolist() == [0] * n                 # every frame from view 0's camera
    source = v[f]
    target = render_from_mesh_to_mesh.target_triangles(os.path.join(golden_dir, "scripts", "target.obj"), "cpu")
    step = render_from_mesh_to_mesh.morph_step(source, target, n)
    for idx in range(n):
        got = render_from_mesh_to_mesh.morph_triangles(source, step, idx)
        assert torch.equal(got, frames[idx]), idx
        assert torch.equal(got, source + (target - source) / n * idx)      # restated
    last = source + step * (n - 1)
    assert not torch.equal(last, target)                           # one step short of the target


def test_transforms_bit_for_bit(golden):
    v, t = torch.from_numpy(golden["fly/vertices"]), torch.from_numpy(golden["fly/t"])
    for i in range(t.shape[0]):
        assert torch.equal(scenes.transform_hotdog_fly(v, t[i]), torch.from_numpy(golden["fly/out"][i])), i
        assert torch.equal(scenes.transform_hotdog(torch.from_numpy(golden["hotdog/triangles"]), t[i]),
                           torch.from_numpy(golden["hotdog/out"][i])), i
    x = torch.from_numpy(golden["tvf/in"])
    assert torch.equal(render_from_mesh_to_mesh.transform_vertices_function(x), torch.from_numpy(golden["tvf/out"]))
    assert torch.equal(x, torch.from_numpy(golden["tvf/in"]))       # out of place


def test_object_triangles_against_the_script(golden, golden_dir):
    path = os.path.join(golden_dir, "scripts", "soup.obj")
    for s in (2, 3):
        got = render_from_object.object_triangles(path, float(s), "cpu")
        assert got.dtype == torch.float32 and torch.equal(got, torch.from_numpy(golden[f"obj/triangles_s{s}"])), s
    # read_obj's triangles are trimesh's for a triangle soup: the float64 vertices[faces], rounded to float32
    rows = [ln.split() for ln in open(path)]
    v64 = np.array([[float(x) for x in r[1:4]] for r in rows if r and r[0] == "v"])
    f = np.array([[int(x) - 1 for x in r[1:4]] for r in rows if r and r[0] == "f"])
    assert torch.equal(edit_pseudomesh.read_triangles(path), torch.tensor(v64[f]).float())


# ------------------------------------------------------------------------------------------------ writers

def test_writers_reproduce_the_scripts_byte_for_byte(golden, golden_dir, tmp_path):
    v, scale = torch.from_numpy(golden["simple/vertices"]), int(golden["simple/scale"])
    P = v.shape[0] // 3
    faces = save_pseudomesh.soup_faces(P)
    assert faces.dtype == torch.float32 and torch.equal(faces, torch.arange(0, 3 * P, dtype=torch.float32).reshape(P, 3))
    io_obj.write_obj(str(tmp_path / "simple.obj"), v * scale, faces)
    io_obj.write_obj(str(tmp_path / "soup.obj"), *io_obj.triangle_soup(v.reshape(P, 3, 3) * scale))
    io_obj.write_obj(str(tmp_path / "mesh.obj"), torch.from_numpy(golden["mesh/vertices"]), golden["mesh/faces"])
    ref = lambda n: open(os.path.join(golden_dir, "scripts", n), "rb").read()
    assert (tmp_path / "simple.obj").read_bytes() == ref("simple.obj")
    assert (tmp_path / "soup.obj").read_bytes() == ref("simple.obj")
    assert (tmp_path / "mesh.obj").read_bytes() == ref("mesh.obj")

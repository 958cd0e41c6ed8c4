"""The command-line programs for the reference's scripts/ end to end on the GPU (gms_b200.cli.render_time_animated and
the others, and cli.render for gs_multi_mesh / gs_flame), on a tiny NeRF-synthetic scene of tests/dataset_cases.py (44
train views, 3 test views) with checkpoints written by the library's savers: every PNG equals the same frame rendered
through the library API and quantized by gms_image_quantize, byte for byte; the directory trees and frame counts; gt/
equal to cli.render's; the FLAME vertex file; the pseudo-mesh files; refusals before any render; no host synchronisation
after a sweep's first frame; an overflowed frame re-renders its split with identical files; cli.metrics on the two new
cli.render types against evaluate(protocol="metrics")."""
import argparse
import os
import shutil

import numpy as np
import pytest
import torch

import dataset_cases
import flame_driver
from gms_b200 import dataset, expansion, io_image, io_obj, io_ply, scenes
from gms_b200.cli import edit_pseudomesh, render, render_flame, render_from_mesh_to_mesh, render_from_object
from gms_b200.cli import metrics as cli_metrics
from gms_b200.cli import render_multi_mesh, render_points_time_animated, render_time_animated, save_pseudomesh
from gms_b200.flame import NativeFlame
from gms_b200.model import FlameCheckpoint, FlameGaussianModel, FreeGaussianModel, MeshGaussianModel, MultiMeshGaussianModel
from gms_b200.model import PointsModel
from gms_b200.render import FlameRenderer, NativeRenderer, PointsRenderer

pytestmark = pytest.mark.gpu
IT = 7
N_TRAIN, N_TEST = 44, 3


def _write_obj(path, v, f):
    io_obj.write_obj(path, torch.as_tensor(v), torch.as_tensor(f))


def _model_dir(root, out, gs_type, white=False):
    os.makedirs(os.path.join(out, "point_cloud", f"iteration_{IT}"), exist_ok=True)
    os.makedirs(os.path.join(out, "point_cloud", "iteration_3"), exist_ok=True)      # --iteration -1 picks 7
    cfg = argparse.Namespace(sh_degree=3, source_path=root, model_path=out, images="images", resolution=-1,
                             white_background=white, data_device="cuda", eval=True, num_splats=[2], meshes=[], gs_type=gs_type)
    with open(os.path.join(out, "cfg_args"), "w") as f:
        f.write(str(cfg))
    return os.path.join(out, "point_cloud", f"iteration_{IT}", "point_cloud.ply")


@pytest.fixture(scope="module")
def work(tmp_path_factory):
    d = tmp_path_factory.mktemp("cli_scripts")
    root = str(d / "scene")
    dataset_cases.write_blender(root, [(25, 17)] * N_TRAIN, [(25, 17)] * N_TEST, seed=11, mesh=True)
    iv, ifc = scenes.icosphere(1, 0.8)
    ply = _model_dir(root, str(d / "mesh"), "gs_mesh")
    io_ply.save_mesh_model(ply, MeshGaussianModel.from_params(scenes.init_mesh_gaussians(iv, ifc, K=2, seed=0), "cuda",
                                                              packed_features=True))
    P = ifc.shape[0]
    g = scenes.flat_gaussians(P, seed=4)
    FreeGaussianModel(g["means3D"] * 0.6, torch.log(g["scales"][:, 1:]).contiguous(), g["rotations"], g["shs"],
                      torch.logit(g["opacities"]), "gs_flat", "cuda", 3).save(_model_dir(root, str(d / "flat"), "gs_flat"))
    pa = scenes.init_mesh_gaussians(*scenes.icosphere(1, 0.5), K=2, seed=1)
    tv, tf = scenes.torus(8, 6, R=0.7, r=0.15)
    pb = scenes.init_mesh_gaussians(tv, tf, K=3, seed=2)
    mm = MultiMeshGaussianModel.from_mesh_params([pa, pb], "cuda", packed_features=True)
    io_ply.save_multi_mesh_model(_model_dir(root, str(d / "multi"), "gs_multi_mesh"), mm)
    torch.manual_seed(0)
    syn = flame_driver.SyntheticFlame(rings=23, segments=24).cuda()
    fl = NativeFlame(v_template=syn.v_template, shapedirs=syn.shapedirs, posedirs=syn.posedirs, J_regressor=syn.J_regressor,
                     parents=flame_driver.PARENTS, lbs_weights=syn.lbs_weights, faces=syn.faces)
    fm = FlameGaussianModel.create(fl, torch.from_numpy(np.asarray(syn.faces, np.int64)).cuda(), K=3, seed=3)
    with torch.no_grad():
        fm._flame_exp.normal_(0, 0.3)
    io_ply.save_flame_model(_model_dir(root, str(d / "flame"), "gs_flame"), fm, point_cloud=fl.to_point_cloud())
    sc = dataset.load_scene(root, "gs_flat", eval=True, shuffle=False)
    assert (len(sc.train_cameras), len(sc.test_cameras)) == (N_TRAIN, N_TEST)
    return dict(root=root, d=d, sc=sc, iv=iv, ifc=ifc)


def _splits(sc, train=True, test=True):
    return ([("train", sc.train_cameras, sc.train_images)] if train else []) + \
           ([("test", sc.test_cameras, sc.test_images)] if test else [])


def _u8(image):
    H, W = image.shape[1:]
    return io_image.quantize(image).reshape(H, W, 3).cpu().numpy()


def _assert_pngs(d, want):
    """d holds exactly the PNGs 00000.png ... with the given uint8 [H,W,3] contents."""
    assert sorted(n for n in os.listdir(d) if n.endswith(".png")) == [f"{i:05d}.png" for i in range(len(want))], d
    for i, w in enumerate(want):
        with open(os.path.join(d, f"{i:05d}.png"), "rb") as f:
            assert np.array_equal(io_image.decode_png(f.read()), w), f"{d} {i}"


def _tree(out, split):
    return sorted(os.listdir(os.path.join(out, split, f"ours_{IT}")))


@pytest.fixture
def strict(monkeypatch):
    """Runs every frame but a sweep's first under sync debug mode "error"; counts the frames drawn; `force` = frame index
    whose first draw gets binning capacity 1 (through capacity_override), which overflows."""
    state = dict(frames=0, force=None, forced=False)
    orig, orig_gt = render.render_frames, render.write_ground_truth

    def frames(model, cls, cams, draw, *a, **k):
        def d(r, idx, cam):
            torch.cuda.set_sync_debug_mode("error" if idx > 0 else 0)
            state["frames"] += 1
            if idx == state["force"] and not state["forced"]:
                state["forced"] = True
                r.capacity_override = 1
                try:
                    return draw(r, idx, cam)
                finally:
                    r.capacity_override = None
            return draw(r, idx, cam)
        try:
            return orig(model, cls, cams, d, *a, **k)
        finally:
            torch.cuda.set_sync_debug_mode(0)

    def gt(*a, **k):
        torch.cuda.set_sync_debug_mode(0)
        return orig_gt(*a, **k)

    monkeypatch.setattr(render, "render_frames", frames)
    monkeypatch.setattr(render, "write_ground_truth", gt)
    return state


def _copy_model(work, name, tmp_path):
    out = str(tmp_path / name)
    shutil.copytree(str(work["d"] / name), out)
    return out


def _assert_gt_like_cli_render(out, gs_type, tmp_path, splits=("train", "test")):
    ref = str(tmp_path / "cli_render_gt")
    shutil.copytree(out, ref, ignore=shutil.ignore_patterns("train", "test"))
    render.main(["-m", ref, "--gs_type", gs_type, "--quiet"])
    for s in splits:
        a, b = os.path.join(out, s, f"ours_{IT}", "gt"), os.path.join(ref, s, f"ours_{IT}", "gt")
        assert sorted(os.listdir(a)) == sorted(os.listdir(b))
        for n in os.listdir(a):
            assert open(os.path.join(a, n), "rb").read() == open(os.path.join(b, n), "rb").read(), (s, n)


# ------------------------------------------------------------------------------------------------ gs_mesh sweeps

def _time_animated_expected(out, sc):
    model, _ = render.load_model("gs_mesh", os.path.join(out, "point_cloud", f"iteration_{IT}", "point_cloud.ply"), 3,
                                 torch.device("cuda"))
    bg = torch.zeros(3, device="cuda")
    want = {}
    for name, cams, _ in _splits(sc):
        r = NativeRenderer(model, cams[0].image_width, cams[0].image_height)
        t = torch.linspace(0, 10 * torch.pi, len(cams))
        want[name] = [_u8(r.render(c, bg, vertices=scenes.transform_hotdog_fly(model.vertices, t[i]))[0]) for i, c in enumerate(cams)]
    return want


def test_render_time_animated(work, strict, tmp_path):
    out = _copy_model(work, "mesh", tmp_path)
    res = render_time_animated.main(["-m", out, "--quiet"])
    assert res == {"iteration": IT, "views": {"train": N_TRAIN, "test": N_TEST}} and strict["frames"] == N_TRAIN + N_TEST
    want = _time_animated_expected(out, work["sc"])
    for name, cams, images in _splits(work["sc"]):
        assert _tree(out, name) == ["gt", "time_animated"]
        _assert_pngs(os.path.join(out, name, f"ours_{IT}", "time_animated"), want[name])
        _assert_pngs(os.path.join(out, name, f"ours_{IT}", "gt"), [im.cpu().numpy() for im in images])
    _assert_gt_like_cli_render(out, "gs_mesh", tmp_path)


def test_overflowed_frame_rerenders_the_split_identically(work, strict, tmp_path):
    out = _copy_model(work, "mesh", tmp_path)
    strict["force"] = 5
    render_time_animated.main(["-m", out, "--quiet", "--skip_test"])
    assert strict["forced"] and strict["frames"] == 2 * N_TRAIN          # the train split was drawn twice
    _assert_pngs(os.path.join(out, "train", f"ours_{IT}", "time_animated"), _time_animated_expected(out, work["sc"])["train"])
    assert not os.path.exists(os.path.join(out, "test"))


def _target_obj(work, path, faces=None):
    v = work["iv"] * np.array([1.2, 0.7, 0.9], np.float32) + np.float32(0.1) * np.sin(5 * work["iv"])
    _write_obj(path, v, work["ifc"] if faces is None else faces)


def test_render_from_mesh_to_mesh(work, strict, tmp_path):
    out = _copy_model(work, "mesh", tmp_path)
    target = str(tmp_path / "target.obj")
    _target_obj(work, target)
    render_from_mesh_to_mesh.main(["-m", out, "--target_mesh", target, "--quiet"])
    assert strict["frames"] == N_TRAIN + N_TEST
    p = io_ply.load_mesh_model(os.path.join(out, "point_cloud", f"iteration_{IT}", "point_cloud.ply"))
    src = p.vertices[p.faces].cuda()
    F = src.shape[0]
    p.vertices, p.faces = src.reshape(3 * F, 3).cpu(), torch.arange(3 * F).reshape(F, 3)
    soup = MeshGaussianModel.from_params(p, "cuda", packed_features=True)
    v, f = io_obj.read_obj(target)
    tgt = (v[:, [0, 2, 1]] * torch.tensor([1.0, -1.0, 1.0]))[f].cuda()
    bg = torch.zeros(3, device="cuda")
    for name, cams, images in _splits(work["sc"]):
        n = len(cams)
        r = NativeRenderer(soup, cams[0].image_width, cams[0].image_height)
        step = (tgt - src) / n
        want = [_u8(r.render(cams[0], bg, vertices=(src + step * i).reshape(3 * F, 3))[0]) for i in range(n)]
        assert _tree(out, name) == ["from_mesh_to_mesh_animated", "gt"]
        _assert_pngs(os.path.join(out, name, f"ours_{IT}", "from_mesh_to_mesh_animated"), want)
        _assert_pngs(os.path.join(out, name, f"ours_{IT}", "gt"), [im.cpu().numpy() for im in images])
    # a target with another face count is refused before anything is rendered
    out2 = _copy_model(work, "mesh", tmp_path / "b")
    _target_obj(work, target, work["ifc"][:-1])
    with pytest.raises(SystemExit):
        render_from_mesh_to_mesh.main(["-m", out2, "--target_mesh", target, "--quiet"])
    assert not os.path.exists(os.path.join(out2, "train"))


# ------------------------------------------------------------------------------------------------ gs_points

def test_render_points_time_animated(work, strict, tmp_path, capsys):
    out = _copy_model(work, "flat", tmp_path)
    with pytest.raises(SystemExit):           # the 3 test views have no t[43]
        render_points_time_animated.main(["-m", out, "--quiet"])
    assert "t[43]" in capsys.readouterr().err and not os.path.exists(os.path.join(out, "train"))
    render_points_time_animated.main(["-m", out, "--quiet", "--skip_test"])
    assert strict["frames"] == N_TRAIN
    model = PointsModel.from_flat_checkpoint(os.path.join(out, "point_cloud", f"iteration_{IT}", "point_cloud.ply"))
    cams = work["sc"].train_cameras
    r = PointsRenderer(model, cams[0].image_width, cams[0].image_height)
    tri = scenes.transform_hotdog(model.triangles, torch.linspace(0, 10 * torch.pi, N_TRAIN)[43])
    bg = torch.zeros(3, device="cuda")
    assert _tree(out, "train") == ["gt", "time_animated_gs_points"] and not os.path.exists(os.path.join(out, "test"))
    _assert_pngs(os.path.join(out, "train", f"ours_{IT}", "time_animated_gs_points"),
                 [_u8(r.render(c, bg, triangles=tri)[0]) for c in cams])
    _assert_gt_like_cli_render(out, "gs_points", tmp_path, splits=("train",))


def test_render_from_object(work, strict, tmp_path):
    out = _copy_model(work, "flat", tmp_path)
    obj = str(tmp_path / "ball.v1.obj")
    tri = torch.from_numpy(work["iv"][work["ifc"]])
    _write_obj(obj, *io_obj.triangle_soup(tri))
    render_from_object.main(["-m", out, "--object_path", obj, "--quiet"])       # --skip_train is store_false: train skipped
    assert not os.path.exists(os.path.join(out, "train")) and _tree(out, "test") == ["ball"]
    render_from_object.main(["-m", out, "--object_path", obj, "--quiet", "--skip_train", "--skip_test", "--scale", "1.5"])
    assert _tree(out, "train") == ["ball"] and strict["frames"] == N_TEST + N_TRAIN
    model = PointsModel.from_flat_checkpoint(os.path.join(out, "point_cloud", f"iteration_{IT}", "point_cloud.ply"))
    bg = torch.zeros(3, device="cuda")
    v, f = io_obj.read_obj(obj)         # (the OBJ holds the triangles to 6 decimals)
    for name, cams, _ in _splits(work["sc"]):
        scale = 2.0 if name == "test" else 1.5
        t = v[f].cuda() / scale
        t[:, :, 0] -= 0.2
        r = PointsRenderer(model, cams[0].image_width, cams[0].image_height)
        _assert_pngs(os.path.join(out, name, f"ours_{IT}", "ball"), [_u8(r.render(c, bg, triangles=t)[0]) for c in cams])


def test_save_and_edit_pseudomesh(work, tmp_path):
    out = _copy_model(work, "flat", tmp_path)
    save_pseudomesh.main(["--model_path", out, "--scale", "1", "--save_faces", "--save_vertices"])
    d = os.path.join(out, "pseudomesh_info", f"ours_{IT}")
    assert sorted(os.listdir(d)) == ["faces.pt", "scale_1.obj", "triangles.pt", "vertices.pt"]
    tri = PointsModel.from_flat_checkpoint(os.path.join(out, "point_cloud", f"iteration_{IT}", "point_cloud.ply")).triangles
    P = tri.shape[0]
    assert torch.equal(torch.load(os.path.join(d, "triangles.pt")), tri)
    assert torch.equal(torch.load(os.path.join(d, "vertices.pt")), tri.reshape(3 * P, 3))
    faces = torch.load(os.path.join(d, "faces.pt"))
    assert faces.dtype == torch.float32 and torch.equal(faces, torch.arange(3 * P, dtype=torch.float32).reshape(P, 3))
    io_obj.write_obj(str(tmp_path / "want.obj"), *io_obj.triangle_soup(tri))
    assert open(os.path.join(d, "scale_1.obj"), "rb").read() == (tmp_path / "want.obj").read_bytes()
    save_pseudomesh.main(["--model_path", out])
    assert os.path.exists(os.path.join(d, "scale_2.obj"))
    # edit: the soup bound to the scene's mesh, re-posed on an edited copy
    mesh = os.path.join(work["root"], "mesh.obj")
    edited = str(tmp_path / "edited.obj")
    _target_obj(work, edited)
    save = str(tmp_path / "edit")
    edit_pseudomesh.main(["--triangle_soup_path", os.path.join(d, "scale_1.obj"), "--mesh_path", mesh, "--edited_mesh_path",
                          edited, "--save_dir", save, "--scale", "3"])
    assert sorted(os.listdir(save)) == ["edited_triangles.pt", "scale_3_edited.obj"]
    sv, sf = io_obj.read_obj(os.path.join(d, "scale_1.obj"))
    mv, mf = io_obj.read_obj(mesh)
    ev, _ = io_obj.read_obj(edited)
    b = expansion.bind_pseudomesh(sv[sf].cuda(), mv.cuda(), mf.cuda())
    want = expansion.repose_pseudomesh(b, ev.cuda())
    assert torch.equal(torch.load(os.path.join(save, "edited_triangles.pt")), want)
    io_obj.write_obj(str(tmp_path / "want_e.obj"), *io_obj.triangle_soup(want * 3))
    assert open(os.path.join(save, "scale_3_edited.obj"), "rb").read() == (tmp_path / "want_e.obj").read_bytes()
    _target_obj(work, edited, work["ifc"][::-1].copy())
    with pytest.raises(SystemExit):
        edit_pseudomesh.main(["--triangle_soup_path", os.path.join(d, "scale_1.obj"), "--mesh_path", mesh,
                              "--edited_mesh_path", edited, "--save_dir", str(tmp_path / "edit2")])
    assert not os.path.exists(str(tmp_path / "edit2"))


# ------------------------------------------------------------------------------------------------ gs_flame, gs_multi_mesh

def _flame(out):
    ply = os.path.join(out, "point_cloud", f"iteration_{IT}", "point_cloud.ply")
    return FlameCheckpoint.load(ply), NativeFlame.from_checkpoint(io_ply.load_flame_model(ply)["point_cloud"])


@pytest.mark.parametrize("animated", [False, True])
def test_render_flame(work, strict, tmp_path, animated):
    out = _copy_model(work, "flame", tmp_path)
    render_flame.main(["-m", out, "--quiet"] + (["--animated"] if animated else []))
    assert strict["frames"] == N_TRAIN + N_TEST
    ck, fl = _flame(out)
    exp = ck._flame_exp.clone()
    if animated:
        exp[0, 0] = exp[0, 5] = exp[0, 7] = exp[0, 9] = 2
    v = ck.driver_vertices(fl, expression_params=exp)
    bg = torch.ones(3, device="cuda")                    # white, whatever -w says
    for name, cams, images in _splits(work["sc"]):
        r = FlameRenderer(ck, cams[0].image_width, cams[0].image_height)
        want = [_u8(r.render(c, bg, vertices=v)[0]) for c in cams]
        sub = "flame_animated" if animated else "renders_gs_flame"
        _assert_pngs(os.path.join(out, name, f"ours_{IT}", sub), want)
        if animated:
            assert _tree(out, name) == ["flame_animated"]
            assert len(os.listdir(os.path.join(out, name, f"ours_{IT}", sub))) == len(cams) + 1     # + the vertex file
        else:
            assert _tree(out, name) == ["gt", "renders_gs_flame"]
            _assert_pngs(os.path.join(out, name, f"ours_{IT}", "gt"), [im.cpu().numpy() for im in images])
    if animated:
        for name in ("train", "test"):
            io_obj.write_obj(str(tmp_path / "v.obj"), v, ck.faces)
            got = os.path.join(out, name, f"ours_{IT}", "flame_animated", f"{IT}_flame_render_vertices.pt")
            assert open(got, "rb").read() == (tmp_path / "v.obj").read_bytes()


def test_render_multi_mesh(work, strict, tmp_path):
    out = _copy_model(work, "multi", tmp_path)
    render_multi_mesh.main(["-m", out, "--quiet"])
    assert strict["frames"] == N_TRAIN + N_TEST
    model = MultiMeshGaussianModel.from_mesh_params(io_ply.load_multi_mesh_model(
        os.path.join(out, "point_cloud", f"iteration_{IT}", "point_cloud.ply")), "cuda", packed_features=True, segmented=True)
    bg = torch.zeros(3, device="cuda")
    for name, cams, images in _splits(work["sc"]):
        r = NativeRenderer(model, cams[0].image_width, cams[0].image_height)
        assert _tree(out, name) == ["gt", "renders"] and len(os.listdir(os.path.join(out, name, f"ours_{IT}", "gt"))) == len(cams)
        _assert_pngs(os.path.join(out, name, f"ours_{IT}", "renders"), [_u8(r.render(c, bg)[0]) for c in cams])
    _assert_gt_like_cli_render(out, "gs_multi_mesh", tmp_path)
    ref = str(tmp_path / "cli_render_gt")
    for name in ("train", "test"):
        a, b = (os.path.join(x, name, f"ours_{IT}") for x in (out, ref))
        for n in os.listdir(os.path.join(a, "renders")):
            assert open(os.path.join(a, "renders", n), "rb").read() == \
                open(os.path.join(b, "renders_gs_multi_mesh", n), "rb").read()


@pytest.mark.parametrize("gs_type", ["gs_multi_mesh", "gs_flame"])
def test_render_and_metrics_cli_for_new_types(work, strict, tmp_path, gs_type):
    out = _copy_model(work, {"gs_multi_mesh": "multi", "gs_flame": "flame"}[gs_type], tmp_path)
    render.main(["-m", out, "--gs_type", gs_type, "--skip_train", "--quiet"])
    assert strict["frames"] == N_TEST
    pv = cli_metrics.main(["-m", out, "--gs_type", gs_type, "--quiet"])[out]["per_view"][f"ours_{IT}"]
    sc = work["sc"]
    if gs_type == "gs_flame":
        model, fl = _flame(out)
        model.vertices = model.driver_vertices(fl)
        cls = FlameRenderer
    else:
        model = render.load_multi_mesh(os.path.join(out, "point_cloud", f"iteration_{IT}", "point_cloud.ply"), 3, "cuda")
        cls = NativeRenderer
    r = cls(model, sc.test_cameras[0].image_width, sc.test_cameras[0].image_height)
    ev = r.evaluate(sc.test_cameras, sc.test_images, torch.zeros(3, device="cuda"), protocol="metrics").per_view
    assert sorted(pv["SSIM"]) == [f"{i:05d}.png" for i in range(N_TEST)]
    for name in pv["SSIM"]:
        i = int(name[:5])
        assert pv["SSIM"][name] == float(np.float32(ev[i, 1])) and pv["PSNR"][name] == float(np.float32(ev[i, 2])), name
    assert os.path.exists(os.path.join(out, f"results_{gs_type}.json"))

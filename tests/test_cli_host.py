"""The command-line programs' host side (gms_b200.cli) against the reference's own output (tests/golden/cli.npz, written by
make_cli_golden.py) and literal restatements of its control flow: cfg_args, cameras.json, input.ply, the per-iteration
schedule, flag handling, the cfg_args merge, the 8-bit ground-truth identity and the metrics JSON files."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import dataset_cases
from gms_b200 import dataset, io_ply
from gms_b200.cli import metrics as cli_metrics
from gms_b200.cli import options
from gms_b200.cli import render as cli_render
from gms_b200.cli import train as cli_train


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "cli.npz"))


@pytest.fixture(scope="module")
def datasets(tmp_path_factory):
    return dataset_cases.write_all(str(tmp_path_factory.mktemp("cli_src")))


# ------------------------------------------------------------------------------------------------ output directory files

def test_cfg_args_equal_reference(golden, datasets, tmp_path, monkeypatch):
    monkeypatch.setenv("OAR_JOB_ID", "0123456789abcdef")
    monkeypatch.chdir(tmp_path)
    src, out = datasets["blender_a"], str(tmp_path / "out")
    i = 0
    while f"cfg/{i}/argv" in golden:
        argv = [src if a == "<SRC>" else out if a == "<OUT>" else a for a in str(golden[f"cfg/{i}/argv"]).split("\x1f")]
        args = cli_train.parse_args(argv)
        cli_train.set_default_model_path(args)
        text = options.cfg_args_string(args).replace(os.path.abspath(src), "<SRC>").replace(out, "<OUT>")
        assert text == str(golden[f"cfg/{i}/text"]), f"command line {i}"
        assert options.parse_cfg_args(options.cfg_args_string(args)).gs_type == args.gs_type
        i += 1
    assert i >= 4


@pytest.mark.parametrize("case", sorted(dataset_cases.CASES))
def test_cameras_json_and_input_ply_equal_reference(golden, datasets, tmp_path, case):
    ds, kw = dataset_cases.CASES[case]
    sc = dataset.read_scene(datasets[ds], **kw)
    cli_train.write_cameras_json(str(tmp_path / "cameras.json"), sc, seed=0)
    with open(tmp_path / "cameras.json") as f:
        assert f.read() == str(golden[f"{case}/cameras_json"])
    cli_train.write_input_ply(str(tmp_path / "input.ply"), sc, datasets[ds], kw["gs_type"], seed=0)
    el, names = io_ply.read_ply_vertices(str(tmp_path / "input.ply"))
    assert el.shape[0] == int(golden[f"{case}/ply_n"])
    assert list(names) == ["x", "y", "z", "nx", "ny", "nz", "red", "green", "blue"]
    for n in names:
        a = np.ascontiguousarray(el[n])
        ref = golden[f"{case}/ply_{n}"]
        assert a.dtype == ref.dtype and np.array_equal(a[:ref.shape[0]], ref), f"{case}: input.ply {n}"
        assert hashlib.sha256(a.tobytes()).hexdigest() == str(golden[f"{case}/ply_{n}_sha256"]), f"{case}: input.ply {n}"


def test_view_order_stream_matches_scene_and_survives_a_checkpoint(datasets, tmp_path):
    ds, kw = dataset_cases.CASES["colmap_bin_eval_r40"]
    sc = dataset.read_scene(datasets[ds], **kw)
    want = sc.view_order(40)
    vo = cli_train.ViewOrder(sc)
    got = [vo.next() for _ in range(13)]
    torch.save(vo.state_dict(), tmp_path / "s.pt")
    vo2 = cli_train.ViewOrder(sc)
    vo2.load_state_dict(torch.load(tmp_path / "s.pt", weights_only=True))
    got += [vo2.next() for _ in range(27)]
    assert got == want


# ------------------------------------------------------------------------------------------------ schedule

def restated_train_py(args):
    """train.py:61-157's control flow for the events the CLI reproduces, written out literally."""
    out = []
    for iteration in range(1, args.iterations + 1):
        ev = []
        if iteration in args.test_iterations:
            ev.append("report")
        if iteration in args.save_iterations:
            ev.append("save")
        if (args.gs_type == "gs") or (args.gs_type == "gs_flat"):
            if iteration < args.densify_until_iter:
                if iteration > args.densify_from_iter and iteration % args.densification_interval == 0:
                    ev.append("densify")
                if iteration % args.opacity_reset_interval == 0 or (args.white_background and iteration == args.densify_from_iter):
                    ev.append("reset")
        if iteration < args.iterations:
            ev.append("step")
        if iteration in args.checkpoint_iterations:
            ev.append("checkpoint")
        out.append(ev)
    return out


SCHEDULES = [
    ["--gs_type", "gs_mesh", "--iterations", "30", "--test_iterations", "10", "30", "--save_iterations", "20",
     "--checkpoint_iterations", "15", "30"],
    ["--gs_type", "gs_flat", "--iterations", "60", "--densify_from_iter", "10", "--densification_interval", "7",
     "--opacity_reset_interval", "25", "--densify_until_iter", "50", "--test_iterations", "-1", "--checkpoint_iterations", "21"],
    ["--gs_type", "gs", "-w", "--iterations", "40", "--densify_from_iter", "12", "--densification_interval", "4",
     "--opacity_reset_interval", "100", "--densify_until_iter", "33", "--save_iterations", "12", "40"],
    ["--gs_type", "gs_flat", "--white_background", "--iterations", "3000", "--test_iterations", "-1"],
    ["--gs_type", "gs_mesh", "--iterations", "1"],
]


@pytest.mark.parametrize("argv", SCHEDULES, ids=[f"s{i}" for i in range(len(SCHEDULES))])
def test_schedule_matches_train_py(argv):
    args = cli_train.parse_args(["-s", "scene"] + argv)
    assert args.save_iterations[-1] == args.iterations
    got = [cli_train.iteration_events(it, args) for it in range(1, args.iterations + 1)]
    assert got == restated_train_py(args)
    if args.gs_type != "gs_mesh":
        assert any("densify" in e for e in got) or args.iterations <= args.densify_from_iter


# ------------------------------------------------------------------------------------------------ flags

@pytest.mark.parametrize("argv,flag", [
    (["--gs_type", "gs_flame"], "--gs_type"), (["--gs_type", "gs_multi_mesh"], "--gs_type"),
    (["--antialiasing"], "--antialiasing"), (["--debug_from", "5"], "--debug_from"), (["--detect_anomaly"], "--detect_anomaly"),
    (["--convert_SHs_python"], "--convert_SHs_python"), (["--compute_cov3D_python"], "--compute_cov3D_python"),
    (["--data_device", "cpu"], "--data_device"), (["--save_xyz"], "--save_xyz"), (["--debug"], "--debug")])
def test_refused_flags_name_themselves(argv, flag, capsys):
    with pytest.raises(SystemExit):
        cli_train.parse_args(["-s", "scene"] + argv)
    assert flag in capsys.readouterr().err


def test_accepted_flags_and_defaults():
    a = cli_train.parse_args(["-s", "scene", "--ip", "0.0.0.0", "--port", "1", "--gs_type", "gs_flat", "--random_background",
                              "--lambda_dssim", "0.3", "--seed", "7"])
    assert (a.random_background, a.lambda_dssim, a.seed, a.sh_degree, a.resolution) == (True, 0.3, 7, 3, -1)
    assert a.save_iterations == [7_000, 20_000, 30_000, 60_000, 90_000, 30_000]
    o = cli_train.free_params(a)
    assert (o.lambda_dssim, o.densify_from_iter, o.min_opacity) == (0.3, 500, 0.005)
    m = cli_train.parse_args(["-s", "scene"])
    assert (m.gs_type, m.vertices_lr, m.alpha_lr, m.num_splats) == ("gs_mesh", 0.0, 0.001, [2])
    assert not hasattr(m, "densify_from_iter")


def test_cfg_args_merge_as_get_combined_args(tmp_path):
    args = cli_train.parse_args(["-s", str(tmp_path / "scene"), "-m", str(tmp_path), "--gs_type", "gs_mesh", "-w", "--eval",
                                 "--sh_degree", "2"])
    (tmp_path / "cfg_args").write_text(options.cfg_args_string(args))
    parser = cli_render.build_parser()
    merged = options.combined_args(parser, ["-m", str(tmp_path)])
    # values the command line leaves at None come from cfg_args; the others (render.py's own defaults included) win
    assert merged.source_path == str(tmp_path / "scene") and merged.white_background is True and merged.eval is True
    assert merged.sh_degree == 2 and merged.images == "images"
    assert merged.gs_type == "gs_flat" and merged.iteration == -1 and merged.num_splats == [2]
    merged = options.combined_args(parser, ["-m", str(tmp_path), "--gs_type", "gs_mesh", "--sh_degree", "1", "-w"])
    assert (merged.gs_type, merged.sh_degree, merged.white_background) == ("gs_mesh", 1, True)


def test_cfg_args_are_parsed_without_eval():
    ns = options.parse_cfg_args("Namespace(a=1, b=[2, 3], c='x', d=None, **{'not-an-identifier': 4.5})")
    assert vars(ns) == {"a": 1, "b": [2, 3], "c": "x", "d": None, "not-an-identifier": 4.5}
    for bad in ("__import__('os').system('true')", "Namespace(a=open('f'))", "Namespace(1)", "Other(a=1)"):
        with pytest.raises(ValueError):
            options.parse_cfg_args(bad)


# ------------------------------------------------------------------------------------------------ 8-bit ground truth

def test_save_image_returns_every_byte(tmp_path):
    """The render CLI writes gt PNGs straight from the resident uint8 images.  The reference writes save_image(byte / 255)
    (PILtoTorch's float32 division): that is the same byte for all 256 values."""
    b = torch.arange(256, dtype=torch.uint8)
    x = b.float() / 255.0
    assert torch.equal(x.mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8), b)      # save_image's rounding, restated
    tv = pytest.importorskip("torchvision")
    from PIL import Image
    img = torch.from_numpy(np.random.default_rng(0).permutation(256).astype(np.uint8).reshape(16, 16))
    img = torch.stack([img, img.flip(0), img.flip(1)])
    tv.utils.save_image(img.float() / 255.0, str(tmp_path / "g.png"))
    assert np.array_equal(np.asarray(Image.open(tmp_path / "g.png"))[..., :3], img.permute(1, 2, 0).numpy())


# ------------------------------------------------------------------------------------------------ metrics JSON

def test_metrics_json_shape_and_order(tmp_path):
    model = tmp_path / "model"
    methods = ["ours_30", "ours_7"]
    for m in methods:
        for sub in ("renders_gs_flat", "gt"):
            os.makedirs(model / "test" / m / sub)
        for n in ("00002.png", "00000.png", "00001.png"):
            (model / "test" / m / "renders_gs_flat" / n).write_bytes(b"")
    rng = np.random.default_rng(0)
    values = {}

    def fake_score(renders_dir, gt_dir, device):
        names = os.listdir(renders_dir)
        pv = torch.tensor(rng.uniform(0.5, 40.0, (len(names), 4)), dtype=torch.float64)
        values[renders_dir.parent.name] = (names, pv)
        return names, pv

    cli_metrics.evaluate("gs_flat", [str(model)], quiet=True, score=fake_score)
    results = json.loads((model / "results_gs_flat.json").read_text())
    per_view = json.loads((model / "per_view_gs_flat.json").read_text())
    assert list(results) == os.listdir(model / "test") == list(per_view)
    for m, (names, pv) in values.items():
        assert list(results[m]) == ["SSIM", "PSNR"] and list(per_view[m]) == ["SSIM", "PSNR"]
        for key, col in (("SSIM", 1), ("PSNR", 2)):
            f32 = pv[:, col].float()
            assert list(per_view[m][key]) == names
            assert list(per_view[m][key].values()) == f32.tolist()
            assert results[m][key] == f32.mean().item()
    text = (model / "results_gs_flat.json").read_text()
    assert text.startswith("{\n \"") and "LPIPS" not in text          # json.dump(..., indent=True), as metrics.py

"""cli.train's gs_multi_mesh and gs_flame loops against bare trainer loops, on generated 1080p scenes.

    python tools/train_cli_mesh_types_eval.py --out DIR                 # writes the scenes
    python tools/train_cli_mesh_types_eval.py --out DIR --bench         # ... and measures

Scenes (deterministic):
  colmap  `--views` views at 1920x1080 (PINHOLE, every eighth held out by --eval) of four meshes, each a scenes.object_mesh
          of `--faces` faces at its own place, rendered by the native renderer from K = 1 mesh-Gaussians; sparse/0/m<i>.obj.
          Trained with --meshes m0 m1 m2 m3 --num_splats 2 4 5 9: 20 x `--faces` Gaussians (1M at the default).
  flame   a FLAME-sized synthetic model file (5023 vertices, 9976 faces: a UV sphere with five unused vertices and its last
          faces dropped; random shape / expression / pose bases), and `--views` NeRF-synthetic views at 1920x1080 rendered
          from the model it starts training from (K = 100: 997,600 Gaussians), the last fifth held out.
Measurements, `--runs` alternating runs per arm, each a host clock around `--steps` iterations ending in a device
synchronisation (the scene is loaded once, outside the clock): cli.train's loop with reports and saves off (and TensorBoard
hidden from the import, as in tools/train_cli_eval.py) against a bare
MeshTrainer.step / FlameTrainer.step loop over the same view order.  The card's name and power limit are printed in the
same run."""
import argparse
import json
import os
import pickle
import struct
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gms_b200 import dataset, io_image, scenes  # noqa: E402
from gms_b200.cli import train as cli_train  # noqa: E402
from gms_b200.flame import NativeFlame  # noqa: E402
from gms_b200.model import FlameGaussianModel, MultiMeshGaussianModel  # noqa: E402
from gms_b200.render import NativeRenderer  # noqa: E402
from gms_b200.trainer import FlameTrainer, MeshTrainer  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from train_cli_eval import tensorboard_hidden  # noqa: E402

W, H = 1920, 1080
NUM_SPLATS = [2, 4, 5, 9]
OFFSETS = [(-0.6, -0.6, 0.0), (0.6, -0.6, 0.0), (-0.6, 0.6, 0.0), (0.6, 0.6, 0.0)]


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable: {e}"


def _png(path, img):
    import dataset_cases
    dataset_cases.write_png(path, io_image.quantize(img).cpu().numpy().reshape(H, W, 3))


def _rgba(path, img):
    import dataset_cases
    rgb = io_image.quantize(img).cpu().numpy().reshape(H, W, 3)
    dataset_cases.write_png(path, np.concatenate([rgb, np.full((H, W, 1), 255, np.uint8)], 2))


def _write_obj(path, v, f):
    with open(path, "w") as fh:
        fh.write("".join("v %.6f %.6f %.6f\n" % tuple(x) for x in v))
        fh.write("".join("f %d %d %d\n" % tuple(t) for t in f + 1))


def write_colmap(root, views, faces):
    from scipy.spatial.transform import Rotation
    sparse = os.path.join(root, "sparse", "0")
    os.makedirs(sparse, exist_ok=True)
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    params = []
    for i, off in enumerate(OFFSETS):
        v, f = scenes.object_mesh(faces)
        v = (0.45 * v + np.array(off)).astype(np.float32)
        _write_obj(os.path.join(sparse, f"m{i}.obj"), v, f)
        params.append(scenes.init_mesh_gaussians(v, f, K=1, seed=3 + i))
    model = MultiMeshGaussianModel.from_mesh_params(params, "cuda", packed_features=True)
    r = NativeRenderer(model, W, H)
    bg = torch.zeros(3, device="cuda")
    ring = scenes.ring_cameras(views, 3.6, W, H, elevation_deg=30.0)
    f = dataset.fov2focal(scenes.NERF_FOVX, W)
    with open(os.path.join(sparse, "cameras.bin"), "wb") as fh:
        fh.write(struct.pack("<Q", 1) + struct.pack("<iiQQ", 1, 1, W, H) + struct.pack("<dddd", f, f, W / 2, H / 2))
    with open(os.path.join(sparse, "images.bin"), "wb") as fh:
        fh.write(struct.pack("<Q", views))
        for k, c in enumerate(ring):
            name = f"view_{k:03d}.png"
            _png(os.path.join(root, "images", name), r.render(c.to("cuda"), bg)[0])
            w2c = c.world_view_transform.numpy().T.astype(np.float64)        # COLMAP's world->camera, OpenCV axes
            x, y, z, w = Rotation.from_matrix(w2c[:3, :3]).as_quat()
            fh.write(struct.pack("<idddddddi", k + 1, w, x, y, z, *w2c[:3, 3], 1) + name.encode() + b"\x00" + struct.pack("<Q", 0))
    with open(os.path.join(sparse, "points3D.bin"), "wb") as fh:
        fh.write(struct.pack("<Q", 0))


def write_flame_model(path):
    from flame_driver import uv_sphere
    rs = np.random.RandomState(5)
    v, f = uv_sphere(57, 88)                                # 5018 vertices, 10032 faces
    v = np.concatenate([v, np.repeat(v[-1:], 5, 0)])          # 5023 vertices
    f = f[:9976]
    V = v.shape[0]
    jr = rs.rand(5, V) ** 4
    jr /= jr.sum(1, keepdims=True)
    w = rs.rand(V, 5) ** 3
    d = dict(v_template=0.1 * v, f=f.astype(np.uint32), shapedirs=(rs.randn(V, 3, 400) * 1e-3).astype(np.float32),
             posedirs=(rs.randn(V, 3, 36) * 1e-3).astype(np.float32), J_regressor=jr,
             kintree_table=np.array([[2 ** 32 - 1, 0, 1, 1, 1], [0, 1, 2, 3, 4]], np.int64), weights=w / w.sum(1, keepdims=True))
    with open(path, "wb") as fh:
        pickle.dump(d, fh, protocol=2)


def write_flame(root, views, model_path):
    from gms_b200.scenes import ring_cameras
    for split in ("train", "test"):
        os.makedirs(os.path.join(root, split), exist_ok=True)
    driver = NativeFlame.from_model_file(model_path)
    m = FlameGaussianModel.create(driver, torch.as_tensor(driver.faces.astype(np.int64)), K=dataset.FLAME_K, seed=7)
    with torch.no_grad():
        m._opacity.fill_(2.0)
    r = NativeRenderer(m, W, H)
    bg = torch.zeros(3, device="cuda")
    ring = ring_cameras(views, 3.0, W, H, elevation_deg=15.0)
    n_test = max(1, views // 5)
    for split, cams in (("train", ring[:views - n_test]), ("test", ring[views - n_test:])):
        frames = []
        for i, c in enumerate(cams):
            _rgba(os.path.join(root, split, f"r_{i}.png"), r.render(c.to("cuda"), bg)[0])
            c2w = np.linalg.inv(c.world_view_transform.numpy().T.astype(np.float64))
            c2w[:3, 1:3] *= -1
            frames.append({"file_path": f"./{split}/r_{i}", "transform_matrix": c2w.tolist()})
        with open(os.path.join(root, f"transforms_{split}.json"), "w") as fh:
            json.dump({"camera_angle_x": scenes.NERF_FOVX, "frames": frames}, fh)


class _NoSave(cli_train.Training):
    def save(self, it):
        pass


def _timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t), out


def bench_train(root, out, gs_type, steps, runs, extra):
    argv = ["-s", root, "-m", os.path.join(out, f"run_{gs_type}"), "--gs_type", gs_type, "--eval", "--iterations", str(steps),
            "--test_iterations", "-1", "--quiet"] + extra
    args = cli_train.parse_args(argv)
    if gs_type == "gs_multi_mesh":
        scene = dataset.load_scene(root, gs_type, eval=True, num_splats=args.num_splats, meshes=args.meshes)
    else:
        scene = dataset.load_scene(root, gs_type, eval=True, flame_model=args.flame_model)
    order = scene.view_order(steps)
    P = None

    def cli():
        with tensorboard_hidden():
            t = _NoSave(cli_train.parse_args(argv), scene=scene).prepare()
        dt, _ = _timed(t.run)
        return dt, int(t.model._opacity.shape[0])

    def bare():
        bg = torch.zeros(3, device="cuda")
        if gs_type == "gs_multi_mesh":
            m = MultiMeshGaussianModel.from_mesh_params(scene.meshes, "cuda", active_sh_degree=0, packed_features=True)
            tr = MeshTrainer(m, bg, native=True)
        else:
            m = FlameGaussianModel.create(NativeFlame.from_model_file(args.flame_model), scene.flame.faces, K=dataset.FLAME_K)
            tr = FlameTrainer(m, bg, cli_train.flame_params(args))

        def loop():
            for i, v in enumerate(order):
                if gs_type == "gs_multi_mesh":
                    tr.optimizer_step = i + 1 < steps
                tr.step(scene.train_cameras[v], scene.train_images[v])
        dt, _ = _timed(loop)
        return dt, int(m._opacity.shape[0])

    cli(), bare()       # warm-up
    res = {"cli": [], "bare": []}
    for _ in range(runs):
        for name, fn in (("cli", cli), ("bare", bare)):
            dt, P = fn()
            res[name].append(1e3 * dt / steps)
    c, b = float(np.median(res["cli"])), float(np.median(res["bare"]))
    spread = {k: (max(v) - min(v)) / float(np.median(v)) * 100 for k, v in (("cli", res["cli"]), ("bare", res["bare"]))}
    res.update(cli_median_ms=c, bare_median_ms=b, diff_ms=c - b, diff_pct=100 * (c - b) / b, spread_pct=spread, P=P)
    print(json.dumps({gs_type: res}), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--views", type=int, default=40)
    ap.add_argument("--faces", type=int, default=50_000)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    colmap, flame = os.path.join(a.out, "colmap"), os.path.join(a.out, "flame")
    model_path = os.path.join(a.out, "flame_model.pkl")
    if not os.path.exists(os.path.join(colmap, "sparse", "0", "images.bin")):
        dt, _ = _timed(lambda: write_colmap(colmap, a.views, a.faces))
        print(f"COLMAP scene written in {dt:.1f} s", flush=True)
    if not os.path.exists(os.path.join(flame, "transforms_test.json")):
        write_flame_model(model_path)
        dt, _ = _timed(lambda: write_flame(flame, a.views, model_path))
        print(f"FLAME scene written in {dt:.1f} s", flush=True)
    if not a.bench:
        return
    print(card(), flush=True)
    bench_train(colmap, a.out, "gs_multi_mesh", a.steps, a.runs,
                ["--meshes"] + [f"m{i}" for i in range(len(NUM_SPLATS))] + ["--num_splats"] + [str(k) for k in NUM_SPLATS])
    bench_train(flame, a.out, "gs_flame", a.steps, a.runs, ["--flame_model", model_path])


if __name__ == "__main__":
    main()

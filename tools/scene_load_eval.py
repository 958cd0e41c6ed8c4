"""Scene loading (gms_b200/dataset.py) against the reference's host sequence, on generated datasets.

    python tools/scene_load_eval.py --out DIR [--blender-views 300] [--colmap-views 100]   # writes the datasets
    python tools/scene_load_eval.py --out DIR --bench [--steps 50]                         # ... and times them

Datasets (deterministic, from fixed seeds; smooth procedural images, so the files compress as photographs do):
  blender  a NeRF-synthetic scene: 800x800 RGBA PNGs, alpha 0 / partial / 255, black background, all views trained
  colmap   a COLMAP scene: 4946x3286 RGB JPEGs (quality 95), PINHOLE, which the automatic 1.6K rule takes to 1600x1063
Arms, each over the whole scene, host clock around the load with a device synchronisation at the end:
  decode     the host decode alone (PIL open + convert / asarray), every image, one thread
  reference  readCamerasFromTransforms' / loadCam's host sequence per view: PIL decode, the float64 numpy composite (Blender),
             Image.resize, PILtoTorch's / 255 in float32, .cuda() -- what the reference keeps resident (float32 [3,H,W])
  native     load_scene: decode on a thread pool, pinned staging, composite and resize kernels, uint8 [H,W,3] resident
Resident bytes are the sums of the images' sizes.  --bench also times one gs_flat training step (FreeTrainer, no
densification) at 1920x1080 fed uint8 against float ground truth, the two arms alternated, CUDA events around each block.
The card's name and power limit are printed in the same run."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gms_b200 import dataset, io_image, scenes  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable: {e}"


def _smooth(rng, H, W, channels):
    y = np.linspace(0, 1, H, dtype=np.float32)[:, None]
    x = np.linspace(0, 1, W, dtype=np.float32)[None, :]
    out = []
    for _ in range(channels):
        a, b, c, d = rng.uniform(2, 12, 4)
        out.append(127.5 + 100 * np.sin(a * x + b * y + c) * np.cos(d * x * y))
    return np.clip(np.stack(out, -1), 0, 255).astype(np.uint8)


def write_blender(root, n, size=800, seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "train"), exist_ok=True)
    frames = []
    for i in range(n):
        img = _smooth(rng, size, size, 4)
        img[..., 3] = np.where(img[..., 3] < 80, 0, np.where(img[..., 3] > 170, 255, img[..., 3]))
        Image.fromarray(img, "RGBA").save(os.path.join(root, "train", f"r_{i}.png"))
        az = 2 * math.pi * i / n
        eye = np.array([4 * math.cos(az), 4 * math.sin(az), 1.5])
        back = eye / np.linalg.norm(eye)
        right = np.cross([0.0, 0.0, 1.0], back)
        right /= np.linalg.norm(right)
        c2w = np.eye(4)
        c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, np.cross(back, right), back, eye
        frames.append({"file_path": f"./train/r_{i}", "transform_matrix": c2w.tolist()})
    for split, fr in (("train", frames), ("test", [])):
        with open(os.path.join(root, f"transforms_{split}.json"), "w") as f:
            json.dump({"camera_angle_x": scenes.NERF_FOVX, "frames": fr}, f)


def write_colmap(root, n, W=4946, H=3286, seed=1):
    import struct
    from PIL import Image
    rng = np.random.default_rng(seed)
    sparse = os.path.join(root, "sparse", "0")
    os.makedirs(sparse, exist_ok=True)
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    with open(os.path.join(sparse, "cameras.bin"), "wb") as f:
        f.write(struct.pack("<Q", 1) + struct.pack("<iiQQ", 1, 1, W, H) + struct.pack("<dddd", 4000.0, 4000.0, W / 2, H / 2))
    with open(os.path.join(sparse, "images.bin"), "wb") as f:
        f.write(struct.pack("<Q", n))
        for i in range(n):
            name = f"DSC_{i:04d}.JPG"
            Image.fromarray(_smooth(rng, H, W, 3), "RGB").save(os.path.join(root, "images", name), quality=95)
            q = rng.normal(size=4)
            q /= np.linalg.norm(q)
            f.write(struct.pack("<idddddddi", i + 1, *q, *rng.normal(size=3), 1) + name.encode() + b"\x00" + struct.pack("<Q", 0))
    with open(os.path.join(sparse, "points3D.bin"), "wb") as f:
        f.write(struct.pack("<Q", 1000))
        for i, (p, c) in enumerate(zip(rng.normal(size=(1000, 3)), rng.integers(0, 256, (1000, 3)))):
            f.write(struct.pack("<QdddBBBd", i + 1, *p, *[int(x) for x in c], 0.5) + struct.pack("<Q", 0))


def reference_load(sc, dev):
    """loadCam's host sequence for every view of a read_scene result -> (seconds, resident bytes)."""
    from PIL import Image
    t0 = time.perf_counter()
    total = 0
    keep = []
    for v, cam in zip(sc.train_views + sc.test_views, sc.train_cameras + sc.test_cameras):
        im = Image.open(v.path)
        if sc.mode == "RGBA":
            norm = np.array(im.convert("RGBA")) / 255.0
            bg = np.array([1, 1, 1]) if sc.white_background else np.array([0, 0, 0])
            arr = norm[:, :, :3] * norm[:, :, 3:4] + bg * (1 - norm[:, :, 3:4])
            im = Image.fromarray(np.array(arr * 255.0, dtype=np.byte).view(np.uint8), "RGB")
        t = torch.from_numpy(np.array(im.resize((cam.image_width, cam.image_height)))) / 255.0
        g = t.permute(2, 0, 1)[:3].clamp(0.0, 1.0).to(dev)
        keep.append(g)
        total += g.numel() * g.element_size()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, total


def decode_only(sc):
    t0 = time.perf_counter()
    for v in sc.train_views + sc.test_views:
        dataset.decode_image(v.path, sc.mode)
    return time.perf_counter() - t0


def native_load(path, gs_type, dev):
    t0 = time.perf_counter()
    sc = dataset.load_scene(path, gs_type, device=dev)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return dt, sum(x.numel() for x in sc.train_images + sc.test_images), sc


def step_cost(steps, dev):
    """ms per FreeTrainer step at 1920x1080, uint8 vs float ground truth, alternated blocks."""
    from gms_b200.model import FreeGaussianModel
    from gms_b200.trainer import FreeOptimizationParams, FreeTrainer
    W, H = 1920, 1080
    cams = [c.to(dev) for c in scenes.ring_cameras(4, 3.0, W, H)]
    for i, c in enumerate(cams):
        c.uid = i
    pts, colors, _ = scenes.random_point_cloud(200_000, 0)
    rng = torch.Generator().manual_seed(0)
    u8 = [torch.randint(0, 256, (H, W, 3), generator=rng, dtype=torch.uint8).to(dev) for _ in cams]
    fl = [io_image.to_device_float(x).clone() for x in u8]
    o = FreeOptimizationParams(iterations=10 ** 9, densify_until_iter=0)
    bg = torch.zeros(3, device=dev)
    res = {"uint8": [], "float": []}
    trainers = {k: FreeTrainer(FreeGaussianModel.from_point_cloud(pts, colors, "gs_flat"), bg, 3.0, o) for k in res}
    for k, gts in (("uint8", u8), ("float", fl)):     # warm-up, learn every view's N
        for it in range(8):
            trainers[k].step(cams[it % 4], gts[it % 4])
    for rep in range(3):
        for k, gts in (("uint8", u8), ("float", fl)):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for it in range(steps):
                trainers[k].step(cams[it % 4], gts[it % 4])
            e.record()
            e.synchronize()
            res[k].append(s.elapsed_time(e) / steps)
    return {k: min(v) for k, v in res.items()}, {k: v for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--blender-views", type=int, default=300)
    ap.add_argument("--colmap-views", type=int, default=100)
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--steps", type=int, default=50)
    a = ap.parse_args()
    paths = {"blender": os.path.join(a.out, "blender"), "colmap": os.path.join(a.out, "colmap")}
    t0 = time.perf_counter()
    if not os.path.exists(os.path.join(paths["blender"], "transforms_train.json")):
        write_blender(paths["blender"], a.blender_views)
    if not os.path.exists(os.path.join(paths["colmap"], "sparse")):
        write_colmap(paths["colmap"], a.colmap_views)
    print(f"datasets ready in {time.perf_counter() - t0:.1f} s under {a.out}", flush=True)
    if not a.bench:
        return
    print(card(), flush=True)
    dev = "cuda"
    torch.zeros(1, device=dev)
    for kind, path in paths.items():
        sc = dataset.read_scene(path, "gs")
        n = len(sc.train_views) + len(sc.test_views)
        w, h = sc.train_cameras[0].image_width, sc.train_cameras[0].image_height
        td = decode_only(sc)
        tr, br = reference_load(sc, dev)
        torch.cuda.empty_cache()
        tn, bn, _ = native_load(path, "gs", dev)
        torch.cuda.empty_cache()
        print(f"[{kind}] {n} views -> {w}x{h}: decode {td:.2f} s | reference {tr:.2f} s, resident {br / 2**20:.1f} MiB float32 | "
              f"load_scene {tn:.2f} s, resident {bn / 2**20:.1f} MiB uint8", flush=True)
    best, all_ = step_cost(a.steps, dev)
    print(f"[step 1920x1080 gs_flat 200k] uint8 gt {best['uint8']:.3f} ms, float gt {best['float']:.3f} ms (best of 3 blocks of "
          f"{a.steps}; all {json.dumps({k: [round(x, 3) for x in v] for k, v in all_.items()})})", flush=True)
    print(card(), flush=True)


if __name__ == "__main__":
    main()

"""cli.train --viewer on the GPU: what listening costs a run with no viewer, and what a connected viewer costs per frame.

    python tools/train_viewer_eval.py --out DIR              # writes the scene (tools/train_cli_eval.py's)
    python tools/train_viewer_eval.py --out DIR --bench      # ... and measures

Scene: tools/train_cli_eval.py's generated 1080p NeRF-synthetic scene, trained as gs_mesh at --num_splats 5 (1M mesh
Gaussians), reports and saves off, TensorBoard hidden from the import (its cost is tools/train_cli_tb_eval.py's to measure).
The scene is loaded once; each run is a fresh Training whose run() is timed by a host clock that ends in a device
synchronisation.  Arms, alternated over `--runs` runs of `--steps` iterations, medians reported:
  none      no --viewer
  listen    --viewer on an ephemeral port, no viewer connected
  served    --viewer with a viewer thread connected over TCP on 127.0.0.1 that asks for a 1920x1080 frame with
            `train: true` at every iteration (the reference's lockstep: one frame per iteration); the frame is view.Frames'
            (render, gms_image_clamp_u8, one pinned copy, one synchronisation)
  refstyle  the same viewer, frames drawn as train.py:72-74 draws them: the renderer, then ATen's
            `(torch.clamp(img, 0, 1) * 255).byte().permute(1, 2, 0).contiguous().cpu()`
Before timing, the served and refstyle frames of one camera are compared byte for byte.  The card's name, power limit and
SM clock are read in the same run (nvidia-smi, read-only query)."""
import argparse
import json
import os
import socket
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gms_b200 import dataset, network_gui, scenes  # noqa: E402
from gms_b200.cli import train as cli_train  # noqa: E402
from train_cli_eval import _NoSave, card, tensorboard_hidden, write_scene  # noqa: E402
from viewer_eval import message  # noqa: E402

W, H = 1920, 1080


def refstyle(frames):
    """train.py:72-74's frame on the renderer Frames would use: ATen's conversion and a pageable .cpu() copy."""
    renderers = {}

    def draw(cam, s):
        key = (cam.image_width, cam.image_height)
        if key not in renderers:
            renderers[key] = frames.renderer_cls(frames.model, *key)
        cam = cam.on(cam.packed().to(frames.dev))
        img = renderers[key].render(cam, frames.bg, scale_modifier=s)[0]
        return memoryview((torch.clamp(img, min=0, max=1.0) * 255).byte().permute(1, 2, 0).contiguous().cpu().numpy())
    return draw


def run_once(argv, scene, arm, msg, steps):
    """(seconds of run(), frames served) of one Training in `arm`."""
    with tensorboard_hidden():
        t = _NoSave(cli_train.parse_args(argv + (["--viewer", "--port", "0"] if arm != "none" else [])), scene=scene).prepare()
    if arm == "refstyle":
        t.viewer.draw = refstyle(t.viewer.draw)
    client, conn = None, None
    if arm in ("served", "refstyle"):
        conn = socket.create_connection(t.viewer.address)

        def ask():
            try:
                for _ in range(steps):
                    network_gui.request(conn, msg)
            finally:
                conn.close()
        client = threading.Thread(target=ask)
        client.start()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    t.run()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    if client is not None:
        client.join()
    return dt, (t.viewer.frames if t.viewer is not None else 0)


def same_bytes(argv, scene, msg):
    """One served frame and the refstyle frame of the same camera on the same (initial) model."""
    with tensorboard_hidden():
        t = _NoSave(cli_train.parse_args(argv + ["--viewer", "--port", "0"]), scene=scene).prepare()
    with torch.no_grad():
        cam = network_gui.parse(msg).camera
        a = bytes(t.viewer.draw(cam, 1.0))
        b = bytes(refstyle(t.viewer.draw)(cam, 1.0))
    t.close_viewer()
    return a == b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--views", type=int, default=40)
    ap.add_argument("--faces", type=int, default=200_000)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    root = os.path.join(a.out, "scene")
    if not os.path.exists(os.path.join(root, "transforms_train.json")):
        write_scene(root, a.views, a.faces)
    if not a.bench:
        return
    print(card(), flush=True)
    argv = ["-s", root, "-m", os.path.join(a.out, "run"), "--eval", "--iterations", str(a.steps), "--test_iterations", "-1",
            "--num_splats", "5", "--quiet"]
    scene = dataset.load_scene(root, "gs_mesh", eval=True, num_splats=5)
    msg = message(scenes.ring_cameras(8, 3.4, W, H, elevation_deg=15.0)[1])
    msg.update(train=True, keep_alive=False)
    print(json.dumps({"served_equals_refstyle": same_bytes(argv, scene, msg)}), flush=True)
    arms = ("none", "listen", "served", "refstyle")
    for arm in arms:                    # warm-up
        run_once(argv, scene, arm, msg, a.steps)
    res = {arm: [] for arm in arms}
    frames = {}
    for r in range(a.runs):
        for arm in (arms if r % 2 == 0 else arms[::-1]):
            dt, n = run_once(argv, scene, arm, msg, a.steps)
            res[arm].append(1e3 * dt / a.steps)
            frames[arm] = n
    med = {arm: float(np.median(v)) for arm, v in res.items()}
    out = {"steps": a.steps, "runs": a.runs, "ms_per_iteration": res, "median_ms": med, "frames_per_run": frames,
           "listen_minus_none_ms": med["listen"] - med["none"], "listen_minus_none_pct": 100 * (med["listen"] - med["none"]) / med["none"],
           "served_it_per_s": 1e3 / med["served"], "refstyle_it_per_s": 1e3 / med["refstyle"],
           "served_frames_per_s": frames["served"] / (med["served"] * a.steps / 1e3),
           "refstyle_frames_per_s": frames["refstyle"] / (med["refstyle"] * a.steps / 1e3),
           "served_over_refstyle": med["refstyle"] / med["served"]}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

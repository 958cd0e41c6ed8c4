"""Served remote-viewer frames on the GPU: gms_b200.cli.view's Frames over an in-process socketpair against a bare loop.

    python tools/viewer_eval.py [--bench] [--runs 7] [--frames 200] > viewer_eval.txt

Workload: a 1M mesh-Gaussian gs_mesh checkpoint (scenes.object_mesh(200_000), 5 splats per face, the trained-like
initialisation bench.py uses), written to a temporary model directory and loaded by cli.view's loader, at 1920x1080 from
16 ring cameras (bench.py's rings).

Always: every camera's served bytes are compared with the bare loop's.  With --bench, the arms alternate `--runs` times,
`--frames` frames each after a warm-up of every camera
(the three arms below):
  * served: a client thread sends each camera as a network_gui request over a socketpair and reads the reply; the
    server answers with Frames (render, gms_image_clamp_u8, one pinned copy, one synchronisation, socket send);
  * frames: the same Frames called directly with each camera, without the socket;
  * bare:   renderer.render plus the reference's `(torch.clamp(img, 0, 1) * 255).byte().permute(1, 2, 0).contiguous()
    .cpu()` (train.py:72-74), with no socket and cameras already on the device.
Frames per second by a host clock around each run (every frame ends in a synchronisation); medians over the runs.  The
card's name, power limit and SM clock are read in the same run (nvidia-smi, read-only query)."""
import argparse
import os
import socket
import statistics
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200")):
    sys.path.insert(0, p)
import torch  # noqa: E402

from gms_b200 import io_ply, network_gui, scenes  # noqa: E402
from gms_b200.cli import view  # noqa: E402
from gms_b200.model import MeshGaussianModel  # noqa: E402

W, H, F, K = 1920, 1080, 200_000, 5


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv"], text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"nvidia-smi unavailable: {e}"


def message(cam):
    """The request a viewer sends for `cam`: its matrices before network_gui's column negations."""
    wv, fp = cam.world_view_transform.clone(), cam.full_proj_transform.clone()
    wv[:, 1:3] = -wv[:, 1:3]
    fp[:, 1] = -fp[:, 1]
    return {"resolution_x": cam.image_width, "resolution_y": cam.image_height, "train": False, "fov_y": cam.FoVy,
            "fov_x": cam.FoVx, "z_near": 0.01, "z_far": 100.0, "shs_python": False, "rot_scale_python": False,
            "keep_alive": True, "scaling_modifier": 1.0, "view_matrix": wv.reshape(-1).tolist(),
            "view_projection_matrix": fp.reshape(-1).tolist()}


def model_dir(root):
    verts, faces = scenes.object_mesh(F)
    params = scenes.init_mesh_gaussians(verts, faces, K, seed=0, trained_like=True)
    out = os.path.join(root, "model")
    os.makedirs(os.path.join(out, "point_cloud", "iteration_1"))
    with open(os.path.join(out, "cfg_args"), "w") as f:
        f.write(str(argparse.Namespace(sh_degree=3, source_path="/data/object", model_path=out, images="images",
                                       resolution=-1, white_background=True, data_device="cuda", eval=False,
                                       num_splats=[K], meshes=[], gs_type="gs_mesh")))
    io_ply.save_mesh_model(os.path.join(out, "point_cloud", "iteration_1", "point_cloud.ply"),
                           MeshGaussianModel.from_params(params, "cuda", packed_features=True))
    return out, faces.shape[0] * K


def served(frames, verify, msgs):
    """Serves msgs to a client thread over a socketpair; returns (seconds, replies' images)."""
    a, b = socket.socketpair()
    images = []

    def client():
        try:
            for m in msgs:
                images.append(network_gui.request(a, m)[0])
        finally:
            a.close()

    t = threading.Thread(target=client)
    t0 = time.perf_counter()
    t.start()
    network_gui.serve(b, frames, verify, log=lambda s: None)
    t.join()
    return time.perf_counter() - t0, images


def direct(frames, cams):
    """Frames called directly (no socket): the served frame's device and copy work alone."""
    t0 = time.perf_counter()
    for c in cams:
        frames(c, 1.0)
    return time.perf_counter() - t0


def bare(renderer, bg, cams):
    t0 = time.perf_counter()
    images = [(torch.clamp(renderer.render(c, bg)[0], 0, 1) * 255).byte().permute(1, 2, 0).contiguous().cpu() for c in cams]
    return time.perf_counter() - t0, images


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bench", action="store_true", help="time the two arms (else: the byte comparison only)")
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--frames", type=int, default=200)
    args = ap.parse_args()
    print(card())
    with tempfile.TemporaryDirectory() as tmp, torch.no_grad():
        d, P = model_dir(tmp)
        _, frames, verify = view.load(["-m", d])
        cams = scenes.ring_cameras(8, 3.4, W, H, elevation_deg=15.0) + \
            scenes.ring_cameras(8, 4.4, W, H, elevation_deg=38.0, phase=0.3)
        msgs = [message(c) for c in cams]
        dev_cams = [network_gui.parse(m).camera for m in msgs]
        dev_cams = [c.on(c.packed().cuda()) for c in dev_cams]
        for i, c in enumerate(dev_cams):
            c.uid = i           # the bare loop sizes each camera from its own last visit, as for a dataset's views
        renderer = frames.renderer_cls(frames.model, W, H)
        _, got = served(frames, verify, msgs + msgs)
        _, want = bare(renderer, frames.bg, dev_cams + dev_cams)
        same = sum(g == w.numpy().tobytes() for g, w in zip(got, want))
        r = frames.sizes[(W, H)][0]
        print(f"P = {P} mesh Gaussians, {W}x{H}, {len(cams)} cameras; served bytes equal the bare loop's on {same} of "
              f"{len(got)} frames; N (last frame) {r.last_num_rendered}; overflows so far: served {r.overflows}, "
              f"bare {renderer.overflows}")
        if not args.bench:
            return
        arms = {"served": lambda order, dorder, corder: served(frames, verify, order)[0],
                "frames": lambda order, dorder, corder: direct(frames, corder),
                "bare": lambda order, dorder, corder: bare(renderer, frames.bg, dorder)[0]}
        host_cams = [network_gui.parse(m).camera for m in msgs]
        res = {arm: [] for arm in arms}
        for run in range(args.runs):
            idx = [(run * 5 + i) % len(msgs) for i in range(args.frames)]
            order, dorder, corder = [msgs[i] for i in idx], [dev_cams[i] for i in idx], [host_cams[i] for i in idx]
            for arm in (list(arms) if run % 2 == 0 else list(arms)[::-1]):
                res[arm].append(args.frames / arms[arm](order, dorder, corder))
        print(f"{args.runs} alternating runs x {args.frames} frames, frames per second:")
        for arm, fps in res.items():
            print(f"  {arm:7s} median {statistics.median(fps):8.1f}  (runs {', '.join(f'{x:.1f}' for x in fps)})")
        print(f"  served / bare: {statistics.median(res['served']) / statistics.median(res['bare']):.3f}; "
              f"frames / bare: {statistics.median(res['frames']) / statistics.median(res['bare']):.3f}")
        print(f"overflows after the runs: served {r.overflows}, bare {renderer.overflows}")


if __name__ == "__main__":
    main()

"""Mesh-driven pseudo-mesh editing on the GPU: binding and animated rendering, native against the reference protocol.

    python tools/pseudomesh_edit_eval.py [--runs 5] [--frames 100] [--faces 20000] [--bench] > pseudomesh_edit_eval.txt

Model: BASELINE config 5 turned into its 499,750-triangle pseudo-mesh (as tools/points_render_eval.py builds it), 1080p,
bound to the same object at about `--faces` faces (scenes.object_mesh), which stands in for the README's dummy mesh.
1. Binding: expansion.bind_pseudomesh against the reference protocol (scripts/edit_pseudomesh_based_on_estimated_mesh.py:
   21-54): ATen centroids, sklearn's KDTree on the host (scipy's cKDTree if sklearn is missing; the output says which), then
   torch.linalg.solve and ATen on the GPU.  Host clock, each run ending in a synchronise, `--runs` alternating runs; index
   agreement and the largest coefficient difference.
2. Animated sweep: the driving mesh moves by transform_hotdog_fly(t), t = linspace(0, 10 pi, frames).
   MeshBoundPointsRenderer.render(vertices=...) against the reference's ATen re-pose (:58-82 on the GPU binding) followed
   by PointsRenderer.render(triangles=...).  CUDA events, `--runs` alternating runs: ms per frame, library launches per
   frame, N, overflows, the largest image difference on the same frame, and the kernel spans per frame (separate pass).
3. With --bench: `bench.py --gpus 1 --steps 100 --warmup 10 --no-comparators --no-cpu-baseline`, the training step this
   change leaves alone.
The card's name, power limit and SM clock are read in the same run (nvidia-smi, read-only query)."""
import argparse
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gaussian-mesh-splatting_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gms_b200 import _lib, expansion, scenes  # noqa: E402
from gms_b200.render import MeshBoundPointsRenderer, PointsRenderer  # noqa: E402
from points_render_eval import points_model  # noqa: E402
from render_eval import card  # noqa: E402


def kd_tree_index(ref_centroids, queries):
    try:
        from sklearn.neighbors import KDTree
        return KDTree(ref_centroids).query(queries, k=1, return_distance=False).reshape(-1), "sklearn KDTree"
    except ImportError:
        from scipy.spatial import cKDTree
        return cKDTree(ref_centroids).query(queries, k=1)[1].reshape(-1), "scipy cKDTree (sklearn missing)"


def ref_frame(tri):
    v1, v2, v3 = tri[:, 0], tri[:, 1], tri[:, 2]
    a, b = v2 - v1, v3 - v1
    n = torch.cross(a, b, dim=-1)
    a = a / torch.linalg.vector_norm(a, dim=-1, keepdim=True)
    b = b / torch.linalg.vector_norm(b, dim=-1, keepdim=True)
    n = n / torch.linalg.vector_norm(n, dim=-1, keepdim=True)
    return n, a, b, v1


def ref_bind(pseudo, mesh_tri):
    """:21-54 (the cross product taken per triangle, dim=-1; the reference's dim-less torch.cross agrees for P != 3)."""
    idx, which = kd_tree_index(torch.mean(mesh_tri, dim=1).cpu().numpy(), torch.mean(pseudo, dim=1).cpu().numpy())
    idx = torch.as_tensor(idx, device=pseudo.device)
    n, a, b, v1 = ref_frame(mesh_tri[idx])
    A = torch.stack([n, a, b]).permute(1, 2, 0)
    coeffs = torch.stack([torch.linalg.solve(A, pseudo[:, j] - v1) for j in range(3)], 1)
    return idx, coeffs, which


def ref_repose(idx, coeffs, mesh_tri_edited):
    """:58-82."""
    n, a, b, v1 = ref_frame(mesh_tri_edited[idx])
    B = torch.stack((n, a, b), dim=1)
    return torch.stack([torch.bmm(coeffs[:, j:j + 1], B).reshape(-1, 3) + v1 for j in range(3)], 1)


def binding(args, model, verts, faces):
    tri = model.triangles
    mesh_tri = verts[faces]
    expansion.bind_pseudomesh(tri, verts, faces)
    ref_bind(tri, mesh_tri)
    t_nat, t_ref = [], []
    for _ in range(args.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        b = expansion.bind_pseudomesh(tri, verts, faces)
        torch.cuda.synchronize()
        t_nat.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        idx, coeffs, which = ref_bind(tri, mesh_tri)
        torch.cuda.synchronize()
        t_ref.append((time.perf_counter() - t0) * 1e3)
    agree = float((b.face.long() == idx).float().mean())
    same = b.face.long() == idx
    cdiff = float((b.coeffs[same] - coeffs[same]).abs().max())
    print(f"== binding: P = {tri.shape[0]} pseudo-triangles to F = {faces.shape[0]} faces, {args.runs} alternating runs "
          f"(host clock, each ends in a sync)")
    print(f"  bind_pseudomesh          ms {np.mean(t_nat):.2f} (runs {', '.join(f'{t:.2f}' for t in t_nat)}); "
          f"degenerate faces {b.n_degenerate}")
    print(f"  reference ({which}) ms {np.mean(t_ref):.2f} (runs {', '.join(f'{t:.2f}' for t in t_ref)})")
    print(f"  nearest-face agreement {agree * 100:.4f} % ({int((~same).sum())} differ); "
          f"max |coeff native - reference| where they agree {cdiff:.3e}")
    return b, idx, coeffs


def sweep(args, model, bm, ref_idx, ref_coeffs, cams, W, H):
    bg = torch.ones(3, device=model.triangles.device)
    ts = torch.linspace(0, 10 * math.pi, args.frames)
    rest, faces = bm.vertices, bm.faces
    poses = [scenes.transform_hotdog_fly(rest, float(t)) for t in ts]
    native = MeshBoundPointsRenderer(bm, W, H)
    tri_r = PointsRenderer(model, W, H)
    arms = {"ATen re-pose + PointsRenderer": lambda cam, V: tri_r.render(cam, bg, triangles=ref_repose(ref_idx, ref_coeffs, V[faces]))[0],
            "MeshBoundPointsRenderer": lambda cam, V: native.render(cam, bg, vertices=V)[0]}

    def frame(arm, i):
        with torch.no_grad():
            return arms[arm](cams[i % len(cams)], poses[i % len(poses)])

    for arm in arms:
        for i in range(2 * len(cams)):
            frame(arm, i)
    torch.cuda.synchronize()
    warm = native.overflows
    res = {arm: [] for arm in arms}
    for _ in range(args.runs):
        for arm in arms:
            _lib.launch_count(reset=True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(args.frames):
                frame(arm, i)
            e1.record()
            torch.cuda.synchronize()
            res[arm].append((e0.elapsed_time(e1) / args.frames, _lib.launch_count(reset=True) / args.frames))
    timed = native.overflows - warm
    spans = {}
    for arm in arms:
        _lib.set_option("time_kernels", 1)
        _lib.kernel_times(reset=True)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        aten_ms = 0.0
        for i in range(args.frames):
            if arm.startswith("ATen"):
                t0.record()
                tri = ref_repose(ref_idx, ref_coeffs, poses[i][faces])
                t1.record()
                torch.cuda.synchronize()
                aten_ms += t0.elapsed_time(t1)
                with torch.no_grad():
                    tri_r.render(cams[i % len(cams)], bg, triangles=tri)
            else:
                frame(arm, i)
        torch.cuda.synchronize()
        spans[arm] = (_lib.kernel_times(reset=True), aten_ms / args.frames)
        _lib.set_option("time_kernels", 0)
    diff = 0.0
    for i in range(0, args.frames, 7):
        a = frame("ATen re-pose + PointsRenderer", i).clone()
        b = frame("MeshBoundPointsRenderer", i)
        diff = max(diff, float((a - b).abs().max()))
    print(f"== mesh-driven animated sweep: P = {bm.binding.P}, F = {faces.shape[0]}, {W}x{H}, transform_hotdog_fly over "
          f"t = linspace(0, 10 pi, {args.frames}), {args.runs} alternating runs x {args.frames} frames (CUDA events)")
    for arm, rs in res.items():
        ms = [r[0] for r in rs]
        print(f"  {arm:30s} ms/frame {np.mean(ms):.3f} (runs {', '.join(f'{m:.3f}' for m in ms)}), launches/frame {rs[-1][1]:.1f}")
    print(f"  N (last frame): triangles path {tri_r.last_num_rendered}, native {native.last_num_rendered}; native overflows "
          f"{warm} in the warm-up, {timed} in the {args.runs * args.frames} timed frames; triangles path overflows {tri_r.overflows}")
    print(f"  max |image(ATen re-pose + PointsRenderer) - image(MeshBoundPointsRenderer)| on the same frame: {diff:.3e}")
    for arm, (kt, aten_ms) in spans.items():
        rows = ", ".join(f"{k} {ms / args.frames:.4f}" for k, (ms, n) in kt.items() if n)
        extra = f"; ATen re-pose {aten_ms:.4f}" if arm.startswith("ATen") else ""
        print(f"  {arm} spans, ms/frame: {rows}{extra}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--faces", type=int, default=20000)
    ap.add_argument("--bench", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pseudomesh_edit_eval.py measures on the GPU; no CUDA device found")
    print(card())
    dev = torch.device("cuda", 0)
    model, cams, W, H = points_model(dev)
    v, f = scenes.object_mesh(args.faces)
    verts, faces = torch.tensor(v, device=dev), torch.tensor(f, device=dev)
    b, ref_idx, ref_coeffs = binding(args, model, verts, faces)
    bm = model.bind_to_mesh(verts, faces)
    sweep(args, model, bm, ref_idx, ref_coeffs, cams, W, H)
    if args.bench:
        cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "100", "--warmup", "10",
               "--no-comparators", "--no-cpu-baseline"]
        print("== training step:", " ".join(cmd[1:]))
        for _ in range(2):
            print(subprocess.run(cmd, capture_output=True, text=True).stdout.strip().splitlines()[-1])
    print(card())


if __name__ == "__main__":
    main()

"""Generate pseudomesh_edit.npz by running the reference's own mesh-driven pseudo-mesh edit,
transform_pseudomesh_based_on_mesh (scripts/edit_pseudomesh_based_on_estimated_mesh.py:14-94), on the CPU.

    python tests/golden/make_pseudomesh_edit_golden.py        (needs /root/reference and scikit-learn)

- The meshes are handed over through a `trimesh` stand-in that carries `.triangles` (all the function reads).
- `.cuda()` returns the tensor itself and device="cuda" allocations go to the CPU, as make_golden.py maps the reference's device allocations to the CPU.
- sklearn's KDTree is wrapped to record `index_of_closest`; torch.linalg.solve is wrapped to record the coefficients of the
  three pseudo-vertices; the `edited_triangles.pt` the function saves is stored.  The .obj it writes is discarded.
- Scene: flat Gaussians on the surface of a small scenes.object_mesh, turned into their pseudo-mesh by the reference's
  PointsGaussianModel.prepare_vertices (what PointsModel.from_gaussians computes), bound to that mesh; the edited pose is
  scenes.transform_hotdog_fly(vertices, 5).  P != 3.
- The generator asserts that no query's best and second-best centroid distances (float64) are within 1e-9 relative of each
  other, so any disagreement of a nearest-face index with the fixture is a defect, not a tie.
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(HERE, "..", "..", "gaussian-mesh-splatting_b200"))
sys.path.insert(0, os.path.join(HERE, ".."))


def _stub(name, **attrs):
    m = types.ModuleType(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


_stub("plyfile", PlyData=object, PlyElement=object)
_stub("simple_knn")
_stub("simple_knn._C", distCUDA2=None)
_stub("trimesh")
_stub("smplx")
_stub("smplx.lbs", lbs=None, batch_rodrigues=None, vertices2landmarks=None, find_dynamic_lmk_idx_and_bcoords=None)
_stub("smplx.utils", Struct=object, to_tensor=None, to_np=None, rot_mat_to_euler=None)
_stub("diff_gaussian_rasterization", GaussianRasterizationSettings=object, GaussianRasterizer=object)

_orig_zeros = torch.zeros


def _zeros_cpu(*a, **k):
    if k.get("device", None) in ("cuda", torch.device("cuda")):
        k["device"] = "cpu"
    return _orig_zeros(*a, **k)


torch.zeros = _zeros_cpu

import sklearn.neighbors  # noqa: E402

from gms_b200 import scenes  # noqa: E402
import pseudomesh_oracle as orc  # noqa: E402

SEED, P, F_TARGET, T_EDIT = 7, 3000, 600, 5.0


def flat_gaussians_on(verts, faces, P, g):
    """xyz on random faces of the mesh (plus a little normal noise), in-plane log-scales, random raw quaternions."""
    v = torch.tensor(verts)
    f = torch.tensor(faces)
    fi = torch.randint(0, f.shape[0], (P,), generator=g)
    bary = torch.rand(P, 3, generator=g)
    bary = bary / bary.sum(1, keepdim=True)
    tri = v[f[fi]]
    xyz = (bary[:, :, None] * tri).sum(1) + 0.01 * torch.randn(P, 3, generator=g)
    sl = torch.log(torch.full((P, 2), 0.015)) + 0.4 * torch.randn(P, 2, generator=g)
    q = torch.randn(P, 4, generator=g)
    return xyz, sl, q


def main():
    from games.flat_splatting.scene.points_gaussian_model import PointsGaussianModel
    g = torch.Generator().manual_seed(SEED)
    verts, faces = scenes.object_mesh(F_TARGET)
    xyz, sl, q = flat_gaussians_on(verts, faces, P, g)
    pm = PointsGaussianModel(3)
    pm._xyz, pm._scaling, pm._rotation = xyz, sl, q
    _cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        pm.prepare_vertices()
    finally:
        torch.Tensor.cuda = _cuda
    triangles = pm.triangles.float().contiguous()

    v_rest = torch.tensor(verts)
    v_edit = scenes.transform_hotdog_fly(v_rest, T_EDIT)
    f_t = torch.tensor(faces, dtype=torch.int64)
    mesh = types.SimpleNamespace(triangles=v_rest[f_t].numpy())
    mesh_edited = types.SimpleNamespace(triangles=v_edit[f_t].numpy())
    pseudo = types.SimpleNamespace(triangles=triangles.numpy())

    rec = {}
    KD = sklearn.neighbors.KDTree

    class RecordingKDTree(KD):
        def query(self, X, *a, **k):
            out = super().query(X, *a, **k)
            rec["index"] = np.asarray(out).reshape(-1).copy()
            return out

    solve = torch.linalg.solve
    sols = []

    def recording_solve(A, B, *a, **k):
        x = solve(A, B, *a, **k)
        sols.append(x.detach().clone())
        return x

    import scripts.edit_pseudomesh_based_on_estimated_mesh as ref
    ref.KDTree = RecordingKDTree
    torch.linalg.solve = recording_solve
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        with tempfile.TemporaryDirectory() as d:
            ref.transform_pseudomesh_based_on_mesh(pseudo, mesh, mesh_edited, d, 1)
            edited = torch.load(os.path.join(d, "edited_triangles.pt"))
    finally:
        torch.Tensor.cuda = _cuda
        torch.linalg.solve = solve
    assert len(sols) == 3 and rec["index"].shape == (P,)
    coeffs = torch.stack(sols, 1).numpy()           # [P,3 (vertex), 3 (n, e1, e2)]

    _, _, _, best2 = orc.bind(triangles.numpy(), verts, faces)
    gap = (best2[:, 1] - best2[:, 0]) / np.maximum(best2[:, 1], 1e-300)
    assert gap.min() > 1e-9, f"a query has two nearly equidistant faces (relative gap {gap.min():.3g}); change SEED"
    np.savez_compressed(os.path.join(HERE, "pseudomesh_edit.npz"), triangles=triangles.numpy(), vertices=verts,
                        faces=faces.astype(np.int64), vertices_edited=v_edit.numpy(), t_edit=np.float32(T_EDIT),
                        index_of_closest=rec["index"].astype(np.int64), coeffs=coeffs.astype(np.float32),
                        edited_triangles=edited.numpy().astype(np.float32))
    print(f"P={P} F={faces.shape[0]} V={verts.shape[0]} min relative gap {gap.min():.3g}")


if __name__ == "__main__":
    main()

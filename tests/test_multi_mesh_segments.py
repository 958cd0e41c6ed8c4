"""CPU-only: gs_multi_mesh with a K per mesh.  The ctypes mirrors of gms_mesh_segment and of the fields gms_frame_args /
gms_render_args gained for it match the C compiler's layout; the reference-written checkpoint (tests/golden/multi_mesh_ply,
from the reference's own GaussianMultiMeshModel.save_ply) loads into the values its generator recorded; and
MultiMeshGaussianModel.from_mesh_params lays a heterogeneous-K scene out in the reference's torch.cat order."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from gms_b200 import _lib, io_ply, scenes
from gms_b200.model import MultiMeshGaussianModel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("cls,cname", [(_lib.MeshSegment, "gms_mesh_segment"), (_lib.FrameArgs, "gms_frame_args"),
                                       (_lib.RenderArgs, "gms_render_args")])
def test_layout_matches_the_ctypes_mirror(tmp_path, cls, cname):
    body = f'    printf("size %zu\\n", sizeof({cname}));\n'
    body += "".join(f'    printf("{f[0]} %zu\\n", offsetof({cname}, {f[0]}));\n' for f in cls._fields_)
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gms_b200.h"\nint main(void) {\n' + body + "    return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).strip().split("\n"))
    assert int(out["size"]) == ctypes.sizeof(cls)
    for f in cls._fields_:
        assert int(out[f[0]]) == getattr(cls, f[0]).offset, f[0]


def test_mesh_segments_array():
    arr = _lib.mesh_segments([(20, 2), (80, 3)])
    assert [(s.F, s.K) for s in arr] == [(20, 2), (80, 3)]


def test_load_reference_written_multi_mesh_checkpoint(golden_dir):
    """model_params.pt as the reference writes it (per-mesh lists, MultiMeshPointCloud entries pickled from the reference's
    own module) loads without the reference, into exactly the generator's tensors."""
    d = os.path.join(golden_dir, "multi_mesh_ply")
    e = np.load(os.path.join(d, "expected.npz"))
    plist = io_ply.load_multi_mesh_model(os.path.join(d, "point_cloud.ply"))
    assert len(plist) == int(e["n_mesh"]) == 2
    g0 = 0
    for k, p in enumerate(plist):
        np.testing.assert_array_equal(p.vertices.numpy(), e[f"vertices{k}"])
        np.testing.assert_array_equal(p.faces.numpy(), e[f"faces{k}"])
        np.testing.assert_array_equal(p._alpha.numpy(), e[f"_alpha{k}"])
        np.testing.assert_array_equal(p._scale.numpy(), e[f"_scale{k}"])
        n = p._scale.shape[0]
        assert p._alpha.shape[0] * p._alpha.shape[1] == n
        for name in ("_opacity", "_features_dc", "_features_rest"):
            np.testing.assert_array_equal(getattr(p, name).numpy(), e[name][g0:g0 + n])
        g0 += n
    assert g0 == e["_xyz"].shape[0]
    assert [p._alpha.shape[1] for p in plist] == [2, 3]


def _two_meshes():
    plist = []
    for k, (lvl, K) in enumerate([(0, 2), (1, 3)]):
        v, f = scenes.icosphere(lvl, radius=0.5 + 0.3 * k)
        p = scenes.init_mesh_gaussians(v + np.float32([1.5 * k, 0, 0]), f, K=K, seed=k)
        p._scale = 0.5 + torch.rand(p._scale.shape, generator=torch.Generator().manual_seed(10 + k))
        plist.append(p)
    return plist


@pytest.mark.parametrize("packed", [False, True])
def test_from_mesh_params_builds_the_segmented_layout(packed):
    plist = _two_meshes()
    m = MultiMeshGaussianModel.from_mesh_params(plist, "cpu", packed_features=packed)
    assert m.segments == [(20, 2), (80, 3)]
    F, K, seg = m.frame_sizes()
    assert (F, K) == (100, 0) and [(s.F, s.K) for s in seg] == m.segments
    # every per-Gaussian tensor is flat, mesh i's rows at P_i = sum_{j<i} F_j K_j: the reference's torch.cat order
    assert torch.equal(m._alpha.detach(), torch.cat([p._alpha.reshape(-1, 3) for p in plist]))
    assert torch.equal(m._scale.detach(), torch.cat([p._scale for p in plist]))
    assert torch.equal(m._opacity.detach(), torch.cat([p._opacity for p in plist]))
    assert torch.equal(m.get_features.detach(), torch.cat([torch.cat((p._features_dc, p._features_rest), 1) for p in plist]))
    assert torch.equal(m.vertices.detach(), torch.cat([p.vertices for p in plist]))
    assert torch.equal(m.faces, torch.cat([plist[0].faces, plist[1].faces + plist[0].vertices.shape[0]]))
    assert m.mesh_face_counts == [20, 80] and m.mesh_vertex_counts == [p.vertices.shape[0] for p in plist]
    for (f, a, s), p, (lo, hi) in zip(m.mesh_views(), plist, [(0, 40), (40, 280)]):
        assert a.shape == p._alpha.shape and torch.equal(a.detach(), p._alpha)
        assert a.data_ptr() == m._alpha.data_ptr() + 4 * 3 * lo            # views of the flat parameter, not copies
        assert s.data_ptr() == m._scale.data_ptr() + 4 * lo and s.shape[0] == hi - lo
        assert torch.equal(f, m.faces[slice(0, 20) if lo == 0 else slice(20, 100)])
    with pytest.raises(RuntimeError, match="FlatAdam"):
        m.training_setup()

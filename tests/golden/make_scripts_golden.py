"""Generate scripts.npz and the OBJ text files under scripts/: what the reference's scripts/ compute on the host, from
their own functions.

    python tests/golden/make_scripts_golden.py        (needs /root/reference and PIL)

Importing make_dataset_golden installs its stubs (trimesh among them: `v` / `f` records into float64 vertices and int64
faces; given `triangles` = vertices[faces] here, what trimesh gives for a mesh whose vertices it does not merge; a real
trimesh is used when it is installed).  `.cuda()` returns the tensor itself, so everything runs on the CPU.  Stored:
- write_simple_obj (save_pseudomesh.py) on a scaled triangle soup with torch.range faces -> scripts/simple.obj;
  write_mesh_obj (games/flame_splatting/utils/general_utils.py) on a small mesh -> scripts/mesh.obj;
- transform_hotdog_fly (render_time_animated.py), transform_hotdog (render_points_time_animated.py) and
  transform_vertices_function (render_from_mesh_to_mesh.py) on seeded inputs;
- the `triangles` each script's render_set hands its renderer, frame by frame, captured by replacing the renderer and
  save_image: render_time_animated (5 views), render_points_time_animated (44 and 45 views; 43 raises IndexError),
  render_from_mesh_to_mesh (4 views, and which view each frame is drawn from) and render_from_object (a triangle soup OBJ,
  scales 2 and 3; the soup is stored as scripts/soup.obj)."""
import os
import shutil
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
try:
    import trimesh as _real_trimesh
except ImportError:
    _real_trimesh = None
import make_dataset_golden as mdg  # noqa: E402  (installs the stubs)

if _real_trimesh is not None:
    sys.modules["trimesh"] = _real_trimesh
else:
    mdg._Mesh.triangles = property(lambda self: self.vertices[self.faces])

import torchvision  # noqa: E402
from games.flame_splatting.utils.general_utils import write_mesh_obj  # noqa: E402
from scripts import render_from_mesh_to_mesh as ref_m2m  # noqa: E402
from scripts import render_from_object as ref_obj  # noqa: E402
from scripts import render_points_time_animated as ref_pta  # noqa: E402
from scripts import render_time_animated as ref_ta  # noqa: E402
from scripts.save_pseudomesh import write_simple_obj  # noqa: E402

OUT = os.path.join(HERE, "scripts")
torchvision.utils.save_image = lambda *a, **k: None


class Capture:
    """Stands in for a script's `render`: records the triangles (and the view) of every frame."""

    def __init__(self, tri_arg: int):
        self.tri_arg, self.frames, self.views = tri_arg, [], []

    def __call__(self, *a):
        self.frames.append(a[self.tri_arg].clone())
        self.views.append(a[self.tri_arg + 1])
        return {"render": torch.zeros(3, 1, 1)}


def views(n):
    return [types.SimpleNamespace(original_image=torch.zeros(3, 1, 1), k=k) for k in range(n)]


def soup_obj_text(rs, P):
    tri = rs.uniform(-1.5, 1.5, (P, 3, 3))
    tri[0, 0] = (1e-7, -0.0, 12345.678901)
    lines = ["# a triangle soup: three vertices per face\n"]
    lines += ["v %.9f %.9f %.9f\n" % tuple(x) for x in tri.reshape(-1, 3)]
    lines += ["f %d %d %d\n" % (3 * i + 1, 3 * i + 2, 3 * i + 3) for i in range(P)]
    return "".join(lines)


def main():
    rs = np.random.RandomState(7)
    res = {}
    os.makedirs(OUT, exist_ok=True)
    with tempfile.TemporaryDirectory() as d:
        # writers
        P = 6
        tri = torch.tensor(rs.uniform(-2, 2, (P, 3, 3)), dtype=torch.float32)
        tri[0, 0] = torch.tensor([1e-7, -0.0, 4.0000005])
        tri[1, 1] = torch.tensor([-1234.5678, 0.5e-6, -1.5e-6])
        faces = torch.range(0, P * 3 - 1).reshape(P, 3)
        vertices = tri.reshape(P * 3, 3)
        res["simple/vertices"], res["simple/scale"] = vertices.numpy(), np.array(2, np.int64)
        write_simple_obj(mesh_v=(vertices * 2).detach().cpu().numpy(), mesh_f=faces, filepath=os.path.join(OUT, "simple.obj"))
        mv = torch.tensor(rs.normal(size=(9, 3)) * 3, dtype=torch.float32)
        mf = rs.randint(0, 9, (7, 3)).astype(np.int64)
        res["mesh/vertices"], res["mesh/faces"] = mv.numpy(), mf
        write_mesh_obj(mv, mf, os.path.join(OUT, "mesh.obj"))
        # transforms
        v = torch.tensor(rs.normal(size=(40, 3)), dtype=torch.float32)
        t = torch.linspace(0, 10 * torch.pi, 7)
        res["fly/vertices"], res["fly/t"] = v.numpy(), t.numpy()
        res["fly/out"] = np.stack([ref_ta.transform_hotdog_fly(v, t[i], None).numpy() for i in range(7)])
        tr = torch.tensor(rs.normal(size=(11, 3, 3)), dtype=torch.float32)
        res["hotdog/triangles"] = tr.numpy()
        res["hotdog/out"] = np.stack([ref_pta.transform_hotdog(tr, t[i]).numpy() for i in range(7)])
        v64 = torch.tensor(rs.normal(size=(13, 3)), dtype=torch.float64)
        res["tvf/in"], res["tvf/out"] = v64.numpy(), ref_m2m.transform_vertices_function(v64.clone()).numpy()
        # render_time_animated: a mesh of 12 vertices, 20 faces
        from gms_b200 import scenes
        iv, ifc = scenes.icosphere(0, 0.8)
        g = types.SimpleNamespace(vertices=torch.tensor(iv), faces=ifc)
        cap = Capture(1)
        ref_ta.render = cap
        ref_ta.render_set(None, d, "train", 7, views(5), g, None, None)
        res["ta/vertices"], res["ta/faces"] = iv, ifc
        res["ta/frames"] = torch.stack(cap.frames).numpy()
        # render_points_time_animated
        pt = torch.tensor(rs.normal(size=(8, 3, 3)), dtype=torch.float32)
        g = types.SimpleNamespace(v1=pt[:, 0].clone(), v2=pt[:, 1].clone(), v3=pt[:, 2].clone())
        res["pta/triangles"] = pt.numpy()
        for n in (44, 45):
            cap = Capture(0)
            ref_pta.render = cap
            ref_pta.render_set(d, "train", 7, views(n), g, None, None)
            res[f"pta/frames{n}"] = torch.stack(cap.frames).numpy()
        try:
            ref_pta.render = Capture(0)
            ref_pta.render_set(d, "train", 7, views(43), g, None, None)
            res["pta/raises43"] = np.array(False)
        except IndexError:
            res["pta/raises43"] = np.array(True)
        # render_from_mesh_to_mesh: the target at the script's fixed path, relative to the working directory
        work = os.path.join(d, "work")
        os.makedirs(os.path.join(d, "data", "ficus"))
        os.makedirs(work)
        tv = rs.normal(size=(12, 3)) * 0.7
        tf = np.roll(ifc, 1, axis=1)[::-1].copy()
        with open(os.path.join(d, "data", "ficus", "ficus_animate.obj"), "w") as f:
            f.write("".join("v %.9f %.9f %.9f\n" % tuple(x) for x in tv) + "".join("f %d %d %d\n" % tuple(x + 1) for x in tf))
        shutil.copy(os.path.join(d, "data", "ficus", "ficus_animate.obj"), os.path.join(OUT, "target.obj"))
        g = types.SimpleNamespace(vertices=torch.tensor(iv), faces=ifc)
        cap = Capture(0)
        ref_m2m.render = cap
        cwd = os.getcwd()
        os.chdir(work)
        try:
            vs = views(4)
            ref_m2m.render_set(d, "train", 7, vs, g, None, None)
        finally:
            os.chdir(cwd)
        res["m2m/frames"] = torch.stack(cap.frames).numpy()
        res["m2m/view"] = np.array([w.k for w in cap.views], np.int64)
        # render_from_object on a triangle soup
        with open(os.path.join(OUT, "soup.obj"), "w") as f:
            f.write(soup_obj_text(rs, 5))
        for scale in (2.0, 3.0):
            cap = Capture(0)
            ref_obj.render = cap
            ref_obj.render_set(d, os.path.join(OUT, "soup.obj"), "train", 7, views(2), None, None, None, scale)
            res[f"obj/triangles_s{int(scale)}"] = cap.frames[0].numpy()
            assert all(torch.equal(x, cap.frames[0]) for x in cap.frames)
    np.savez_compressed(os.path.join(HERE, "scripts.npz"), **res)
    print(f"{len(res)} arrays, {os.path.getsize(os.path.join(HERE, 'scripts.npz'))} bytes")


if __name__ == "__main__":
    main()

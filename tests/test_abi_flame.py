"""CPU-only: the ctypes mirrors of the structs that gained `alpha_activation` (gms_expand_args, gms_frame_args,
gms_render_args) and of gms_flame_render_args have the sizes and field offsets the C compiler gives the header, the activation constants match, and
FlatAdam packs the ten gs_flame groups into gms_adam_step's eight segments without changing any group's hyper-parameters."""
import os
import subprocess

import ctypes
import torch

from gms_b200 import _lib
from gms_b200.optim import FlatAdam

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _layout(tmp_path, cls, cname):
    body = f'    printf("size %zu\\n", sizeof({cname}));\n'
    body += "".join(f'    printf("{f[0]} %zu\\n", offsetof({cname}, {f[0]}));\n' for f in cls._fields_)
    body += '    printf("relu %d\\n", GMS_ALPHA_RELU);\n    printf("softmax %d\\n", GMS_ALPHA_SOFTMAX);\n'
    src = tmp_path / f"{cname}.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gms_b200.h"\nint main(void) {\n' + body + "    return 0;\n}\n")
    exe = tmp_path / cname
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    return dict(l.split() for l in subprocess.check_output([str(exe)], text=True).strip().split("\n"))


def test_alpha_activation_structs_match_the_header(tmp_path):
    out = _layout(tmp_path, _lib.FlameRenderArgs, "gms_flame_render_args")
    assert int(out["size"]) == ctypes.sizeof(_lib.FlameRenderArgs)
    for f in _lib.FlameRenderArgs._fields_:
        assert int(out[f[0]]) == getattr(_lib.FlameRenderArgs, f[0]).offset, f[0]
    for cls, cname in ((_lib.ExpandArgs, "gms_expand_args"), (_lib.FrameArgs, "gms_frame_args"), (_lib.RenderArgs, "gms_render_args")):
        out = _layout(tmp_path, cls, cname)
        assert int(out["size"]) == ctypes.sizeof(cls), cname
        for f in cls._fields_:
            assert int(out[f[0]]) == getattr(cls, f[0]).offset, (cname, f[0])
        assert cls._fields_[-1] == ("alpha_activation", ctypes.c_int32), f"{cname}: alpha_activation must be the trailing field"
        assert (int(out["relu"]), int(out["softmax"])) == (_lib.ALPHA_RELU, _lib.ALPHA_SOFTMAX)


def test_zero_initialised_args_select_relu():
    for cls in (_lib.ExpandArgs, _lib.FrameArgs, _lib.RenderArgs):
        assert cls().alpha_activation == _lib.ALPHA_RELU


def test_flat_adam_merges_equal_neighbouring_groups_past_eight():
    from gms_b200.trainer import FlameOptimizationParams, flame_model_groups

    class M:
        pass
    m = M()
    z = lambda *s: torch.zeros(*s)
    m._flame_shape, m._flame_exp, m._flame_pose, m._flame_neck_pose, m._flame_trans = z(1, 100), z(1, 50), z(1, 6), z(1, 3), z(1, 3)
    m._vertices_enlargement, m._alpha, m._opacity, m._scales, m._features = z(50, 3), z(10, 4, 3), z(40, 1), z(40, 1), z(40, 16, 3)
    descs = []
    opt = FlatAdam(flame_model_groups(m, FlameOptimizationParams()), kernel=descs.append, sh_factored=True)
    assert len(opt.groups) == 10
    opt.step_rest()
    d = descs[-1]
    # shape | expression, pose, neck_pose, transl | vertices_enlargement | alpha | opacity | scaling  (+ features, stripped)
    assert d["lr0"] == [0.01, 0.001, 0.0002, 0.001, 0.05, 0.005]
    assert d["seg_end"] == [opt.ends[0], opt.ends[4], opt.ends[5], opt.ends[6], opt.ends[7], opt.ends[8]]
    # every element's learning rate is its group's
    for i, g in enumerate(opt.groups[:-1]):
        lo = opt.ends[i - 1] if i else 0
        k = next(j for j, e in enumerate(d["seg_end"]) if lo < e)
        assert d["lr0"][k] == g["lr"], g["name"]

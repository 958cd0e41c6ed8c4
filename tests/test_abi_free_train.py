"""CPU-only: the ctypes mirrors of the free-Gaussian structs (gms_free_train_frame, gms_free_render_frame, gms_densify_plan /
gms_densify_apply) have the sizes and field offsets the C compiler gives the header's structs, and the new entry points
are listed."""
import ctypes
import os
import subprocess

import pytest

from gms_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRUCTS = [(_lib.FreeFrameArgs, "gms_free_frame_args"), (_lib.FreeRenderArgs, "gms_free_render_args"),
           (_lib.DensifyPlanArgs, "gms_densify_plan_args"), (_lib.FreeSet, "gms_free_set"),
           (_lib.DensifyApplyArgs, "gms_densify_apply_args")]


@pytest.mark.parametrize("cls,cname", STRUCTS, ids=[c for _, c in STRUCTS])
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


def test_free_symbols_are_listed():
    assert {"gms_free_train_frame", "gms_free_render_frame", "gms_densify_scratch_bytes", "gms_densify_plan",
            "gms_densify_apply"} <= set(_lib.ABI_SYMBOLS)

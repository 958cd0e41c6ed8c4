"""CPU-only: the ctypes mirrors of gms_pseudomesh_bind_args, gms_pseudomesh_repose_args and gms_bound_points_render_args
have the size and field offsets the C compiler gives the header's structs, and the library lists the new entry points."""
import ctypes
import os
import subprocess

import pytest

from gms_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("cls,cname", [(_lib.PseudomeshBindArgs, "gms_pseudomesh_bind_args"),
                                       (_lib.PseudomeshReposeArgs, "gms_pseudomesh_repose_args"),
                                       (_lib.BoundPointsRenderArgs, "gms_bound_points_render_args")])
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


def test_pseudomesh_symbols_are_listed():
    assert {"gms_pseudomesh_bind_scratch_bytes", "gms_pseudomesh_bind", "gms_pseudomesh_repose",
            "gms_bound_points_render_workspace_bytes", "gms_bound_points_render_frame"} <= set(_lib.ABI_SYMBOLS)

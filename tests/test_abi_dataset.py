"""CPU-only: the ctypes mirror of gms_resize_args has the size and field offsets the C compiler gives the header's struct
(compiled as C99), and the library exports the ground-truth preparation entry points."""
import ctypes
import os
import subprocess

from gms_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_layout_matches_the_ctypes_mirror(tmp_path):
    cls, cname = _lib.ResizeArgs, "gms_resize_args"
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


def test_dataset_symbols_are_exported():
    names = {"gms_image_composite_rgba", "gms_image_resize_u8"}
    assert names <= set(_lib.ABI_SYMBOLS)
    L = _lib.lib()
    for n in names:
        assert hasattr(L, n), n

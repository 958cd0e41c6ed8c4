"""CPU-only checks of FLAME's native vertex model (gms_b200.flame, csrc/gms_flame.cuh):
  - the loader against FLAME.__init__'s own buffers (tests/golden/flame_lbs, written by the reference's FLAME class) for a
    dense, a scipy-sparse and a chumpy-style model file, and from_checkpoint on a reference-written checkpoint, bit for bit;
  - the float64 restatement (tests/flame_lbs_oracle) against FLAME.forward's vertices on that model;
  - gms_flame_lbs_args against the header (gcc), and every GMS_E_ARG case, without a device;
  - the joint stage (Rodrigues, the chain, the pose feature and their backward), compiled for the CPU from the product
    header, against float64 at zero pose, at |theta| down to 1e-7 where the +1e-8 dominates, and near pi and 2 pi."""
import ctypes as C
import os
import pickle
import subprocess

import numpy as np
import pytest
import torch

import flame_lbs_oracle as oracle
from gms_b200 import _lib, io_ply
from gms_b200.flame import NativeFlame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "flame_lbs")
CSRC = os.path.join(ROOT, "gaussian-mesh-splatting_b200", "csrc")
KEYS = ("v_template", "shapedirs", "posedirs", "J_regressor", "parents", "lbs_weights", "faces_tensor")


@pytest.fixture(scope="module")
def buffers():
    return dict(np.load(os.path.join(GOLD, "buffers.npz")))


def _check_model(fl: NativeFlame, buf, name, n_shape=100, n_exp=50):
    ref = {k: torch.tensor(buf[f"{name}/{k}"]) for k in KEYS}
    assert torch.equal(fl.v_template, ref["v_template"])
    assert torch.equal(fl.shapedirs, oracle.packed(ref["shapedirs"], n_shape, n_exp).permute(2, 0, 1).reshape(n_shape + n_exp, -1))
    for k in ("posedirs", "J_regressor", "lbs_weights"):
        assert torch.equal(getattr(fl, k), ref[k]), (name, k)
    assert fl.parents == tuple(ref["parents"].tolist())
    assert torch.equal(fl.faces_tensor, ref["faces_tensor"])


@pytest.mark.parametrize("name", ["dense", "sparse", "ch"])
def test_model_file_gives_flame_init_buffers(buffers, name):
    fl = NativeFlame.from_model_file(os.path.join(GOLD, f"model_{name}.pkl"), device="cpu")
    _check_model(fl, buffers, name)


def test_model_file_with_other_active_columns(buffers, tmp_path):
    fl = NativeFlame.from_model_file(os.path.join(GOLD, "model_dense.pkl"), n_shape=300, n_exp=100, device="cpu")
    assert torch.equal(fl.shapedirs, torch.tensor(buffers["dense/shapedirs"]).permute(2, 0, 1).reshape(400, -1))


def test_model_file_without_an_array_names_the_key(tmp_path):
    with open(os.path.join(GOLD, "model_dense.pkl"), "rb") as fh:
        d = pickle.load(fh, encoding="latin1")
    d["posedirs"] = "not an array"
    p = tmp_path / "bad.pkl"
    p.write_bytes(pickle.dumps(d, protocol=2))
    with pytest.raises(ValueError, match="'posedirs'"):
        NativeFlame.from_model_file(str(p), device="cpu")
    del d["posedirs"]
    p.write_bytes(pickle.dumps(d, protocol=2))
    with pytest.raises(ValueError, match="'posedirs'"):
        NativeFlame.from_model_file(str(p), device="cpu")


def test_from_checkpoint_reads_the_reference_module_bit_for_bit(buffers):
    ck = io_ply.load_flame_model(os.path.join(GOLD, "point_cloud.ply"))
    fl = NativeFlame.from_checkpoint(ck["point_cloud"], device="cpu")
    _check_model(fl, buffers, "dense")
    # the self-contained form round-trips
    back = NativeFlame.from_checkpoint(fl.to_point_cloud(), device="cpu")
    for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights", "faces_tensor"):
        assert torch.equal(getattr(back, k), getattr(fl, k)), k
    assert (back.parents, back.n_shape, back.n_exp) == (fl.parents, fl.n_shape, fl.n_exp)


def test_restatement_matches_flame_forward(buffers):
    e = np.load(os.path.join(GOLD, "expected.npz"))
    b = {k: torch.tensor(buffers[f"dense/{k}"]).double() for k in KEYS[:-2] + ("lbs_weights",)}
    b["shapedirs"] = oracle.packed(b["shapedirs"], 100, 50)
    b["parents"] = buffers["dense/parents"].tolist()
    t = lambda k: torch.tensor(e[k]).double()
    v = oracle.lbs(b, t("shape_params"), t("expression_params"), t("pose_params"), t("neck_pose"), t("transl"))
    np.testing.assert_allclose(v.numpy(), e["vertices"], rtol=0, atol=2e-6)


# ---- the C ABI

def test_lbs_args_match_the_header(tmp_path):
    cls, cname = _lib.FlameLbsArgs, "gms_flame_lbs_args"
    body = f'    printf("size %zu\\n", sizeof({cname}));\n'
    body += "".join(f'    printf("{f[0]} %zu\\n", offsetof({cname}, {f[0]}));\n' for f in cls._fields_)
    body += '    printf("joints %d\\n", GMS_FLAME_JOINTS);\n'
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gms_b200.h"\nint main(void) {\n' + body + "    return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).strip().split("\n"))
    assert int(out["size"]) == C.sizeof(cls)
    for f in cls._fields_:
        assert int(out[f[0]]) == getattr(cls, f[0]).offset, f[0]
    assert int(out["joints"]) == _lib.FLAME_JOINTS
    assert {"gms_flame_lbs_workspace_bytes", "gms_flame_lbs_forward", "gms_flame_lbs_backward"} <= set(_lib.ABI_SYMBOLS)


def _valid_args(V=10, n_shape=4, n_exp=3):
    keep = []

    def buf(n):
        a = np.zeros(max(n, 1) + 64, np.float32)
        keep.append(a)
        return a.ctypes.data + (-a.ctypes.data) % 16
    L = _lib.lib()
    a = _lib.FlameLbsArgs()
    a.V, a.n_shape, a.n_exp, a.n_joints = V, n_shape, n_exp, 5
    for j, p in enumerate((-1, 0, 1, 1, 1)):
        a.parents[j] = p
    B = n_shape + n_exp
    sizes = dict(v_template=3 * V, shapedirs=3 * V * B, posedirs=108 * V, J_regressor=5 * V, lbs_weights=5 * V, shape=n_shape,
                 expression=n_exp, pose=6, neck_pose=3, transl=3, enlargement=3 * V, vertices=3 * V, vertices_grad=3 * V,
                 d_shape=n_shape, d_expression=n_exp, d_pose=6, d_neck_pose=3, d_transl=3, d_enlargement=3 * V)
    for k, n in sizes.items():
        setattr(a, k, buf(n))
    a.workspace_bytes = int(L.gms_flame_lbs_workspace_bytes(V))
    a.workspace = buf(a.workspace_bytes // 4 + 1)
    return a, keep


def _expect_arg_error(mutate, backward=False):
    a, keep = _valid_args()
    mutate(a)
    L = _lib.lib()
    fn = L.gms_flame_lbs_backward if backward else L.gms_flame_lbs_forward
    assert fn(C.byref(a), None) == _lib.GMS_E_ARG, L.gms_last_error()


@pytest.mark.parametrize("backward", [False, True])
def test_bad_arguments_are_refused_before_any_launch(backward):
    def setp(j, v):
        def f(a):
            a.parents[j] = v
        return f
    cases = [lambda a: setattr(a, "n_joints", 4), lambda a: setattr(a, "n_joints", 6), setp(0, 0), setp(1, 1), setp(2, 2), setp(4, 5),
             setp(3, -1), lambda a: setattr(a, "V", 0), lambda a: setattr(a, "V", -3), lambda a: setattr(a, "n_shape", 301),
             lambda a: setattr(a, "n_exp", 101), lambda a: setattr(a, "n_shape", -1), lambda a: setattr(a, "n_exp", -1),
             lambda a: setattr(a, "workspace_bytes", a.workspace_bytes - 1)]
    for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights", "shape", "expression", "pose", "neck_pose",
              "transl", "enlargement", "workspace"):
        cases.append(lambda a, k=k: setattr(a, k, None))
        cases.append(lambda a, k=k: setattr(a, k, getattr(a, k) + 2))
    out = ("d_shape", "d_expression", "d_pose", "d_neck_pose", "d_transl", "d_enlargement", "vertices_grad") if backward else ("vertices",)
    for k in out:
        cases.append(lambda a, k=k: setattr(a, k, None))
        cases.append(lambda a, k=k: setattr(a, k, getattr(a, k) + 1))
    for c in cases:
        _expect_arg_error(c, backward)


def test_workspace_bytes_refuses_nonpositive_v():
    L = _lib.lib()
    assert L.gms_flame_lbs_workspace_bytes(0) == 0 and L.gms_flame_lbs_workspace_bytes(-1) == 0
    assert L.gms_flame_lbs_workspace_bytes(5023) > 3 * 3 * 5023 * 4


# ---- the joint stage on the CPU

SHIM = r'''
#include <stdint.h>
#include "gms_flame.cuh"
extern "C" int shim_flame_joints(const float* pose, const float* neck, const float* J, const int32_t* parents, const float* dA,
                                 const float* dfeat, float* R, float* A, float* feat, float* dpose, float* dneck, float* dJ) {
    GmsFlameJoints o;
    gms_flame_joints_fwd(pose, neck, J, parents, o);
    for (int k = 0; k < 45; k++) R[k] = (&o.R[0][0])[k];
    for (int k = 0; k < 60; k++) A[k] = (&o.A[0][0])[k];
    for (int k = 0; k < 36; k++) feat[k] = o.feat[k];
    gms_flame_joints_bwd(pose, neck, J, parents, o, dA, dfeat, dpose, dneck, dJ);
    return 0;
}
'''


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("flame_shim")
    src, so = d / "shim.cpp", d / "libflame_shim.so"
    src.write_text(SHIM)
    subprocess.check_call(["/usr/bin/g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I", CSRC, "-o", str(so), str(src)])
    return C.CDLL(str(so))


def _run_shim(shim, pose, neck, J, parents, dA, dfeat):
    f32 = lambda x: np.ascontiguousarray(x, np.float32)
    ins = [f32(pose), f32(neck), f32(J), np.ascontiguousarray(parents, np.int32), f32(dA), f32(dfeat)]
    outs = [np.zeros(n, np.float32) for n in (45, 60, 36, 6, 3, 15)]
    shim.shim_flame_joints(*[x.ctypes.data_as(C.c_void_p) for x in ins + outs])
    return outs


def _torch(pose, neck, J, parents, dA, dfeat, dtype):
    """Forward and gradients through the restatement in `dtype` (the fp32 inputs widened for float64)."""
    d = lambda x: torch.tensor(np.asarray(x, np.float32), dtype=dtype, requires_grad=True)
    p, n, j = d(pose), d(neck), d(J)
    R, feat, A = oracle.joints(oracle.full_pose(p, n), j.view(5, 3), list(parents))
    ((A.reshape(-1) * torch.tensor(dA, dtype=dtype)).sum() + (feat * torch.tensor(dfeat, dtype=dtype)).sum()).backward()
    return [x.detach().double().numpy().reshape(-1) for x in (R, A, feat, p.grad, n.grad, j.grad)]


POSES = {
    "zero": np.zeros(9),
    "tiny 1e-7": np.array([1e-7, -2e-7, 1.5e-7, -1e-7, 0.0, 1e-7, 2e-7, 1e-7, -1e-7]),
    "small 1e-4": np.array([1e-4, -2e-4, 3e-4, 2e-4, 1e-4, -1e-4, -3e-4, 2e-4, 1e-4]),
    "random": None,
    "near pi": None,
    "near 2 pi": None,
}


@pytest.mark.parametrize("case", list(POSES))
def test_joint_stage_vs_float64(shim, case):
    rs = np.random.RandomState(abs(hash(case)) % 2 ** 31)
    pose9 = POSES[case]
    if pose9 is None:
        ax = rs.randn(3, 3)
        ax /= np.linalg.norm(ax, axis=1, keepdims=True)
        ang = {"random": rs.uniform(0.1, 1.5, 3), "near pi": np.pi - np.array([1e-3, 0.0, -1e-3]),
               "near 2 pi": 2 * np.pi - np.array([1e-3, 0.0, -1e-3])}[case]
        pose9 = (ax * ang[:, None]).reshape(-1)
    pose = np.concatenate([pose9[:3], pose9[6:9]]).astype(np.float32)
    neck = pose9[3:6].astype(np.float32)
    J = (rs.randn(15) * 0.05).astype(np.float32)
    parents = (-1, 0, 1, 1, 1)
    dA, dfeat = rs.randn(60).astype(np.float32), rs.randn(36).astype(np.float32)
    got = _run_shim(shim, pose, neck, J, parents, dA, dfeat)
    ref = _torch(pose, neck, J, parents, dA, dfeat, torch.float64)
    aten = _torch(pose, neck, J, parents, dA, dfeat, torch.float32)
    names = ("R", "A", "feat", "dpose", "dneck", "dJ")
    U = 2.0 ** -24
    for nm, g, r, t in zip(names, got, ref, aten):
        assert np.isfinite(g).all(), (case, nm)
        # smplx's fp32 sequence itself loses accuracy where 1 - cos(angle) rounds away (small angles): the product must be
        # no further from float64 than ATen running that sequence in fp32, within a factor of 4, or within a few ulps
        e_native, e_aten = float(np.abs(g - r).max()), float(np.abs(t - r).max())
        floor = 64 * U * float(np.abs(r).max() + 1.0)
        print(f"[{case}] {nm}: max |native - f64| = {e_native:.3e}, max |ATen fp32 - f64| = {e_aten:.3e}")
        assert e_native <= 4 * e_aten + floor, (case, nm, e_native, e_aten)
    if case == "zero":
        np.testing.assert_array_equal(got[0], np.tile(np.eye(3, dtype=np.float32).reshape(-1), 5))

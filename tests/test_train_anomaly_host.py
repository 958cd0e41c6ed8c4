"""CPU: anomaly detection of the native trainers (the reference's train.py --detect_anomaly).  The header's anomaly structs,
ids and the two appended frame fields against the ctypes mirror; the record key's encoding and its decoding into stage,
tensor and (channel, y, x), (vertex, coordinate) or (mesh, face, splat); gms_nan_scan's refusals before any launch; the
trainers' defaults, their refusal of data parallel, and what a step does when the record names a NaN.  The scan and the
frames' hooks are checked on the GPU (test_gpu_train_anomaly.py)."""
import ctypes
import inspect
import os
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from gms_b200 import _lib, anomaly, scenes
from gms_b200.anomaly import AnomalyError, AnomalyRecord, Layout
from gms_b200.model import FreeGaussianModel, MeshGaussianModel
from gms_b200.trainer import FlameTrainer, FreeOptimizationParams, FreeTrainer, MeshTrainer, NativeFreeFrame
from helpers import random_gaussians

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDS = ["NONE", "LOSS", "COMPOSITE_BWD", "PREPROCESS_BWD", "EXPAND_BWD", "ACTIVATION_BWD", "FLAME_BWD", "STAGES", "DIMAGE", "DGEOM",
       "DMEANS3D", "DSCALES", "DROTATIONS", "DOPACITY_RAW", "DSHS", "DCOLOR_SH", "DVERTICES", "DALPHA_RAW", "DSCALE_RAW",
       "DSCALING_RAW", "DROTATION_RAW", "ACCUM", "DSHAPE", "DEXPRESSION", "DPOSE", "DNECK_POSE", "DTRANSL", "DENLARGEMENT"]


def test_header_structs_fields_and_ids_match_the_mirror(tmp_path):
    structs = {"gms_nan_buffer": _lib.NanBuffer, "gms_nan_scan_args": _lib.NanScanArgs, "gms_frame_args": _lib.FrameArgs,
               "gms_free_frame_args": _lib.FreeFrameArgs}
    body = "".join(f'    printf("{n} %zu\\n", sizeof({n}));\n' for n in structs)
    body += "".join(f'    printf("{n}.{f[0]} %zu\\n", offsetof({n}, {f[0]}));\n' for n, cls in structs.items() for f in cls._fields_)
    body += "".join(f'    printf("GMS_ANOMALY_{i} %llu\\n", (unsigned long long)GMS_ANOMALY_{i});\n' for i in IDS)
    body += '    printf("GMS_NAN_SCAN_MAX_BUFFERS %d\\n", GMS_NAN_SCAN_MAX_BUFFERS);\n'
    src = tmp_path / "anomaly.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gms_b200.h"\nint main(void) {\n' + body + "    return 0;\n}\n")
    exe = tmp_path / "anomaly"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict((l.split()[0], int(l.split()[1])) for l in subprocess.check_output([str(exe)], text=True).strip().split("\n"))
    for n, cls in structs.items():
        assert got[n] == ctypes.sizeof(cls), n
        for f in cls._fields_:
            assert got[f"{n}.{f[0]}"] == getattr(cls, f[0]).offset, (n, f[0])
    # gms_free_frame_args: appended; gms_frame_args: right before alpha_activation, which stays its trailing field
    assert [f[0] for f in _lib.FreeFrameArgs._fields_][-2:] == ["anomaly", "anomaly_stages"]
    assert [f[0] for f in _lib.FrameArgs._fields_][-4:] == ["n_segments", "anomaly_stages", "anomaly", "alpha_activation"]
    for i in IDS:
        assert got[f"GMS_ANOMALY_{i}"] == getattr(_lib, f"ANOMALY_{i}"), i
    assert got["GMS_NAN_SCAN_MAX_BUFFERS"] == _lib.NAN_SCAN_MAX_BUFFERS
    assert len(anomaly.STAGE_NAMES) == _lib.ANOMALY_STAGES


def test_keys_round_trip_and_order_by_stage_tensor_index():
    rng = np.random.default_rng(0)
    keys = []
    for _ in range(200):
        s, t, i = int(rng.integers(0, 6)), int(rng.integers(0, 256)), int(rng.integers(0, 1 << 48))
        k = anomaly.encode(s, t, i)
        assert anomaly.decode(k) == (s, t, i)
        assert anomaly.decode(k - (1 << 64) if k >= 1 << 63 else k) == (s, t, i)     # as the int64 word reads back
        keys.append(((s, t, i), k))
    assert sorted(keys) == sorted(keys, key=lambda x: x[1]), "the smallest key is the earliest stage, tensor, index"
    assert anomaly.decode(_lib.ANOMALY_NONE) is None and anomaly.decode(-1) is None
    for bad in ((6, 0, 0), (0, 256, 0), (0, 0, 1 << 48), (-1, 0, 0)):
        with pytest.raises(ValueError):
            anomaly.encode(*bad)


def _rows_numpy(segments):
    """(mesh, face, splat) of every Gaussian row, restated: mesh i's F_i x K_i block, face-major."""
    return np.concatenate([np.stack([np.full(F * K, i), np.repeat(np.arange(F), K), np.tile(np.arange(K), F)], 1)
                           for i, (F, K) in enumerate(segments)])


@pytest.mark.parametrize("segments", [[(7, 3)], [(5, 2), (3, 4), (4, 5)], [(1, 1), (2, 7), (1, 16)]])
def test_gaussian_rows_map_to_mesh_face_splat(segments):
    want = _rows_numpy(segments)
    for row in range(want.shape[0]):
        assert anomaly.gaussian_of(row, segments) == tuple(int(x) for x in want[row])
    with pytest.raises(ValueError):
        anomaly.gaussian_of(want.shape[0], segments)


def test_messages_name_every_part():
    lay = Layout(H=48, W=64, M=16, segments=[(5, 2), (3, 4)])
    e = AnomalyError(anomaly.encode(_lib.ANOMALY_LOSS, _lib.ANOMALY_DIMAGE, 2 * 48 * 64 + 7 * 64 + 9), lay, iteration=12)
    assert (e.stage, e.tensor, e.index) == (0, 0, 2 * 48 * 64 + 7 * 64 + 9)
    assert "Function 'loss' returned nan values" in str(e) and "dL/dimage" in str(e) and "channel 2, y 7, x 9" in str(e)
    assert "iteration 12" in str(e) and isinstance(e, RuntimeError)
    # dL/drotations of Gaussian 13 = mesh 1 (rows 10..21), face 0, splat 3; column 2
    e = AnomalyError(anomaly.encode(_lib.ANOMALY_PREPROCESS_BWD, _lib.ANOMALY_DROTATIONS, 13 * 4 + 2), lay)
    assert "preprocess backward" in str(e) and "dL/drotations" in str(e)
    assert "Gaussian 13, column 2 (mesh 1, face 0, splat 3)" in str(e)
    e = AnomalyError(anomaly.encode(_lib.ANOMALY_PREPROCESS_BWD, _lib.ANOMALY_DSHS, 3 * 48 + 47), lay)
    assert "Gaussian 3, column 47 (mesh 0, face 1, splat 1)" in str(e)
    e = AnomalyError(anomaly.encode(_lib.ANOMALY_COMPOSITE_BWD, _lib.ANOMALY_DGEOM, 12 * 9 + 5), lay)
    assert "per-Gaussian gradient records" in str(e) and "Gaussian 9, column 5 (mesh 0, face 4, splat 1)" in str(e)
    e = AnomalyError(anomaly.encode(_lib.ANOMALY_EXPAND_BWD, _lib.ANOMALY_DVERTICES, 3 * 17 + 1), lay)
    assert "expansion backward" in str(e) and "d_vertices" in str(e) and "vertex 17, coordinate 1" in str(e)
    flame = Layout(H=48, W=64, segments=[(5, 10)], meshes=False)
    e = AnomalyError(anomaly.encode(_lib.ANOMALY_EXPAND_BWD, _lib.ANOMALY_DALPHA_RAW, 3 * 23), flame)
    assert "Gaussian 23, column 0 (face 2, splat 3)" in str(e)
    e = AnomalyError(anomaly.encode(_lib.ANOMALY_FLAME_BWD, _lib.ANOMALY_DPOSE, 4), flame)
    assert "FLAME backward" in str(e) and "d_pose" in str(e) and "element 4" in str(e)
    free = Layout(H=48, W=64, scale_cols=2)
    e = AnomalyError(anomaly.encode(_lib.ANOMALY_ACTIVATION_BWD, _lib.ANOMALY_DSCALING_RAW, 2 * 40 + 1), free)
    assert "activation backward" in str(e) and "d_scaling_raw" in str(e) and str(e).endswith("Gaussian 40, column 1")
    e = AnomalyError(anomaly.encode(_lib.ANOMALY_ACTIVATION_BWD, _lib.ANOMALY_ACCUM, 40), free)
    assert "accum" in str(e) and str(e).endswith("Gaussian 40, column 0")


def _scan(**kw):
    a = _lib.NanScanArgs()
    a.n_buffers, a.stage, a.record = 1, 0, 0x1000       # never dereferenced: every call below is refused before a launch
    a.buffers[0].ptr, a.buffers[0].n, a.buffers[0].tensor = 0x2000, 16, 0
    for k, v in kw.items():
        if k.startswith("b_"):
            setattr(a.buffers[0], k[2:], v)
        else:
            setattr(a, k, v)
    return _lib.lib().gms_nan_scan(ctypes.byref(a), None)


@pytest.mark.parametrize("bad", [dict(record=None), dict(b_n=-1), dict(b_n=1 << 48), dict(n_buffers=_lib.NAN_SCAN_MAX_BUFFERS + 1),
                                 dict(n_buffers=-1), dict(b_ptr=None), dict(b_ptr=0x2002), dict(stage=-1),
                                 dict(stage=_lib.ANOMALY_STAGES), dict(b_tensor=256), dict(b_tensor=-1)])
def test_nan_scan_refuses_before_any_launch(bad):
    n0 = _lib.launch_count()
    assert _scan(**bad) == _lib.GMS_E_ARG
    assert "gms_nan_scan" in _lib.lib().gms_last_error().decode()
    assert _lib.launch_count() == n0
    assert _lib.lib().gms_nan_scan(None, None) == _lib.GMS_E_ARG


@pytest.mark.parametrize("fn", [MeshTrainer.__init__, FreeTrainer.__init__, FlameTrainer.__init__])
def test_detect_anomaly_defaults_to_off(fn):
    assert inspect.signature(fn).parameters["detect_anomaly"].default is False


def _mesh_model():
    m = MeshGaussianModel()
    m._adopt_params(scenes.init_mesh_gaussians(*scenes.icosphere(1, 0.8), K=2, seed=1), "cpu", 3, packed_features=True)
    return m


def _free_model():
    g = random_gaussians(64, seed=5, extent=0.8, flat_frac=0.0)
    return FreeGaussianModel(g["means3D"], torch.log(g["scales"]), g["rotations"], g["shs"], torch.logit(g["opacities"]), "gs", "cpu", 3)


def test_trainers_refuse_data_parallel_anomaly_detection():
    with pytest.raises(ValueError, match="detect_anomaly needs one GPU"):
        MeshTrainer(_mesh_model(), torch.zeros(3), world=2, rank=0, native=True, detect_anomaly=True)
    with pytest.raises(ValueError, match="detect_anomaly needs one GPU"):
        FreeTrainer(_free_model(), torch.zeros(3), 1.0, world=2, detect_anomaly=True)


class _Frame:
    """Stands in for a training frame: records run()'s keyword arguments, adds to the statistics as the real frame does,
    and writes `key` (when set) into the record it is handed."""
    W = H = 1 << 14
    last_num_rendered = 0
    dev = torch.device("cpu")

    def __init__(self, P, key=None):
        self.calls, self.key = [], key
        self.loss = torch.zeros(3)
        self.accum, self.denom = torch.zeros(P), torch.zeros(P)

    def run(self, cam, gt, bg, **kw):
        self.calls.append(kw)
        self.accum += 1.0
        self.denom += 1.0
        if self.key is not None and kw.get("anomaly") is not None:
            kw["anomaly"].word[0] = self.key - (1 << 64) if self.key >= 1 << 63 else self.key
        return self.loss[0]


def _cam():
    return SimpleNamespace(image_width=64, image_height=48, uid=0)


def test_frames_hand_the_record_and_stages_to_the_library():
    fr = object.__new__(NativeFreeFrame)
    m = _free_model()
    fr.model, fr.lam, fr.dev = m, 0.2, torch.device("cpu")
    fr.ev_loss = SimpleNamespace(cuda_event=None)
    fr.loss = torch.zeros(3)
    fr._check = lambda gt, bg, cam: None
    seen = []
    fr._launch = lambda fn, a, cam, bg, **kw: seen.append((a.anomaly, a.anomaly_stages))
    for n in m.NAMES:
        getattr(m, n).grad = torch.zeros_like(getattr(m, n))
    fr.run(_cam(), torch.zeros(3, 48, 64), torch.zeros(3), stats=False)
    rec = AnomalyRecord("cpu")
    fr.run(_cam(), torch.zeros(3, 48, 64), torch.zeros(3), stats=False, anomaly=rec, anomaly_stages=1 << _lib.ANOMALY_LOSS)
    assert seen == [(None, 0), (rec.ptr, 1)]


@pytest.mark.parametrize("detect", [False, True])
def test_clean_step_passes_the_record_and_unfuses_the_sh_step(detect):
    ft = FreeTrainer(_free_model(), torch.zeros(3), 1.0, FreeOptimizationParams(iterations=1), detect_anomaly=detect,
                     generator=torch.Generator().manual_seed(0))
    ft.frame = _Frame(64)
    ft.step(_cam(), torch.zeros(3, 48, 64), before_update=lambda: None)
    kw = ft.frame.calls[-1]
    assert (kw["anomaly"] is not None) is detect and kw["sh_adam"] is None
    assert ft.iteration == 1 and "detect_anomaly" not in ft.state_dict()
    mt = MeshTrainer(_mesh_model(), torch.zeros(3), native=True, optimizer_step=False, detect_anomaly=detect)
    mt._frame = _Frame(1)
    mt.step(_cam(), torch.zeros(3, 48, 64))
    assert (mt._frame.calls[-1]["anomaly"] is not None) is detect


def test_anomalous_step_raises_and_leaves_the_state_as_it_was():
    ft = FreeTrainer(_free_model(), torch.zeros(3), 1.0, FreeOptimizationParams(iterations=100), detect_anomaly=True,
                     generator=torch.Generator().manual_seed(0))
    key = anomaly.encode(_lib.ANOMALY_PREPROCESS_BWD, _lib.ANOMALY_DOPACITY_RAW, 5)
    ft.frame = _Frame(64, key)
    ft.frame.accum.fill_(0.5)
    before = ft.state_dict()
    ft.adam.g.fill_(3.0)
    calls = []
    with pytest.raises(AnomalyError, match=r"preprocess backward.*dL/dopacity_raw.*iteration 1: first at flat index 5, "
                                           r"Gaussian 5, column 0") as e:
        ft.step(_cam(), torch.zeros(3, 48, 64), before_update=lambda: calls.append(1))
    assert (e.value.stage, e.value.tensor, e.value.index) == (_lib.ANOMALY_PREPROCESS_BWD, _lib.ANOMALY_DOPACITY_RAW, 5)
    assert calls == [], "the error comes before before_update"
    after = ft.state_dict()
    assert ft.iteration == 0 and after["iteration"] == 0
    for k in ("accum", "denom", "generator"):
        assert torch.equal(after[k], before[k]), k
    for k in ("p", "m", "v"):
        assert torch.equal(after["adam"][k], before["adam"][k]), k
    assert after["adam"]["steps"] == before["adam"]["steps"]
    assert not bool(ft.adam.g.any()), "the step's gradients are discarded"

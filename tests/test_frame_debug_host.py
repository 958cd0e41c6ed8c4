"""CPU: debug mode of the native trainers (the reference's pipe.debug, train.py --debug and --debug_from).  The trainers'
defaults and their refusal of data parallel; the steps whose frame runs with settings.debug under the reference's rule; a
failing debug step, which writes the snapshot, prints the reference's message, re-raises and leaves the state as it was;
the header's GMS_E_DEBUG, check ids and gms_debug_bins_args against the ctypes mirror; gms_debug_check_bins's refusals
before any launch.  The frames' debug launches and the binning check itself run on the GPU (test_gpu_frame_debug.py)."""
import contextlib
import ctypes
import inspect
import os
import subprocess
from types import SimpleNamespace

import pytest
import torch

from gms_b200 import _lib, capacity, debug, scenes
from gms_b200.model import FreeGaussianModel, MeshGaussianModel
from gms_b200.trainer import FlameTrainer, FreeOptimizationParams, FreeTrainer, MeshTrainer, NativeFreeFrame
from helpers import random_gaussians

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mesh_model():
    m = MeshGaussianModel()
    m._adopt_params(scenes.init_mesh_gaussians(*scenes.icosphere(1, 0.8), K=2, seed=1), "cpu", 3, packed_features=True)
    return m


def _free_model():
    g = random_gaussians(64, seed=5, extent=0.8, flat_frac=0.0)
    return FreeGaussianModel(g["means3D"], torch.log(g["scales"]), g["rotations"], g["shs"], torch.logit(g["opacities"]), "gs", "cpu", 3)


class _Frame:
    """Stands in for a training frame: records run()'s `debug`, adds to the statistics as the real frame does, and raises
    `error` (when set) as a library refusal would."""
    W = H = 1 << 14
    last_num_rendered = 0
    dev = torch.device("cpu")

    def __init__(self, P, error=None):
        self.debug, self.error = [], error
        self.loss = torch.zeros(3)
        self.accum, self.denom = torch.zeros(P), torch.zeros(P)

    def run(self, cam, gt, bg, **kw):
        self.debug.append(kw["debug"])
        self.accum += 1.0
        self.denom += 1.0
        if self.error is not None:
            raise self.error
        return self.loss[0]

    def resize(self):
        pass


def _cam():
    return scenes.Camera(64, 48, 0.9, 0.7, torch.eye(4), torch.eye(4), torch.zeros(3), uid=0)


def _free_trainer(**kw):
    # iterations=1: no Adam step on any iteration (FlatAdam's kernels need a device)
    ft = FreeTrainer(_free_model(), torch.zeros(3), 1.0, FreeOptimizationParams(iterations=1), generator=torch.Generator().manual_seed(0),
                     **kw)
    ft.frame = _Frame(64)
    return ft


def _mesh_trainer(**kw):
    mt = MeshTrainer(_mesh_model(), torch.zeros(3), native=True, optimizer_step=False, **kw)
    mt._frame = _Frame(1)
    return mt


def _frame(tr):
    return tr._frame if isinstance(tr, MeshTrainer) else tr.frame


@pytest.mark.parametrize("fn", [MeshTrainer.__init__, FreeTrainer.__init__, FlameTrainer.__init__])
def test_trainer_defaults_are_off(fn):
    p = inspect.signature(fn).parameters
    assert p["debug"].default is False and p["debug_from"].default == -1 and p["debug_snapshot"].default == "snapshot_frame.dump"


def test_trainers_refuse_data_parallel_debug():
    with pytest.raises(ValueError, match="debug needs one GPU"):
        MeshTrainer(_mesh_model(), torch.zeros(3), world=2, rank=0, native=True, debug=True)
    with pytest.raises(ValueError, match="debug needs one GPU"):
        MeshTrainer(_mesh_model(), torch.zeros(3), world=2, rank=0, native=True, debug_from=5)
    with pytest.raises(ValueError, match="debug needs one GPU"):
        FreeTrainer(_free_model(), torch.zeros(3), 1.0, world=2, debug=True)


@pytest.mark.parametrize("make", [_free_trainer, _mesh_trainer])
@pytest.mark.parametrize("kw, on", [(dict(debug=True), [1] * 6), (dict(debug_from=0), [1] * 6), (dict(debug_from=3), [0, 0, 0, 1, 1, 1]),
                                    (dict(debug_from=-1), [0] * 6), (dict(), [0] * 6)])
def test_debug_bit_follows_the_reference_rule(make, kw, on, tmp_path):
    tr = make(debug_snapshot=str(tmp_path / "s.dump"), **kw)
    for _ in range(6):
        tr.step(_cam(), torch.zeros(3, 48, 64))
    assert _frame(tr).debug == [bool(b) for b in on]
    assert "debug" not in tr.state_dict() and "debug_from" not in tr.state_dict()
    assert not (tmp_path / "s.dump").exists()


def test_a_run_resumed_past_debug_from_never_turns_debug_on(tmp_path):
    ft = _free_trainer(debug_from=3, debug_snapshot=str(tmp_path / "s.dump"))
    state = ft.state_dict()
    state["iteration"] = 5
    ft.load_state_dict(state)
    for _ in range(3):
        ft.step(_cam(), torch.zeros(3, 48, 64))
    assert ft.frame.debug == [False] * 3 and ft.iteration == 8


def test_evaluate_uses_the_current_setting(monkeypatch):
    seen = []
    monkeypatch.setattr("gms_b200.trainer.renderer_set",
                        lambda rs, cls, model, P: SimpleNamespace(evaluate=lambda *a, **kw: seen.append(kw["debug"])))
    ft = _free_trainer(debug_from=1)
    ft.evaluate([], [])
    ft.step(_cam(), torch.zeros(3, 48, 64))
    ft.evaluate([], [])
    ft.step(_cam(), torch.zeros(3, 48, 64))
    ft.evaluate([], [])
    assert seen == [False, False, True]


def _equal(a, b):
    if torch.is_tensor(a):
        return torch.equal(a.cpu(), b.cpu())
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_equal(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    return a == b


@pytest.mark.parametrize("make", [_free_trainer, _mesh_trainer])
def test_failing_debug_step_writes_the_snapshot_prints_and_reraises(make, tmp_path, capsys):
    path = str(tmp_path / "snapshot_frame.dump")
    tr = make(debug=True, debug_snapshot=path)
    tr.step(_cam(), torch.zeros(3, 48, 64))
    msg = "gms_free_train_frame failed (code -5): binning check 1 (point list order) failed at list index 7, tile 3, Gaussian 2"
    _frame(tr).error = RuntimeError(msg)
    if isinstance(tr, FreeTrainer):
        tr.frame.accum.fill_(0.5)
    before = tr.state_dict()
    gt = torch.rand(3, 48, 64)
    with pytest.raises(RuntimeError, match="binning check 1"):
        tr.step(_cam(), gt, bg=torch.ones(3))
    out = capsys.readouterr().out
    assert f"An error occured in the training frame: {msg}. Please forward {path} for debugging." in out
    snap = torch.load(path, weights_only=False)
    assert _equal(snap["state_dict"], before), "the snapshot holds the state before the step, bit for bit"
    assert snap["trainer"] == type(tr).__name__ and snap["iteration"] == 2
    assert torch.equal(snap["gt"], gt) and torch.equal(snap["bg"], torch.ones(3))
    assert snap["camera"]["image_width"] == 64 and snap["camera"]["image_height"] == 48
    assert snap["active_sh_degree"] == tr.model.active_sh_degree and snap["antialiasing"] is False
    assert _equal(tr.state_dict(), before), "the trainer's state is as it was before the step"
    assert tr.iteration == 1


def test_frames_put_debug_into_the_settings(monkeypatch):
    """SyncFreeCapacity._launch, which every one-call frame calls: settings.debug is the call's `debug` and nothing else
    about the call changes."""
    seen = []

    def fake(a_ref, cb, user, stream):
        a = a_ref._obj
        seen.append((a.settings.debug, a.settings.antialiasing, a.binning_capacity))
        return 0
    monkeypatch.setattr(_lib, "lib", lambda: SimpleNamespace(gms_free_train_frame=fake))
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: SimpleNamespace(cuda_stream=None))
    fr = object.__new__(NativeFreeFrame)
    fr.model = SimpleNamespace(active_sh_degree=2)
    fr.dev, fr.ws, fr._cb = torch.device("cpu"), torch.zeros(16, dtype=torch.uint8), None
    fr.n_rendered, fr.sync_free, fr.capacity, fr._epoch, fr._view_epoch = ctypes.c_int64(0), False, 0, 0, {}
    t = torch.zeros(4)
    cam = SimpleNamespace(image_width=64, image_height=48, tanfovx=0.5, tanfovy=0.4, world_view_transform=t, full_proj_transform=t,
                          camera_center=t)
    for dbg in (False, True, False):
        fr._launch("gms_free_train_frame", _lib.FreeFrameArgs(), cam, t, antialiasing=True, debug=dbg)
    assert seen == [(0, 1, 0), (1, 1, 0), (0, 1, 0)]


def test_header_error_code_check_ids_and_args_match_the_mirror(tmp_path):
    cls, cname = _lib.DebugBinsArgs, "gms_debug_bins_args"
    body = f'    printf("size %zu\\n", sizeof({cname}));\n'
    body += "".join(f'    printf("{f[0]} %zu\\n", offsetof({cname}, {f[0]}));\n' for f in cls._fields_)
    ids = ["E_DEBUG", "DEBUG_ORDER", "DEBUG_RANGES", "DEBUG_GAUSSIAN", "DEBUG_SURVIVOR"]
    body += "".join(f'    printf("{i} %lld\\n", (long long)GMS_{i});\n' for i in ids)
    body += '    printf("DEBUG_NONE %llu\\n", (unsigned long long)GMS_DEBUG_NONE);\n'
    src = tmp_path / "dbg.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gms_b200.h"\nint main(void) {\n' + body + "    return 0;\n}\n")
    exe = tmp_path / "dbg"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict((l.split()[0], int(l.split()[1])) for l in subprocess.check_output([str(exe)], text=True).strip().split("\n"))
    assert got["size"] == ctypes.sizeof(cls)
    for f in cls._fields_:
        assert got[f[0]] == getattr(cls, f[0]).offset, f[0]
    assert got["E_DEBUG"] == _lib.GMS_E_DEBUG == -5
    for i in ids[1:]:
        assert got[i] == getattr(_lib, i), i
    assert got["DEBUG_NONE"] == _lib.DEBUG_NONE
    assert "gms_debug_check_bins" in _lib.ABI_SYMBOLS


def _valid_bins_args(keep):
    def buf(n, dtype=torch.int32):
        t = torch.zeros(max(n, 1), dtype=dtype)
        keep.append(t)
        return t.data_ptr()
    a = _lib.DebugBinsArgs()
    a.P, a.tiles_x, a.tiles_y, a.n = 4, 3, 2, 5
    a.point_list, a.ranges, a.radii, a.rect, a.depth_keys = buf(5), buf(12), buf(4), buf(8), buf(4)
    return a


@pytest.mark.parametrize("name, mutate", [
    ("null args", None),
    ("null point_list", lambda a: setattr(a, "point_list", None)),
    ("null ranges", lambda a: setattr(a, "ranges", None)),
    ("null radii", lambda a: setattr(a, "radii", None)),
    ("null rect", lambda a: setattr(a, "rect", None)),
    ("null depth keys", lambda a: setattr(a, "depth_keys", None)),
    ("P < 0", lambda a: setattr(a, "P", -1)),
    ("no tiles", lambda a: setattr(a, "tiles_x", 0)),
    ("too many tile rows", lambda a: setattr(a, "tiles_y", 65536)),
    ("n < 0", lambda a: setattr(a, "n", -1)),
    ("n >= 2^31", lambda a: setattr(a, "n", 1 << 31)),
    ("key bits", lambda a: (setattr(a, "tile_keys", a.point_list), setattr(a, "key_bits", 8))),
    ("surv without nsurv", lambda a: setattr(a, "surv", a.point_list)),
    ("nsurv without surv", lambda a: setattr(a, "nsurv", a.point_list)),
])
def test_check_bins_refuses_bad_arguments_before_any_launch(name, mutate):
    keep = []
    a = _valid_bins_args(keep)
    L = _lib.lib()
    n0 = _lib.launch_count()
    if mutate is None:
        rc = L.gms_debug_check_bins(None, None)
    else:
        mutate(a)
        rc = L.gms_debug_check_bins(ctypes.byref(a), None)
    assert rc == _lib.GMS_E_ARG, (name, L.gms_last_error())
    assert b"gms_debug_check_bins" in L.gms_last_error()
    assert _lib.launch_count() == n0


def test_mesh_trainer_refuses_debug_on_the_autograd_arms():
    for kw in (dict(native=False), dict(native=True, fast=False)):
        for dbg in (dict(debug=True), dict(debug_from=2)):
            with pytest.raises(ValueError, match="debug runs the native frame"):
                MeshTrainer(_mesh_model(), torch.zeros(3), **kw, **dbg)


def test_an_unwritable_snapshot_path_keeps_the_step_error(tmp_path, capsys):
    tr = _free_trainer(debug=True, debug_snapshot=str(tmp_path / "missing" / "dir" / "s.dump"))
    tr.frame.error = RuntimeError("gms_free_train_frame failed (code -5): binning check 3")
    with pytest.raises(RuntimeError, match="binning check 3"):
        tr.step(_cam(), torch.zeros(3, 48, 64))
    assert "The snapshot could not be written" in capsys.readouterr().out


@pytest.mark.parametrize("make", [_free_trainer, _mesh_trainer])
def test_snapshot_model_holds_structure_and_gradient_buffers(make):
    """The snapshot's model keeps no copy of the optimizer's parameters (they are in its state_dict()), and every tensor that
    had a gradient buffer gets a zero one back when it is rebuilt (a FlameGaussianModel's `vertices.grad`)."""
    import io
    tr = make()
    m = tr.model
    extra = torch.zeros(5, 3)
    extra.grad = torch.ones(5, 3)
    m.extra_with_grad = extra
    flat = tr._debug_flat()
    buf = io.BytesIO()
    torch.save(debug.model_structure(m, flat), buf)
    assert buf.getbuffer().nbytes < flat.numel() * 4 // 2, "the parameters are not serialised twice"
    back = debug.rebuild_model(torch.load(io.BytesIO(buf.getvalue()), weights_only=False), "cpu")
    for k, v in m.__dict__.items():
        if torch.is_tensor(v) and (v.untyped_storage().data_ptr() == flat.untyped_storage().data_ptr() or v.grad is not None):
            b = getattr(back, k)
            assert b.shape == v.shape and isinstance(b, torch.nn.Parameter) == isinstance(v, torch.nn.Parameter), k
            assert (b.grad is not None) == (v.grad is not None), k
    assert torch.equal(back.extra_with_grad.grad, torch.zeros(5, 3))

"""CPU: the antialiasing setting of the trainers (the reference's pipe.antialiasing).  It defaults to off everywhere; every
training frame a trainer runs (native or autograd arm) receives it, and the one-call frames put it into the settings
struct they launch with; state_dict() records it and load_state_dict() refuses a state written with the other setting
before it changes anything, naming both.  The frames' results with the flag on are checked on the GPU
(test_gpu_train_antialiasing.py)."""
import inspect
from types import SimpleNamespace

import pytest
import torch

from gms_b200 import scenes, trainer
from gms_b200.model import FreeGaussianModel, MeshGaussianModel
from gms_b200.trainer import (FlameTrainer, FreeOptimizationParams, FreeTrainer, MeshTrainer, NativeFrame, NativeFreeFrame,
                              check_antialiasing)
from helpers import random_gaussians


@pytest.mark.parametrize("fn", [MeshTrainer.__init__, FreeTrainer.__init__, FlameTrainer.__init__, NativeFrame.run,
                                NativeFreeFrame.run])
def test_antialiasing_defaults_to_off(fn):
    assert inspect.signature(fn).parameters["antialiasing"].default is False


def _free_trainer(antialiasing, iterations=30_000):
    g = random_gaussians(64, seed=5, extent=0.8, flat_frac=0.0)
    m = FreeGaussianModel(g["means3D"], torch.log(g["scales"]), g["rotations"], g["shs"], torch.logit(g["opacities"]), "gs",
                          "cpu", 3)
    return FreeTrainer(m, torch.zeros(3), 1.0, FreeOptimizationParams(iterations=iterations), antialiasing=antialiasing,
                       generator=torch.Generator().manual_seed(0))


def _mesh_trainer(antialiasing, native):
    m = MeshGaussianModel()
    m._adopt_params(scenes.init_mesh_gaussians(*scenes.icosphere(1, 0.8), K=2, seed=1), "cpu", 3, packed_features=True)
    return MeshTrainer(m, torch.zeros(3), native=native, optimizer_step=False, antialiasing=antialiasing)


class _Frame:
    """Stands in for a training frame: records the keyword arguments of run()."""
    W = H = 1 << 14
    last_num_rendered = 0

    def __init__(self):
        self.calls = []
        self.loss = torch.zeros(3)

    def run(self, cam, gt, bg, **kw):
        self.calls.append(kw)
        return self.loss[0]


def _cam(W=64, H=48):
    return SimpleNamespace(image_width=W, image_height=H, uid=0)


@pytest.mark.parametrize("aa", [False, True])
def test_trainers_hand_their_setting_to_every_frame(aa, monkeypatch):
    ft = _free_trainer(aa, iterations=1)
    ft.frame = _Frame()
    ft.step(_cam(), torch.zeros(3, 48, 64), before_update=lambda: None)
    assert ft.frame.calls[-1]["antialiasing"] is aa
    mt = _mesh_trainer(aa, native=True)
    mt._frame = _Frame()
    mt.step(_cam(), torch.zeros(3, 48, 64))
    assert mt._frame.calls[-1]["antialiasing"] is aa
    seen = []

    def fake_render_frame(model, cam, bg, fused=True, antialiasing=False):
        seen.append(antialiasing)
        raise StopIteration

    monkeypatch.setattr(trainer, "render_frame", fake_render_frame)
    with pytest.raises(StopIteration):
        _mesh_trainer(aa, native=False).step(_cam(), torch.zeros(3, 48, 64))
    assert seen == [aa]


@pytest.mark.parametrize("aa", [False, True])
def test_free_frame_launches_with_the_flag(aa):
    """NativeFreeFrame.run passes the flag to the shared launch, which writes it into the settings struct (0 or 1)."""
    fr = object.__new__(NativeFreeFrame)
    ft = _free_trainer(aa)
    fr.model, fr.lam, fr.dev = ft.model, 0.2, torch.device("cpu")
    fr.ev_loss = SimpleNamespace(cuda_event=None)
    fr.loss = torch.zeros(3)
    fr._check = lambda gt, bg, cam: None
    launched = []
    fr._launch = lambda fn, a, cam, bg, **kw: launched.append((fn, kw))
    fr.run(_cam(), torch.zeros(3, 48, 64), torch.zeros(3), stats=False, antialiasing=aa)
    assert launched == [("gms_free_train_frame", {"antialiasing": aa})]


def test_state_records_the_setting_and_a_mismatch_is_refused_untouched():
    on, off = _free_trainer(True), _free_trainer(False)
    s_on, s_off = on.state_dict(), off.state_dict()
    assert s_on["antialiasing"] is True and s_off["antialiasing"] is False
    before = off.adam.p.clone()
    with torch.no_grad():
        on.adam.p.add_(1.0)
    s_on = on.state_dict()
    with pytest.raises(ValueError, match=r"FreeTrainer\.load_state_dict: the state was trained with antialiasing=True, "
                                         r"but this trainer runs antialiasing=False"):
        off.load_state_dict(s_on)
    assert torch.equal(off.adam.p, before), "a refused state changes nothing"
    with pytest.raises(ValueError, match=r"antialiasing=False.*antialiasing=True"):
        on.load_state_dict(s_off)
    fresh = _free_trainer(True)
    fresh.load_state_dict(s_on)
    assert torch.equal(fresh.adam.p, on.adam.p) and fresh.antialiasing


def test_a_state_without_the_entry_trained_without_antialiasing():
    """States written before the setting was recorded (checkpoints of earlier runs) were all trained without it."""
    check_antialiasing({"adam": {}}, False, "MeshTrainer")
    with pytest.raises(ValueError, match=r"MeshTrainer\.load_state_dict: .*antialiasing=False.*antialiasing=True"):
        check_antialiasing({"adam": {}}, True, "MeshTrainer")
    old = _free_trainer(False).state_dict()
    del old["antialiasing"]
    _free_trainer(False).load_state_dict(old)
    with pytest.raises(ValueError, match="antialiasing"):
        _free_trainer(True).load_state_dict(old)

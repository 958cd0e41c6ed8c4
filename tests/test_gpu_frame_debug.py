"""-m gpu: debug mode of the one-call frames and the native trainers (the reference's pipe.debug).

Checked here: a training frame run with settings.debug equals the same frame without it (image, radii and inverse depth
bit for bit, the loss to 2e-6, the gradients within the spread bound) for gs_mesh, gs_multi_mesh, gs_flame, gs and gs_flat
at SH degrees 0 and 3, antialiasing off and on, with and without the anomaly record, and issues the same launches plus the
three binning check launches; all five render frames likewise plus two; the check stays silent on clean frames under every
binning and sort option, with tile keys wider than 16 bits, on the 34 scenes of raster_edge_cases, the parity scenes and
BASELINE configs 2-5 at their sizes; gms_debug_check_bins reports each invariant broken on a hand-built list at its own
check and index; a trainer loop with debug_from=3 follows a loop without debug; a failing debug step of gs_flat, gs_flame
and gs_multi_mesh writes a snapshot that debug.replay repeats.  No test provokes a device fault."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

import bench
import mesh_types_cases
import raster_edge_cases as E
from gms_b200 import _lib, dataset, debug, io_ply, scenes
from gms_b200.anomaly import AnomalyRecord
from gms_b200.flame import NativeFlame
from gms_b200.model import (FlameCheckpoint, FlameGaussianModel, FreeGaussianModel, MeshGaussianModel, MultiMeshGaussianModel,
                            PointsModel)
from gms_b200.render import FlameRenderer, MeshBoundPointsRenderer, NativeFreeRenderer, NativeRenderer, PointsRenderer
from gms_b200.trainer import FlameOptimizationParams, FlameTrainer, FreeOptimizationParams, FreeTrainer, MeshTrainer
from helpers import random_gaussians, settings_from_camera

pytestmark = pytest.mark.gpu

TYPES = ["gs_mesh", "gs_multi_mesh", "gs_flame", "gs", "gs_flat"]
MESH_TYPES = ("gs_mesh", "gs_multi_mesh")
W, H = 256, 144
BG = (0.2, 0.5, 0.9)
# the sync-free / atomics spread bound of the frame tests (test_gpu_train_mixed_sizes), max |diff| / max |grad| per tensor
BOUND = {"_xyz": 1.5e-4, "_scaling": 4e-3, "_rotation": 1.5e-3, "_opacity": 1e-6, "_features": 1e-6, "vertices": 4e-3, "_alpha": 4e-3,
         "_scale": 4e-3, "_scales": 4e-3}
CHECKS = 3          # binning check launches of a training frame: ranges, list, survivor lists


def _model(gs_type, degree=3, multi_K=(2, 4, 5)):
    if gs_type == "gs_mesh":
        m = MeshGaussianModel.from_params(scenes.init_mesh_gaussians(*scenes.icosphere(3, 0.8), K=3, seed=1), "cuda", packed_features=True)
    elif gs_type == "gs_multi_mesh":
        p = []
        for i, K in enumerate(multi_K):
            v, f = scenes.icosphere(2 if i == 0 else 1, 0.7 / (i + 1))
            p.append(scenes.init_mesh_gaussians(v + np.array([0.3 * i, -0.1 * i, 0.2 * i]), f, K=K, seed=2 + i))
        m = MultiMeshGaussianModel.from_mesh_params(p, "cuda", packed_features=True)
    elif gs_type == "gs_flame":
        init = dataset.flame_init(mesh_types_cases.FLAME_MODEL)
        m = FlameGaussianModel.create(NativeFlame.from_model_file(mesh_types_cases.FLAME_MODEL), init.faces, K=60, seed=4)
    else:
        g = random_gaussians(3000, seed=5, extent=0.8, flat_frac=0.0)
        s = torch.log(g["scales"])
        m = FreeGaussianModel(g["means3D"], (s[:, 1:] if gs_type == "gs_flat" else s).contiguous(), g["rotations"], g["shs"],
                              torch.logit(g["opacities"]), gs_type, "cuda", 3)
    m.active_sh_degree = degree
    return m


def _trainer(gs_type, model, aa=False, **kw):
    bg = torch.tensor(BG, device="cuda")
    if gs_type in MESH_TYPES:
        return MeshTrainer(model, bg, 0.2, native=True, antialiasing=aa, **kw)
    if gs_type == "gs_flame":
        return FlameTrainer(model, bg, FlameOptimizationParams(iterations=1000), antialiasing=aa, **kw)
    return FreeTrainer(model, bg, 1.0, FreeOptimizationParams(iterations=1000, densify_from_iter=10 ** 9), antialiasing=aa, **kw)


def _names(gs_type):
    if gs_type in MESH_TYPES:
        return ("vertices", "_alpha", "_scale", "_features", "_opacity")
    if gs_type == "gs_flame":
        return FlameGaussianModel.FLAME_NAMES + ("_alpha", "_scales", "_features", "_opacity")
    return FreeGaussianModel.NAMES


def _views(n=3, seed=0):
    cams, gts = [], []
    g = torch.Generator().manual_seed(seed)
    for k, c in enumerate(scenes.ring_cameras(n, 2.6, W, H, phase=0.3)):
        c.uid = ("view", k)
        cams.append(c.to("cuda"))
        gts.append(torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8).cuda())
    return cams, gts


def _frame_once(tr, gs_type, cam, gt, dbg, anomaly):
    """One frame of the trainer's native frame (no optimizer step): its outputs, its gradients and its launches."""
    fr = tr.native_frame
    opt = tr.opt if gs_type in MESH_TYPES else tr.adam
    opt.zero_grad()
    if gs_type == "gs_flame":
        tr.model.refresh_vertices()
    kw = dict(antialiasing=tr.antialiasing, debug=dbg)
    if anomaly:
        kw["anomaly"] = AnomalyRecord(fr.dev).reset()
    if gs_type not in MESH_TYPES and gs_type != "gs_flame":
        kw["stats"] = False
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    fr.run(cam, gt, tr.bg, **kw)
    torch.cuda.synchronize()
    launches = _lib.launch_count() - n0
    out = debug.frame_outputs(fr, cam)
    out["grads"] = {n: getattr(tr.model, n).grad.clone() for n in _names(gs_type)}
    return out, launches


def _assert_same(a, b, what):
    for k in ("image", "radii", "invdepth"):
        assert torch.equal(a[k], b[k]), (what, k)
    assert abs(float(a["loss"][0]) - float(b["loss"][0])) <= 2e-6 * abs(float(b["loss"][0])), what
    for n, g in b["grads"].items():
        scale = float(g.abs().max())
        assert float((a["grads"][n] - g).abs().max()) <= BOUND.get(n, 4e-3) * max(scale, 1e-30), (what, n)


@pytest.mark.parametrize("gs_type", TYPES)
@pytest.mark.parametrize("degree", [0, 3])
@pytest.mark.parametrize("aa", [False, True])
def test_debug_training_frame_equals_the_frame_without_it(gs_type, degree, aa):
    cams, gts = _views()
    tr = _trainer(gs_type, _model(gs_type, degree), aa)
    for v in range(len(cams)):           # every view learned its N; the frames below are sync-free
        tr.step(cams[v], gts[v])
    for anomaly in (False, True):
        for v in range(len(cams)):
            off, n_off = _frame_once(tr, gs_type, cams[v], gts[v], False, anomaly)
            on, n_on = _frame_once(tr, gs_type, cams[v], gts[v], True, anomaly)
            _assert_same(on, off, (gs_type, degree, aa, anomaly, v))
            assert n_on == n_off + CHECKS, (n_on, n_off)


def test_debug_adds_only_the_check_launches_per_kernel():
    cams, gts = _views()
    tr = _trainer("gs_mesh", _model("gs_mesh"))
    for v in range(len(cams)):
        tr.step(cams[v], gts[v])
    _lib.set_option("time_kernels", 1)
    try:
        counts = {}
        for dbg in (False, True):
            _lib.kernel_times(reset=True)
            _frame_once(tr, "gs_mesh", cams[0], gts[0], dbg, False)
            counts[dbg] = {k: n for k, (_, n) in _lib.kernel_times(reset=True).items()}
    finally:
        _lib.set_option("time_kernels", 0)
    for k in counts[False]:
        assert counts[True][k] == counts[False][k] + (CHECKS if k == "debug_check" else 0), k


@pytest.mark.parametrize("kind", ["mesh", "gs_flat"])
def test_debug_render_equals_the_render_without_it(kind):
    cams, _ = _views()
    bg = torch.tensor(BG, device="cuda")
    m = _model("gs_mesh" if kind == "mesh" else "gs_flat")
    r = (NativeRenderer if kind == "mesh" else NativeFreeRenderer)(m, W, H)
    for cam in cams:
        r.render(cam, bg)
    for cam in cams:
        for aa in (False, True):
            n0 = _lib.launch_count()
            ref = [t.clone() for t in r.render(cam, bg, antialiasing=aa)]
            n1 = _lib.launch_count()
            got = [t.clone() for t in r.render(cam, bg, antialiasing=aa, debug=True)]
            n2 = _lib.launch_count()
            for a, b in zip(got, ref):
                assert torch.equal(a, b)
            assert n2 - n1 == n1 - n0 + 2, "a render frame adds the ranges and list checks"


OPTIONS = [dict(), dict(bin_impl=1), dict(sort_impl=1), dict(key16=0), dict(bin_impl=1, sort_impl=1), dict(composite_fwd=3),
           dict(tile_order=0), dict(warp_emit=0)]


@pytest.mark.parametrize("opts", OPTIONS, ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()) or "default")
@pytest.mark.parametrize("gs_type", ["gs_flat", "gs_mesh"])
def test_check_is_silent_on_clean_frames_under_every_option(opts, gs_type):
    old = {k: _lib.set_option(k, v) for k, v in opts.items()}
    try:
        cams, gts = _views(4, seed=1)
        tr = _trainer(gs_type, _model(gs_type), debug=True)
        for v in range(len(cams)):
            tr.step(cams[v], gts[v])
        for v in range(len(cams)):           # sync-free frames
            tr.step(cams[v], gts[v])
    finally:
        for k, v in old.items():
            _lib.set_option(k, v)


def test_check_is_silent_with_wide_keys_on_a_large_grid():
    """More than 65535 tiles: 17-bit tile keys (32-bit key arrays)."""
    bg = torch.tensor(BG, device="cuda")
    m = _model("gs_flat")
    cam = scenes.ring_cameras(1, 2.6, 4400, 4400)[0].to("cuda")
    r = NativeFreeRenderer(m, 4400, 4400)
    ref = [t.clone() for t in r.render(cam, bg)]
    got = r.render(cam, bg, debug=True)
    for a, b in zip(got, ref):
        assert torch.equal(a, b)


# ---- gms_debug_check_bins on hand-built lists

GX, GY = 3, 2


def _clean_list():
    """Four Gaussians on a 3x2 tile grid, binned as the frames bin them: per tile in tile order, the Gaussians whose
    rectangle holds it in (depth key, index) order."""
    rect = np.array([[0, 0, 2, 1], [1, 0, 3, 2], [0, 1, 1, 2], [0, 0, 3, 2]], np.int64)        # x0, y0, x1, y1
    dkey = np.array([30, 10, 20, 10], np.uint32)
    radii = np.array([3, 4, 2, 9], np.int32)
    lst, keys, ranges = [], [], np.zeros((GX * GY, 2), np.int32)
    for t in range(GX * GY):
        tx, ty = t % GX, t // GX
        gs = sorted((int(dkey[g]), g) for g in range(4) if rect[g, 0] <= tx < rect[g, 2] and rect[g, 1] <= ty < rect[g, 3])
        ranges[t] = (len(lst), len(lst) + len(gs)) if gs else (0, 0)
        lst += [g for _, g in gs]
        keys += [t] * len(gs)
    packed = np.stack([rect[:, 0] | rect[:, 1] << 16, rect[:, 2] | rect[:, 3] << 16], 1).astype(np.uint32)
    # survivors: every quad keeps every second position of its tile's list
    n = len(lst)
    surv, nsurv = np.zeros(4 * n, np.uint32), np.zeros(4 * GX * GY, np.uint32)
    for t in range(GX * GY):
        x, y = ranges[t]
        for q in range(4):
            s = list(range(q % 2, y - x, 2))
            nsurv[4 * t + q] = len(s)
            surv[4 * x + q * (y - x): 4 * x + q * (y - x) + len(s)] = s
    return dict(point_list=np.array(lst, np.uint32), keys=np.array(keys, np.uint32), ranges=ranges, radii=radii, rect=packed, dkey=dkey,
                surv=surv, nsurv=nsurv)


def _check(d, key_bits=32):
    t = {k: torch.from_numpy(v.astype(np.int32) if v.dtype == np.uint32 else v).cuda() for k, v in d.items()}
    if key_bits == 16:
        t["keys"] = torch.from_numpy(d["keys"].astype(np.int16)).cuda()
    a = _lib.DebugBinsArgs()
    a.P, a.tiles_x, a.tiles_y, a.n = len(d["radii"]), GX, GY, len(d["point_list"])
    a.point_list, a.tile_keys, a.key_bits = t["point_list"].data_ptr(), t["keys"].data_ptr(), key_bits
    a.ranges, a.radii, a.rect, a.depth_keys = t["ranges"].data_ptr(), t["radii"].data_ptr(), t["rect"].data_ptr(), t["dkey"].data_ptr()
    a.surv, a.nsurv = t["surv"].data_ptr(), t["nsurv"].data_ptr()
    key = C.c_uint64(0)
    a.key = C.pointer(key)
    rc = _lib.lib().gms_debug_check_bins(C.byref(a), torch.cuda.current_stream().cuda_stream)
    return rc, int(key.value), _lib.lib().gms_last_error().decode()


@pytest.mark.parametrize("key_bits", [16, 32])
def test_check_bins_passes_a_clean_list(key_bits):
    rc, key, msg = _check(_clean_list(), key_bits)
    assert rc == _lib.GMS_OK and key == _lib.DEBUG_NONE, msg


def _swap(d):
    t = 3                                   # tile 3 holds Gaussians 3 (key 10), 2 (key 20): swap them
    x, y = d["ranges"][t]
    assert y - x == 2
    d["point_list"][[x, x + 1]] = d["point_list"][[x + 1, x]]
    return _lib.DEBUG_ORDER, x + 1


def _range_end(d):
    t = 1
    d["ranges"][t, 1] -= 1
    return _lib.DEBUG_RANGES, d["ranges"][t + 1, 0]


def _outside(d):
    t = 0                                   # Gaussian 2's rectangle is column 0, row 1: move tile 0's first entry to it
    x = d["ranges"][t, 0]
    d["point_list"][x] = 2
    return _lib.DEBUG_GAUSSIAN, x


def _index_beyond_P(d):
    x = d["ranges"][4, 0]
    d["point_list"][x] = 4
    return _lib.DEBUG_GAUSSIAN, x


def _survivor(d):
    t = 2
    x, y = d["ranges"][t]
    slot = 4 * x + 1 * (y - x)              # quad 1's first survivor
    d["surv"][slot] = y - x                  # one past its tile's range
    return _lib.DEBUG_SURVIVOR, slot


@pytest.mark.parametrize("corrupt", [_swap, _range_end, _outside, _index_beyond_P, _survivor])
def test_check_bins_reports_each_invariant_at_its_index(corrupt):
    d = _clean_list()
    check, index = corrupt(d)
    rc, key, msg = _check(d)
    assert rc == _lib.GMS_E_DEBUG, msg
    assert (key >> 56, key & ((1 << 56) - 1)) == (check, int(index)), msg
    assert f"binning check {check}" in msg and str(int(index)) in msg


# ---- trainers

@pytest.mark.parametrize("gs_type", ["gs_mesh", "gs_flat"])
def test_trainer_loop_with_debug_from_follows_the_loop_without(gs_type, tmp_path):
    cams, gts = _views(4, seed=2)
    runs = {}
    for dbg in (False, True):
        m = _model(gs_type)
        kw = dict(debug_from=3, debug_snapshot=str(tmp_path / "s.dump")) if dbg else {}
        if gs_type == "gs_flat":
            tr = FreeTrainer(m, torch.tensor(BG, device="cuda"), 1.0, FreeOptimizationParams(iterations=1000, densify_from_iter=4,
                             densification_interval=5, densify_grad_threshold=1e-7), generator=torch.Generator("cuda").manual_seed(0),
                             **kw)
        else:
            tr = _trainer(gs_type, m, **kw)
        for it in range(10):
            tr.step(cams[it % 4], gts[it % 4])
        runs[dbg] = {n: getattr(m, n).detach().clone() for n in _names(gs_type)}
        assert tr._debug.on is dbg
    for n, p in runs[False].items():
        assert p.shape == runs[True][n].shape, n          # a densifying run ends with the same P
        d = float((runs[True][n] - p).abs().max())
        assert d <= 1e-3 * max(float(p.abs().max()), 1.0), (n, d)
    assert not (tmp_path / "s.dump").exists()


@pytest.mark.parametrize("gs_type", ["gs_flat", "gs_flame", "gs_multi_mesh"])
def test_failing_debug_step_snapshot_replays(gs_type, tmp_path, capsys):
    path = str(tmp_path / "snapshot_frame.dump")
    cams, gts = _views(2, seed=3)
    m = _model(gs_type)
    tr = _trainer(gs_type, m, debug=True, debug_snapshot=path)
    tr.step(cams[0], gts[0])
    before = tr.state_dict()
    m.active_sh_degree = 5                  # refused by the frame before its first launch
    with pytest.raises(Exception, match="gms_free_train_frame|gms_train_frame") as e:
        tr.step(cams[1], gts[1])
    msg = str(e.value)
    assert f"An error occured in the training frame: {msg}. Please forward {path} for debugging." in capsys.readouterr().out
    after = tr.state_dict()
    for k in ("p", "m", "v"):
        assert torch.equal(after["adam"][k], before["adam"][k]), k
    assert after.get("iteration", tr.iteration) == tr.iteration == 1
    with pytest.raises(Exception, match=re.escape(msg)):
        debug.replay(path, snapshot=str(tmp_path / "replay.dump"))
    assert (tmp_path / "replay.dump").exists()
    snap = torch.load(path, weights_only=False)
    snap["active_sh_degree"] = 3
    snap["state_dict"]["active_sh_degree"] = 3
    fixed = str(tmp_path / "fixed.dump")
    torch.save(snap, fixed)
    got = debug.replay(fixed)
    m.active_sh_degree = 3
    tr.step(cams[1], gts[1])
    own = debug.frame_outputs(tr.native_frame, cams[1])
    assert torch.equal(got["image"], own["image"]) and torch.equal(got["radii"], own["radii"])
    assert abs(float(got["loss"]) - float(own["loss"][0])) <= 2e-6 * abs(float(own["loss"][0]))


# ---- the check on the scenes that reach the binning's edges, and on BASELINE's configurations

class _Options:
    def __init__(self, opts):
        self.opts = opts

    def __enter__(self):
        self.old = {k: _lib.set_option(k, v) for k, v in self.opts.items()}

    def __exit__(self, *exc):
        for k, v in self.old.items():
            _lib.set_option(k, v)


EDGE_OPTIONS = [dict(), dict(bin_impl=1), dict(sort_impl=1)]
OPT_IDS = ["default", "bin_impl=1", "sort_impl=1"]


def _scene_camera(S):
    return scenes.Camera(int(S.image_width), int(S.image_height), 2 * np.arctan(S.tanfovx), 2 * np.arctan(S.tanfovy),
                         torch.tensor(np.asarray(S.viewmatrix, np.float32)).cuda(), torch.tensor(np.asarray(S.projmatrix, np.float32)).cuda(),
                         torch.tensor(np.asarray(S.campos, np.float32)).cuda(), uid="scene")


def _silent_on_scene(S, g):
    """A gs model of the scene's Gaussians: two debug training steps (the first learns N, the second is sync-free) and a
    debug render equal to the render without debug."""
    m = FreeGaussianModel(g["means3D"].float(), torch.log(g["scales"].float()), g["rotations"].float(), g["shs"].float(),
                          torch.logit(g["opacities"].float()), "gs", "cuda", int(S.sh_degree))
    m.active_sh_degree = int(S.sh_degree)
    bg = torch.tensor(np.asarray(S.bg, np.float32)).cuda()
    cam = _scene_camera(S)
    W, H = cam.image_width, cam.image_height
    r = NativeFreeRenderer(m, W, H)
    ref = [t.clone() for t in r.render(cam, bg, antialiasing=bool(S.antialiasing))]
    got = [t.clone() for t in r.render(cam, bg, antialiasing=bool(S.antialiasing), debug=True)]
    for a, b in zip(got, ref):
        assert torch.equal(a, b)
    # iterations=1: no Adam step (the scenes' degenerate rows hold infinite raw parameters), the frames alone
    tr = FreeTrainer(m, bg, 1.0, FreeOptimizationParams(iterations=1, densify_from_iter=10 ** 9), antialiasing=bool(S.antialiasing),
                     debug=True)
    gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(0)).cuda()
    for _ in range(2):
        tr.step(cam, gt)


@pytest.mark.parametrize("opts", EDGE_OPTIONS, ids=OPT_IDS)
@pytest.mark.parametrize("name", list(E.CASES))
def test_check_is_silent_on_the_edge_scenes(name, opts):
    S, g = E.CASES[name]()
    with _Options(opts):
        _silent_on_scene(S, g)


PARITY = [(3000, 320, 208, -2.6), (20000, 400, 300, -2.6), (500, 64, 48, -2.6), (1, 32, 32, -2.6), (600, 640, 400, -0.8),
          (40000, 96, 64, -2.0), (400, 800, 608, -0.7), (5000, 1920, 1080, -2.4), (50000, 640, 480, -2.4)]


@pytest.mark.parametrize("opts", EDGE_OPTIONS, ids=OPT_IDS)
@pytest.mark.parametrize("P,W,H,mu", PARITY)
def test_check_is_silent_on_the_parity_scenes(P, W, H, mu, opts):
    cam = scenes.look_at_camera((2.8, 0.6, 1.1), (0, 0, 0), W, H)
    S = settings_from_camera(cam, bg=(0.1, 0.4, 0.8))
    with _Options(opts):
        _silent_on_scene(S, random_gaussians(P, seed=7, extent=1.2, scale_mu=mu))


def _config_model(name):
    params, cams, _ = bench.build_scene(name)
    return MeshGaussianModel.from_params(params, "cuda", packed_features=True, active_sh_degree=3), [c.to("cuda") for c in cams]


@pytest.mark.parametrize("opts", EDGE_OPTIONS, ids=OPT_IDS)
@pytest.mark.parametrize("name", ["gs_mesh_100k_800", "gs_mesh_1M_1080p", "gs_multi_mesh_2M_1080p", "gs_mesh_500k_1080p"])
def test_check_is_silent_on_the_baseline_configs(name, opts):
    """BASELINE configs 2-5 at their sizes: debug training frames on two views equal the frames without debug; config 5's
    animated-vertex sweep renders in debug mode equal to the renders without it."""
    m, cams = _config_model(name)
    bg = torch.ones(3, device="cuda")
    W, H = cams[0].image_width, cams[0].image_height
    gts = [torch.randint(0, 256, (H, W, 3), generator=torch.Generator().manual_seed(k), dtype=torch.uint8).cuda() for k in range(2)]
    with _Options(opts):
        tr = MeshTrainer(m, bg, 0.2, native=True)
        for v in range(2):
            tr.step(cams[v], gts[v])
        for v in range(2):
            off, _ = _frame_once(tr, "gs_mesh", cams[v], gts[v], False, False)
            on, _ = _frame_once(tr, "gs_mesh", cams[v], gts[v], True, False)
            _assert_same(on, off, (name, v))
        if name == "gs_mesh_500k_1080p":
            r = NativeRenderer(m, W, H)
            v0 = m.vertices.detach().clone()
            for t in (0.0, 9.7, 10 * np.pi):
                verts = scenes.transform_hotdog_fly(v0, float(t)).contiguous()
                ref = [x.clone() for x in r.render(cams[0], bg, vertices=verts)]
                got = r.render(cams[0], bg, vertices=verts, debug=True)
                for a, b in zip(got, ref):
                    assert torch.equal(a, b), t


# ---- the three other render frames

def _points_model():
    p = scenes.init_mesh_gaussians(*scenes.icosphere(3), K=3, seed=21, trained_like=True)
    with torch.no_grad():
        xyz, sl, rr = MeshGaussianModel.from_params(p, "cuda").expand_fused(activated=False)
    return PointsModel.from_gaussians(xyz, sl, rr, p._features_dc, p._features_rest, p._opacity, "cuda")


def _flame_checkpoint(tmp_path):
    m = _model("gs_flame")
    cams, gts = _views()
    tr = _trainer("gs_flame", m)
    for v in range(2):
        tr.step(cams[v], gts[v])
    ply = str(tmp_path / "point_cloud.ply")
    io_ply.save_flame_model(ply, m)
    ck = FlameCheckpoint.load(ply, active_sh_degree=m.active_sh_degree)
    ck.vertices = ck.driver_vertices(m.driver)
    return ck


@pytest.mark.parametrize("kind", ["points", "bound_points", "flame"])
def test_debug_render_of_the_other_frames_equals_the_render_without_it(kind, tmp_path):
    cams, _ = _views()
    bg = torch.tensor(BG, device="cuda")
    if kind == "flame":
        r = FlameRenderer(_flame_checkpoint(tmp_path), W, H)
    else:
        pm = _points_model()
        if kind == "points":
            r = PointsRenderer(pm, W, H)
        else:
            v, f = scenes.icosphere(3)
            r = MeshBoundPointsRenderer(pm.bind_to_mesh(torch.tensor(v).cuda(), torch.tensor(f).cuda()), W, H)
    for cam in cams:
        r.render(cam, bg)
    for cam in cams:
        for aa in (False, True):
            n0 = _lib.launch_count()
            ref = [t.clone() for t in r.render(cam, bg, antialiasing=aa)]
            n1 = _lib.launch_count()
            got = [t.clone() for t in r.render(cam, bg, antialiasing=aa, debug=True)]
            n2 = _lib.launch_count()
            for a, b in zip(got, ref):
                assert torch.equal(a, b), (kind, aa)
            assert n2 - n1 == n1 - n0 + 2, (kind, n2 - n1, n1 - n0)

"""-m gpu: anomaly detection of native training (the reference's train.py --detect_anomaly) for gs_mesh, segmented
gs_multi_mesh, gs_flame, gs and gs_flat.

Checked here: gms_nan_scan against numpy over sizes, pointer offsets and several buffers and calls; clean frames with the
record equal the frames without it and add one launch per stage; every hook reports its own stage at a tensor element the
seeded NaN reaches; NaN left in the accumulated buffers (d_vertices, accum) is found at its index; each trainer raises
AnomalyError at the iteration whose view holds the NaN with its state untouched, and the autograd arm raises torch's
anomaly error there; clean runs with the flag match runs without it.

No NaN or Inf is ever put into geometry (positions, vertices, _alpha, scales, rotations): only into ground-truth pixels, into
buffers a frame accumulates into, or straight into gms_nan_scan's inputs."""
import ctypes as C

import numpy as np
import pytest
import torch

from gms_b200 import _lib, anomaly
from gms_b200.anomaly import AnomalyError, AnomalyRecord
from gms_b200.trainer import FlameOptimizationParams, FlameTrainer, FreeOptimizationParams, FreeTrainer, MeshTrainer
from test_gpu_train_antialiasing import BG, FREE_TYPES, H, LAMBDA, MESH_TYPES, TYPES, W, _frame, _model, _names, _views
from test_gpu_train_mixed_sizes import _bound, _outputs, _rel

pytestmark = pytest.mark.gpu

NONE = _lib.ANOMALY_NONE


def _trainer(gs_type, model, detect, iterations=1, **free):
    bg = torch.tensor(BG, device="cuda")
    if gs_type in MESH_TYPES:
        return MeshTrainer(model, bg, LAMBDA, native=True, optimizer_step=iterations > 1, detect_anomaly=detect)
    if gs_type == "gs_flame":
        return FlameTrainer(model, bg, FlameOptimizationParams(iterations=iterations), detect_anomaly=detect)
    return FreeTrainer(model, bg, 1.0, FreeOptimizationParams(iterations=iterations, **free), detect_anomaly=detect,
                       generator=torch.Generator(device="cuda").manual_seed(3))


# ---------------------------------------------------------------------------------------------- 1. the scan itself

def _np_first(stage, bufs):
    """numpy's smallest key over (tensor id, float32 array) pairs, or NONE."""
    keys = [anomaly.encode(stage, t, int(np.flatnonzero(np.isnan(a))[0])) for t, a in bufs if np.isnan(a).any()]
    return min(keys) if keys else NONE


def _read(rec):
    torch.cuda.synchronize()
    return int(rec.item()) & NONE


@pytest.mark.parametrize("n", [0, 1, 3, 4, 5, (1 << 20) + 3])
def test_scan_matches_numpy(n):
    """Every pointer offset 0..3 floats; NaN at the first element, the last, inside the scalar tail, or nowhere, among +-inf,
    large values and denormals (never reported); one call with several buffers, then calls that must keep a smaller earlier
    key; a clean scan leaves the record untouched."""
    rng = np.random.default_rng(n)
    rec = torch.empty(1, dtype=torch.int64, device="cuda")
    noise = np.float32([np.inf, -np.inf, 3e38, -3e38, 1e-45, -1e-45, -0.0, 1e-39])
    for off in range(4):
        base = torch.empty(n + 8, dtype=torch.float32, device="cuda")
        for where in ("none", "first", "last", "tail"):
            host = rng.standard_normal(n).astype(np.float32)
            if n:
                host[rng.integers(0, n, size=min(n, 8))] = noise[:min(n, 8)]
                pos = {"none": None, "first": 0, "last": n - 1, "tail": max(n - 2, 0)}[where]
                if pos is not None:
                    host[pos] = np.nan
            view = base[off:off + n]
            view.copy_(torch.from_numpy(host))
            other = torch.from_numpy(host[::-1].copy()).cuda()          # a second buffer, second tensor id
            rec.fill_(-1)
            anomaly.nan_scan(rec, 2, [(3, view), (1, other)])
            assert _read(rec) == _np_first(2, [(3, host), (1, host[::-1])]), (n, off, where)
            got = _read(rec)
            anomaly.nan_scan(rec, 3, [(0, view)])                       # a later stage never replaces an earlier key
            assert _read(rec) == (got if got != NONE else _np_first(3, [(0, host)]))
    clean = torch.from_numpy(np.resize(noise, n)).cuda()
    rec.fill_(12345)
    anomaly.nan_scan(rec, 0, [(0, clean)])
    assert _read(rec) == 12345, "a clean scan writes nothing"
    if n > 5:
        x = torch.zeros(n, device="cuda")
        x[n - 1] = float("nan")
        rec.fill_(-1)
        anomaly.nan_scan(rec, 1, [(2, x)])
        x[n - 1], x[3] = 0.0, float("nan")
        anomaly.nan_scan(rec, 1, [(2, x)])                              # smaller index, same stage and tensor: replaces
        assert _read(rec) == anomaly.encode(1, 2, 3)


def test_scan_of_many_buffers_reports_the_lowest_tensor():
    rec = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    bufs = [(t, torch.zeros(1000 + 37 * t, device="cuda")) for t in range(_lib.NAN_SCAN_MAX_BUFFERS)]
    for t, b in bufs[3:]:
        b[999 - t] = float("nan")
    anomaly.nan_scan(rec, 4, bufs[::-1])
    assert _read(rec) == anomaly.encode(4, 3, 996)
    n0 = _lib.launch_count()
    anomaly.nan_scan(rec, 4, [(0, torch.zeros(0, device="cuda"))])
    anomaly.nan_scan(rec, 4, bufs)
    assert _lib.launch_count() - n0 == 1, "one launch per call, none for empty buffers"


# ---------------------------------------------------------------------------------------------- 2. clean frames

def _grab_step(tr, gs_type, cam, gt):
    grads = {}

    def grab():
        for n in _names(gs_type):
            grads[n] = getattr(tr.model, n).grad.detach().clone()

    n0 = _lib.launch_count()
    tr.step(cam, gt, before_update=grab)
    torch.cuda.synchronize()
    out = _outputs(_frame(tr), cam)
    out["grads"], out["launches"] = grads, _lib.launch_count() - n0
    return out


@pytest.mark.parametrize("degree", [0, 3])
@pytest.mark.parametrize("gs_type", TYPES)
def test_clean_frames_are_the_frames_without_the_record(gs_type, degree):
    """A clean view through a trainer with detect_anomaly and one without: the record stays NONE; image and radii bit for
    bit; the loss to 2e-6 relative; every gradient within the spread bound; each scanned stage adds exactly one launch (four
    per frame, and the FLAME backward's for a NativeFlame driver)."""
    cams, gts = _views(gs_type, 1)
    runs = {}
    for detect in (False, True):
        m = _model(gs_type, degree)
        tr = _trainer(gs_type, m, detect)
        _grab_step(tr, gs_type, cams[0], gts[0])            # the view's synchronising first frame
        runs[detect] = [_grab_step(tr, gs_type, cams[0], gts[0]) for _ in range(2)]
        if detect:
            assert tr._anomaly.read() == NONE
    off, on = runs[False][1], runs[True][1]
    assert torch.equal(off["image"], on["image"]) and torch.equal(off["radii"], on["radii"])
    assert abs(float(on["loss"][0]) - float(off["loss"][0])) <= 2e-6 * abs(float(off["loss"][0]))
    for n in _names(gs_type):
        spread = _rel(runs[False][0]["grads"][n], off["grads"][n])
        assert _rel(on["grads"][n], off["grads"][n]) <= max(_bound(n), 10 * spread), n
    extra = 4 + (1 if gs_type == "gs_flame" else 0)
    assert on["launches"] - off["launches"] == extra, (on["launches"], off["launches"])


# ---------------------------------------------------------------------------------------------- 3. every hook fires

REACH = 10      # the 11x11 SSIM window applied twice: dL/dimage at a pixel depends on pixels up to 10 away


def _means2d(fr, P, radii):
    """The frame's screen positions [P,2] (gms_debug_unpack of its geometry scratch)."""
    s = _lib.RasterSaved()
    s.geom = fr._scratch[_lib.BUF_GEOM].data_ptr()
    xy = torch.zeros(P, 2, device="cuda")
    _lib.check(_lib.lib().gms_debug_unpack(C.byref(s), P, radii.data_ptr(), xy.data_ptr(), None, None, None, None,
                                           torch.cuda.current_stream().cuda_stream), "gms_debug_unpack")
    torch.cuda.synchronize()
    return xy.cpu().numpy()


def _reaches(xy, radius, y0, x0):
    """Whether a splat's tile rectangle (gms_get_rect) covers a tile that holds a pixel within REACH of (y0, x0)."""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    r = float(radius)
    tx0, ty0 = min(gx, max(0, int((xy[0] - r) / 16))), min(gy, max(0, int((xy[1] - r) / 16)))
    tx1, ty1 = min(gx, max(0, int((xy[0] + r + 15) / 16))), min(gy, max(0, int((xy[1] + r + 15) / 16)))
    px0, px1 = max(0, x0 - REACH) // 16, min(W - 1, x0 + REACH) // 16
    py0, py1 = max(0, y0 - REACH) // 16, min(H - 1, y0 + REACH) // 16
    return radius > 0 and tx0 <= px1 and px0 < tx1 and ty0 <= py1 and py0 < ty1


def _gaussian_rows_of_vertex(model, v):
    """Rows of the Gaussians on faces that use vertex v."""
    faces = model.faces.cpu().numpy()
    F, K, _ = model.frame_sizes()
    segs = list(model.segments) if model.segments is not None else [(F, K)]
    rows, f0, p0 = [], 0, 0
    for Fi, Ki in segs:
        for f in np.flatnonzero((faces[f0:f0 + Fi] == v).any(1)):
            rows.extend(range(p0 + f * Ki, p0 + (f + 1) * Ki))
        f0, p0 = f0 + Fi, p0 + Fi * Ki
    return rows


@pytest.mark.parametrize("gs_type", TYPES)
def test_every_hook_reports_its_own_stage(gs_type):
    """One NaN ground-truth pixel, the frame's stages selected one at a time: each hook reports its own stage, at a pixel of
    dL/dimage within the loss's reach of the seeded pixel, or at a Gaussian (radii > 0) whose tile rectangle covers a pixel
    within that reach (a vertex of such a Gaussian's face for d_vertices)."""
    cams, gts = _views(gs_type, 1)
    cam = cams[0]
    m = _model(gs_type)
    tr = _trainer(gs_type, m, True)
    tr.step(cam, gts[0])
    fr = _frame(tr)
    P = fr._gaussians()
    c0, y0, x0 = 1, 77, 131
    bad = gts[0].clone()
    bad[c0, y0, x0] = float("nan")
    last = _lib.ANOMALY_ACTIVATION_BWD if gs_type in FREE_TYPES else _lib.ANOMALY_EXPAND_BWD
    rec = AnomalyRecord("cuda")
    bg = torch.tensor(BG, device="cuda")
    for stage in (_lib.ANOMALY_LOSS, _lib.ANOMALY_COMPOSITE_BWD, _lib.ANOMALY_PREPROCESS_BWD, last):
        if gs_type in MESH_TYPES or gs_type == "gs_flame":
            m.vertices.grad.zero_()
        fr.run(cam, bad, bg, anomaly=rec.reset(), anomaly_stages=1 << stage)
        out = _outputs(fr, cam)
        found = anomaly.decode(rec.read())
        assert found is not None and found[0] == stage, (stage, found)
        _, t, i = found
        if stage == _lib.ANOMALY_LOSS:
            c, r = divmod(i, H * W)
            assert c == c0 and abs(r // W - y0) <= REACH and abs(r % W - x0) <= REACH, (c, r // W, r % W)
            continue
        xy = _means2d(fr, P, out["radii"])
        radii = out["radii"].cpu().numpy()
        if stage == _lib.ANOMALY_EXPAND_BWD and t == _lib.ANOMALY_DVERTICES:
            rows = _gaussian_rows_of_vertex(m, i // 3)
        else:
            rows = [i // anomaly._row_width(stage, t, anomaly.layout_of(m, cam))]
        assert any(_reaches(xy[r], int(radii[r]), y0, x0) for r in rows), (stage, t, i)
        print(f"[{gs_type}] stage {anomaly.STAGE_NAMES[stage]}: {anomaly.TENSOR_NAMES[stage][t]} at {i}")


@pytest.mark.parametrize("gs_type", ["gs_mesh", "gs_multi_mesh", "gs_flame", "gs_flat"])
def test_nan_left_in_accumulated_buffers_is_found_at_its_index(gs_type):
    """A NaN the caller left in d_vertices (mesh types) or accum (free types) is reported by the expansion or activation hook
    at exactly its index, with a clean ground truth."""
    cams, gts = _views(gs_type, 1)
    m = _model(gs_type)
    tr = _trainer(gs_type, m, True)
    tr.step(cams[0], gts[0])
    fr = _frame(tr)
    rec = AnomalyRecord("cuda")
    bg = torch.tensor(BG, device="cuda")
    if gs_type in FREE_TYPES:
        k, stage, tensor = fr.accum.numel() - 2, _lib.ANOMALY_ACTIVATION_BWD, _lib.ANOMALY_ACCUM
        fr.accum[k] = float("nan")
        fr.run(cams[0], gts[0], bg, anomaly=rec.reset())
    else:
        k, stage, tensor = 3 * (m.vertices.shape[0] // 2) + 1, _lib.ANOMALY_EXPAND_BWD, _lib.ANOMALY_DVERTICES
        m.vertices.grad.zero_()
        m.vertices.grad.view(-1)[k] = float("nan")
        fr.run(cams[0], gts[0], bg, anomaly=rec.reset())
        m.vertices.grad.zero_()
    assert anomaly.decode(rec.read()) == (stage, tensor, k)


# ---------------------------------------------------------------------------------------------- 4. trainers

def _same_state(a, b):
    for k in ("p", "m", "v"):
        assert torch.equal(a["adam"][k], b["adam"][k]), k
    assert a["adam"]["steps"] == b["adam"]["steps"]
    for k, v in a.items():
        if k != "adam":
            assert (torch.equal(v, b[k]) if torch.is_tensor(v) else v == b[k]), k


@pytest.mark.parametrize("gs_type", TYPES)
def test_trainer_raises_at_the_iteration_of_the_nan_view_with_its_state_untouched(gs_type):
    """A NaN ground-truth pixel in the view of iteration 4: steps 1-3 run, step 4 raises AnomalyError (before_update is not
    called), state_dict() afterwards equals the one taken before that step bit for bit, and the trainer steps on."""
    cams, gts = _views(gs_type, 4)
    bad = gts[3].clone()
    bad[2, 100, 60] = float("nan")
    m = _model(gs_type)
    tr = _trainer(gs_type, m, True, iterations=100)
    for i in range(3):
        tr.step(cams[i], gts[i])
    torch.cuda.synchronize()
    before = tr.state_dict()
    hook = []
    with pytest.raises(AnomalyError) as e:
        tr.step(cams[3], bad, before_update=lambda: hook.append(1))
    print(f"[{gs_type}] {e.value}")
    assert e.value.stage == _lib.ANOMALY_LOSS and hook == []
    if not isinstance(tr, MeshTrainer):
        assert "iteration 4" in str(e.value) and tr.iteration == 3
    _same_state(before, tr.state_dict())
    tr.step(cams[3], gts[3])
    torch.cuda.synchronize()
    assert tr._anomaly.read() == NONE


def test_autograd_arm_raises_torch_anomaly_error_at_the_same_iteration():
    cams, gts = _views("gs_mesh", 4)
    bad = gts[3].clone()
    bad[2, 100, 60] = float("nan")
    tr = MeshTrainer(_model("gs_mesh"), torch.tensor(BG, device="cuda"), LAMBDA, native=False, detect_anomaly=True)
    for i in range(3):
        tr.step(cams[i], gts[i])
    with pytest.raises(RuntimeError, match="returned nan values") as e:
        tr.step(cams[3], bad)
    assert not isinstance(e.value, AnomalyError)


# ---------------------------------------------------------------------------------------------- 5. clean runs

def _run(gs_type, detect, steps, **free):
    cams, gts = _views(gs_type, 4)
    m = _model(gs_type)
    tr = _trainer(gs_type, m, detect, iterations=1000, **free)
    init = {n: getattr(m, n).detach().clone() for n in _names(gs_type)}
    for i in range(steps):
        tr.step(cams[i % 4], gts[i % 4])
    torch.cuda.synchronize()
    return init, {n: getattr(m, n).detach().clone() for n in _names(gs_type)}, tr


@pytest.mark.parametrize("gs_type,free", [("gs_mesh", {}),
                                          ("gs_flat", dict(densify_from_iter=3, densification_interval=4, densify_grad_threshold=1e-5))])
def test_clean_run_with_the_flag_matches_one_without(gs_type, free):
    """Ten steps with the flag against ten without (which fuse the SH Adam step): every parameter within 10x the run-to-run
    spread of two runs without it, or 1 % of how far training moved it; gs_flat densifies and ends with the same P."""
    init, a, ta = _run(gs_type, False, 10, **free)
    _, a2, _ = _run(gs_type, False, 10, **free)
    _, b, tb = _run(gs_type, True, 10, **free)
    if gs_type in FREE_TYPES:
        assert ta.densifications and tb.model.P == ta.model.P, (ta.densifications, tb.densifications)
    for n in _names(gs_type):
        spread = float((a[n] - a2[n]).abs().max())
        moved = float((a[n] - init[n]).abs().max()) if a[n].shape == init[n].shape else float(a[n].abs().max())
        d = float((a[n] - b[n]).abs().max())
        print(f"[{gs_type} clean run] {n}: |on - off| {d:.2e}, run-to-run {spread:.2e}, moved {moved:.2e}")
        assert d <= max(10 * spread, 1e-2 * moved), n

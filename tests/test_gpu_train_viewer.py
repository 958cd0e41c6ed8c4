"""cli.train --viewer on the GPU, with an in-process viewer on 127.0.0.1 at an ephemeral port and the small generated
scenes of the other CLI tests: the frames served at a save iteration N equal, byte for byte, what cli.view draws from
point_cloud/iteration_N (all five training types, both backgrounds, two image sizes and scaling modifiers); `train: false`
pauses the run without changing where it ends; `keep_alive` holds the last iteration until the viewer lets go or leaves;
gs_flat frames across a densification; and the host synchronisations: none added to a run with no viewer, exactly one
per served frame with one."""
import os
import socket
import threading

import numpy as np
import pytest
import torch

import mesh_types_cases as cases
from gms_b200 import network_gui
from gms_b200.cli import train as cli_train
from gms_b200.cli import view
from test_gpu_dataset import _write_rendered_blender
from test_gpu_train_mesh_types import _write_colmap_from_blender
from test_gpu_viewer import _counted, _message

pytestmark = pytest.mark.gpu

COMMON = ["--eval", "--test_iterations", "-1", "--quiet", "--port", "0", "--viewer"]
TYPE_ARGV = {"gs_mesh": [], "gs_flat": ["--gs_type", "gs_flat"], "gs": ["--gs_type", "gs"],
             "gs_multi_mesh": ["--gs_type", "gs_multi_mesh", "--meshes", "a", "b", "--num_splats", "2", "3"],
             "gs_flame": ["--gs_type", "gs_flame", "--flame_model", cases.FLAME_MODEL]}
MESH_NAMES = ("vertices", "_alpha", "_scale", "_features", "_opacity")


@pytest.fixture(scope="module")
def roots(tmp_path_factory):
    base = tmp_path_factory.mktemp("train_viewer")
    blender = str(base / "blender")
    _write_rendered_blender(blender)
    return {"blender": blender, "colmap": _write_colmap_from_blender(blender, str(base / "colmap"))}


def _root(roots, gs_type):
    return roots["colmap" if gs_type == "gs_multi_mesh" else "blender"]


def _request(**kw):
    """A camera request (test_gpu_viewer's look_at view), train / keep_alive as given."""
    eye = kw.pop("eye", (2.4, 0.8, 1.0))
    m = _message(kw.pop("W", 16), kw.pop("H", 16), kw.pop("s", 1.0), eye=eye)
    m.update(kw)
    return m


RELEASE = _request(train=True, keep_alive=False)


def _training(roots, gs_type, out, argv, viewer=True):
    common = COMMON if viewer else [a for a in COMMON if a != "--viewer"]
    return cli_train.Training(cli_train.parse_args(["-s", _root(roots, gs_type), "-m", out] + TYPE_ARGV[gs_type] + common + argv)).prepare()


def _drive(run, script):
    """run.run() here while script(conn, run) talks to it from a thread over a TCP connection made before the first
    iteration (so accepted at it); the connection is closed when the script returns or fails.  The script reads the run's
    state only after a reply to a request that did not release the iteration: the loop then waits for the next request."""
    conn = socket.create_connection(run.viewer.address)
    err = []

    def client():
        try:
            script(conn, run)
        except BaseException as e:      # noqa: BLE001 -- re-raised below
            err.append(e)
        finally:
            conn.close()

    t = threading.Thread(target=client)
    t.start()
    try:
        run.run()
    finally:
        t.join()
    if err:
        raise err[0]
    return run


def _view_frames(out, gs_type, it, degree):
    """cli.view's Frames of point_cloud/iteration_it at the live model's active SH degree."""
    _, frames, verify = view.load(["-m", out, "--gs_type", gs_type, "--iteration", str(it)])
    frames.model.active_sh_degree = degree
    return frames, verify


def _drawn(frames, msg) -> bytes:
    with torch.no_grad():
        return bytes(frames(network_gui.parse(msg).camera, msg["scaling_modifier"]))


# ------------------------------------------------------------------------------------------------ frame content

@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("gs_type", ["gs_mesh", "gs_multi_mesh", "gs_flame", "gs_flat", "gs"])
def test_frames_at_a_save_iteration_equal_cli_view(roots, tmp_path, gs_type, white):
    N, SAVE = 12, 8
    out = str(tmp_path / "out")
    msgs = [_request(W=64, H=48, s=1.0), _request(W=37, H=23, s=0.6, eye=(0.5, 2.6, 0.9)),
            _request(W=64, H=48, s=0.6, eye=(-2.0, 1.5, 1.2)), _request(W=37, H=23, s=1.0, eye=(0.3, -2.2, -1.4))]
    got, seen = [], {}

    def script(conn, run):
        for it in range(1, N + 1):
            if it == SAVE:
                for m in msgs:
                    image, v = network_gui.request(conn, m)
                    got.append(bytes(image))
                    seen["verify"] = bytes(v)
                seen["degree"], seen["events"] = run.model.active_sh_degree, len(run.events)
            network_gui.request(conn, RELEASE)

    argv = ["--iterations", str(N), "--save_iterations", str(SAVE)] + (["-w", "--random_background"] if white else [])
    run = _drive(_training(roots, gs_type, out, argv), script)
    assert seen["events"] == SAVE - 1 and len(run.ema) == N
    assert run.viewer.frames == N + len(msgs)
    frames, verify = _view_frames(out, gs_type, SAVE, seen["degree"])
    assert seen["verify"] == verify == os.path.abspath(_root(roots, gs_type)).encode()
    assert frames.bg.tolist() == [float(white)] * 3
    for m, image in zip(msgs, got):
        assert image == _drawn(frames, m), (gs_type, white, m["resolution_x"], m["scaling_modifier"])
        assert set(image) != {255 * white}, "the frame should show the model, not the background"
        if gs_type in ("gs_mesh", "gs_multi_mesh"):     # (gs and gs_flat start from a random cloud: fog at iteration 8)
            assert len(set(image[::3])) > 8, "the camera should see the model"


# ------------------------------------------------------------------------------------------------ pausing and keep_alive

def _final(run):
    return {n: getattr(run.model, n).detach().clone() for n in MESH_NAMES}


def test_train_false_pauses_the_run_and_changes_nothing(roots, tmp_path):
    N, AT, K = 20, 7, 5
    pause = _request(W=48, H=40, train=False, keep_alive=True)
    replies, state = [], []

    def script(conn, run):
        for it in range(1, N + 1):
            if it == AT:
                for _ in range(K):
                    replies.append(bytes(network_gui.request(conn, pause)[0]))
                    state.append((len(run.events), len(run.ema) + len(run._pending), run.order.state_dict()))
            network_gui.request(conn, RELEASE)

    paused = _drive(_training(roots, "gs_mesh", str(tmp_path / "paused"), ["--iterations", str(N)]), script)
    assert len(replies) == K and len(set(replies)) == 1 and len(set(replies[0][::3])) > 8
    assert all(s == state[0] for s in state) and state[0][0] == AT - 1
    assert len(paused.ema) == N

    def unpaused(name):
        run = _training(roots, "gs_mesh", str(tmp_path / name), ["--iterations", str(N)], viewer=False)
        assert run.viewer is None
        return _final(run.run())

    a, b = unpaused("a"), unpaused("b")
    got = _final(paused)
    for n in MESH_NAMES:
        d_got, d_other = float((got[n] - a[n]).abs().max()), float((b[n] - a[n]).abs().max())
        print(f"[paused vs unpaused] {n}: {d_got:.3e}, run-to-run {d_other:.3e}")
        assert d_got <= 10 * d_other + 1e-7, n


@pytest.mark.parametrize("leave", ["release", "disconnect at the last", "disconnect early"])
def test_keep_alive_holds_the_last_iteration(roots, tmp_path, leave):
    N = 6
    hold = _request(train=True, keep_alive=True)
    seen = []

    def script(conn, run):
        for it in range(1, N + 1):
            if leave == "disconnect early" and it == 3:
                return
            network_gui.request(conn, hold)
        for _ in range(3):              # the last iteration stays held
            seen.append((len(run.events), len(run.ema) + len(run._pending)))
            network_gui.request(conn, hold)
        if leave == "release":
            network_gui.request(conn, _request(train=True, keep_alive=False))

    run = _drive(_training(roots, "gs_flat", str(tmp_path / "out"), ["--iterations", str(N)]), script)
    if leave != "disconnect early":
        assert seen == [(N - 1, N - 1)] * 3
        assert run.viewer.frames == N + 3 + (leave == "release")
    assert [it for it, _, _ in run.ema] == list(range(1, N + 1))
    assert os.path.exists(os.path.join(str(tmp_path / "out"), "point_cloud", f"iteration_{N}", "point_cloud.ply"))
    assert run.viewer.conn is None and run.viewer.listener.fileno() == -1


# ------------------------------------------------------------------------------------------------ densification

def test_gs_flat_frames_follow_densification(roots, tmp_path):
    N = 12
    out = str(tmp_path / "out")
    msg = _request(W=64, H=48, train=False)
    got, P = {}, {}

    def script(conn, run):
        for it in range(1, N + 1):
            if it in (8, 9):
                got[it] = bytes(network_gui.request(conn, msg)[0])
                P[it] = run.model.P
            network_gui.request(conn, RELEASE)

    argv = ["--iterations", str(N), "--densify_from_iter", "5", "--densification_interval", "8", "--densify_grad_threshold", "1e-9",
            "--save_iterations", "8", "9"]
    run = _drive(_training(roots, "gs_flat", out, argv), script)
    assert [d[0] for d in run.trainer.densifications] == [8] and P[8] != P[9], (P, run.trainer.densifications)
    r = run.viewer.draw.sizes[(64, 48)][0]
    assert r.radii.shape[0] == P[9] and not r.stale
    for it in (8, 9):
        frames, _ = _view_frames(out, "gs_flat", it, 0)
        assert frames.model.P == P[it]
        assert got[it] == _drawn(frames, msg), it


# ------------------------------------------------------------------------------------------------ synchronisation

def test_viewer_without_a_client_adds_no_synchronisation(roots, tmp_path):
    """test_gpu_cli's window: every iteration but the first and the save iterations runs under sync debug mode "error"."""
    sync_ok = {1, 10, 20, 30}

    class Strict(cli_train.Training):
        def _relaxed(self, fn, *a, **k):
            torch.cuda.set_sync_debug_mode(0)
            try:
                return fn(*a, **k)
            finally:
                torch.cuda.set_sync_debug_mode("error")

        def save(self, it):
            assert it in sync_ok
            self._relaxed(super().save, it)

        def checkpoint(self, it):
            self._relaxed(super().checkpoint, it)

        def _consume(self, block=False):
            return self._relaxed(super()._consume, block) if block else super()._consume(block)

    argv = ["-s", roots["blender"], "-m", str(tmp_path)] + COMMON + ["--iterations", "30", "--save_iterations", "10", "20",
                                                                      "--checkpoint_iterations", "15"]
    run = Strict(cli_train.parse_args(argv)).prepare()
    step = run.trainer.step

    def first_relaxed(*a, **k):
        return run._relaxed(step, *a, **k) if run._first else step(*a, **k)

    run._first = True
    run.trainer.step = lambda *a, **k: (first_relaxed(*a, **k), setattr(run, "_first", False))[0]
    torch.cuda.set_sync_debug_mode("error")
    try:
        run.run()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(run.ema) == 30 and run.viewer.frames == 0


def test_one_synchronisation_per_served_frame(roots, tmp_path):
    N = 10
    syncs = []
    msgs = [_request(W=64, H=48, train=False), _request(W=37, H=23, s=0.7, train=False)]

    def script(conn, run):
        for it in range(1, N + 1):
            for m in msgs:
                network_gui.request(conn, m)
            network_gui.request(conn, RELEASE)

    run = _training(roots, "gs_mesh", str(tmp_path / "out"), ["--iterations", str(N)])
    run.viewer.draw = _counted(run.viewer.draw, syncs)
    _drive(run, script)
    assert run.viewer.frames == 3 * N
    assert len(syncs) == 3 * N - 3 and [len(x) for x in syncs] == [1] * len(syncs), syncs
    assert np.isfinite(run.ema[-1][1])

"""The remote viewer's protocol (gms_b200.network_gui) and gms_b200.cli.view's command line, without a GPU: the camera and
the reply bytes against the reference's own network_gui run on the CPU (tests/golden/viewer.npz, make_viewer_golden.py),
short reads and writes over a socketpair, malformed requests that end one session only, and the cfg_args merge.  No test
opens a network socket: socket.socket refuses everything but the wrapping of a socketpair's ends."""
import argparse
import json
import math
import os
import socket
import threading
import time

import numpy as np
import pytest
import torch

from gms_b200 import _lib, network_gui
from gms_b200.cli import render, view

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "viewer.npz"))
CASES = ("camera", "flags", "ints", "zero", "zero_width")
VERIFY = GOLDEN["verify"].tobytes()


@pytest.fixture(autouse=True)
def no_network(monkeypatch):
    real = socket.socket

    def local_only(family=-1, type=-1, proto=-1, fileno=None):
        if fileno is None or family != socket.AF_UNIX:
            raise AssertionError("network socket opened")
        return real(family, type, proto, fileno)

    def refuse(*a, **k):
        raise AssertionError("network connection attempted")

    monkeypatch.setattr(socket, "socket", local_only)
    monkeypatch.setattr(socket, "create_connection", refuse)
    monkeypatch.setattr(socket, "create_server", refuse)


def _serve_requests(data: bytes, draw, chunk=None):
    """Sends `data` to a session on a socketpair, then hangs up; returns (reply bytes, frames served, log)."""
    a, b = socket.socketpair()
    log = []

    def client():
        if chunk is None:
            a.sendall(data)
        else:
            for i in range(0, len(data), chunk):
                a.sendall(data[i:i + chunk])
                time.sleep(0.001)
        a.shutdown(socket.SHUT_WR)

    t = threading.Thread(target=client)
    t.start()
    out = {}
    srv = threading.Thread(target=lambda: out.setdefault("frames", network_gui.serve(b, draw, VERIFY, log=log.append)))
    srv.start()
    reply = bytearray()
    while True:
        k = a.recv(4093 if chunk else 1 << 16)
        if not k:
            break
        reply += k
        if chunk and len(reply) % 64 == 0:
            time.sleep(0.001)
    t.join()
    srv.join()
    a.close()
    return bytes(reply), out["frames"], log


def test_camera_and_reply_match_the_reference():
    for c in CASES:
        request = GOLDEN[f"{c}/request"].tobytes()
        seen = []

        def draw(cam, s):
            seen.append((cam, s))
            return GOLDEN[f"{c}/image"].tobytes()

        reply, frames, _ = _serve_requests(request, draw)
        assert reply == GOLDEN[f"{c}/reply"].tobytes(), c
        assert frames == int(GOLDEN[f"{c}/has_camera"]) == len(seen), c
        req = network_gui.parse(json.loads(request[4:].decode("utf-8")))
        if not GOLDEN[f"{c}/has_camera"]:
            assert req.camera is None
            continue
        cam, s = seen[0]
        for got in (cam, req.camera):
            assert got.world_view_transform.dtype == got.full_proj_transform.dtype == torch.float32
            assert np.array_equal(got.world_view_transform.numpy().view(np.uint32), GOLDEN[f"{c}/world_view"].view(np.uint32)), c
            assert np.array_equal(got.full_proj_transform.numpy().view(np.uint32), GOLDEN[f"{c}/full_proj"].view(np.uint32)), c
            np.testing.assert_array_max_ulp(got.camera_center.numpy(), GOLDEN[f"{c}/camera_center"], maxulp=1)
            assert [got.image_width, got.image_height] == GOLDEN[f"{c}/size"].tolist()
            assert [got.FoVy, got.FoVx] == GOLDEN[f"{c}/fov"].tolist()
            assert [got.znear, got.zfar] == GOLDEN[f"{c}/z"].tolist()
            assert (got.tanfovx, got.tanfovy) == (math.tan(got.FoVx * 0.5), math.tan(got.FoVy * 0.5))    # render()'s
        assert s == req.scaling_modifier == float(GOLDEN[f"{c}/scaling_modifier"])
        assert [req.train, req.shs_python, req.rot_scale_python, req.keep_alive] == GOLDEN[f"{c}/flags"].tolist()


def test_camera_packs_and_unpacks():
    req = network_gui.parse(json.loads(GOLDEN["camera/request"].tobytes()[4:]))
    cam = req.camera.on(req.camera.packed().clone())
    for name in ("world_view_transform", "full_proj_transform", "camera_center"):
        assert torch.equal(getattr(cam, name), getattr(req.camera, name))
    assert (cam.tanfovx, cam.tanfovy, cam.uid) == (req.camera.tanfovx, req.camera.tanfovy, 0)


def test_short_reads_and_writes():
    """A request that arrives a few bytes at a time, and a 3 MB image the peer drains slowly, 4093 bytes at a time."""
    msg = json.loads(GOLDEN["camera/request"].tobytes()[4:])
    msg.update(resolution_x=1000, resolution_y=1000)
    body = json.dumps(msg).encode()
    zero = json.dumps({"resolution_x": 0, "resolution_y": 0}).encode()
    data = len(body).to_bytes(4, "little") + body + len(zero).to_bytes(4, "little") + zero
    image = bytes(np.random.default_rng(0).integers(0, 256, 3_000_000, dtype=np.uint8))
    reply, frames, _ = _serve_requests(data, lambda cam, s: image, chunk=3)
    tail = len(VERIFY).to_bytes(4, "little") + VERIFY
    assert frames == 1 and reply == image + tail + tail


class Trickle:
    """A socket-like object whose recv_into returns one byte per call."""
    def __init__(self, data):
        self.data = data

    def recv_into(self, view, n):
        if not self.data:
            return 0
        view[0], self.data = self.data[0], self.data[1:]
        return 1


def test_read_takes_exactly_the_announced_bytes():
    request = GOLDEN["flags/request"].tobytes()
    assert network_gui.read(Trickle(request)) == json.loads(request[4:])
    with pytest.raises(ConnectionError):
        network_gui.read(Trickle(request[:-1]))


def _good(res=(3, 2)):
    msg = json.loads(GOLDEN["camera/request"].tobytes()[4:])
    msg.update(resolution_x=res[0], resolution_y=res[1])
    body = json.dumps(msg).encode()
    return len(body).to_bytes(4, "little") + body


def _raw(body: bytes):
    return len(body).to_bytes(4, "little") + body


def _malformed():
    msg = json.loads(GOLDEN["camera/request"].tobytes()[4:])
    bad = {"not json": _raw(b"{resolution_x: 3"), "not utf-8": _raw(b"\xff\xfe"), "a list": _raw(b"[1, 2]"),
           "too long": (network_gui.MAX_REQUEST + 1).to_bytes(4, "little") + b"{}"}
    for key in ("fov_x", "view_matrix", "scaling_modifier", "keep_alive"):
        m = dict(msg)
        del m[key]
        bad[f"no {key}"] = _raw(json.dumps(m).encode())
    for name, change in (("15 values", dict(view_matrix=msg["view_matrix"][:15])), ("negative", dict(resolution_x=-3)),
                         ("float size", dict(resolution_x=3.0)), ("text fov", dict(fov_y="wide")),
                         ("singular", dict(view_matrix=[0.0] * 16))):
        bad[name] = _raw(json.dumps(dict(msg, **change)).encode())
    return bad


def _rest(conn) -> bytes:
    """Everything conn receives until the peer closes (a close with our bytes unread resets the connection)."""
    out = bytearray()
    try:
        while True:
            k = conn.recv(1 << 16)
            if not k:
                break
            out += k
    except ConnectionResetError:
        pass
    return bytes(out)


def test_malformed_request_closes_only_its_session():
    def draw(cam, s):
        return bytes(cam.image_width * cam.image_height * 3)

    tail = len(VERIFY).to_bytes(4, "little") + VERIFY
    for name, bad in _malformed().items():
        a, b = socket.socketpair()
        log, out = [], {}
        srv = threading.Thread(target=lambda: out.setdefault("frames", network_gui.serve(b, draw, VERIFY, log=log.append)))
        srv.start()
        a.sendall(_good())
        assert network_gui.recv_exact(a, 18 + len(tail)) == bytes(18) + tail, name
        a.sendall(bad + _good((5, 4)))
        assert _rest(a) == b"", name                # the session ends: the request after the bad one is not answered
        srv.join()
        a.close()
        assert out["frames"] == 1 and "closing the session" in log[-1], (name, log)
        reply, frames, log = _serve_requests(_good((5, 4)), draw)        # the next viewer is served
        assert reply == bytes(60) + tail and frames == 1 and "disconnected" in log[-1], name


def test_draw_failure_closes_the_session():
    def draw(cam, s):
        raise RuntimeError("out of memory")
    reply, frames, log = _serve_requests(_good(), draw)
    assert reply == b"" and frames == 0 and "out of memory" in log[-1]


def _model_dir(tmp_path, **cfg):
    d = tmp_path / "model"
    d.mkdir()
    (d / "cfg_args").write_text(str(argparse.Namespace(**cfg)))
    return str(d)


def test_parser_merges_cfg_args(tmp_path):
    d = _model_dir(tmp_path, sh_degree=1, source_path="/data/scene", model_path="elsewhere", images="images",
                   resolution=-1, white_background=True, data_device="cuda", eval=False, num_splats=[5], meshes=[],
                   gs_type="gs_mesh")
    args = render.combined_args(view.build_parser(), ["-m", d])
    assert (args.gs_type, args.white_background, args.source_path, args.sh_degree, args.model_path) == \
        ("gs_mesh", True, "/data/scene", 1, d)
    assert (args.ip, args.port, args.iteration, args.antialiasing) == ("127.0.0.1", 6009, -1, False)
    args = render.combined_args(view.build_parser(), ["-m", d, "--gs_type", "gs_points", "--ip", "0.0.0.0", "--port", "7001",
                                                      "--iteration", "3", "--antialiasing", "-s", "/other"])
    assert (args.gs_type, args.ip, args.port, args.iteration, args.antialiasing, args.source_path) == \
        ("gs_points", "0.0.0.0", 7001, 3, True, "/other")


def test_parser_refuses_an_unknown_or_missing_gs_type(tmp_path, capsys):
    d = _model_dir(tmp_path, sh_degree=3, source_path="/data/scene", white_background=False)
    with pytest.raises(SystemExit):
        view.load(["-m", d])
    assert "--gs_type is not given" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        view.load(["-m", d, "--gs_type", "gs_cube"])
    assert "--gs_type gs_cube is not supported" in capsys.readouterr().err


def test_clamp_u8_refuses_bad_arguments_without_a_launch():
    L = _lib.lib()
    before = _lib.launch_count()
    for args in ((None, 1, 3, 2, 2), (1, None, 3, 2, 2), (1, 1, 0, 2, 2), (1, 1, 5, 2, 2), (1, 1, 3, 0, 2),
                 (1, 1, 3, 65536, 2), (1, 1, 3, 2, 0)):
        assert L.gms_image_clamp_u8(*args, None) == _lib.GMS_E_ARG, args
    assert _lib.launch_count() == before

"""The training side of the remote viewer without a GPU: network_gui.serve_iteration and try_connect against a literal
restatement of the reference's train.py:65-79 (with its network_gui's read / send / receive), run on the same scripted
request sequences over socketpairs; the --viewer / --ip / --port flags; and when cli.train binds, reports and closes its
listener.  No test opens a network socket: socket.socket is replaced by a fake listener or by one that refuses."""
import errno
import json
import os
import socket
import traceback

import pytest
import torch

from gms_b200 import network_gui
from gms_b200.cli import options
from gms_b200.cli import train as cli_train

VERIFY = "/data/scenes/lego"
ITERATIONS = 4


def _frame(cam, s):
    return bytes((7 * i + int(cam.image_width)) % 256 for i in range(cam.image_width * cam.image_height * 3))


def _message(train=True, keep_alive=False, w=2, h=1, **drop):
    m = {"resolution_x": w, "resolution_y": h, "train": train, "fov_y": 0.8, "fov_x": 1.1, "z_near": 0.01, "z_far": 100.0,
         "shs_python": False, "rot_scale_python": False, "keep_alive": keep_alive, "scaling_modifier": 0.7,
         "view_matrix": [1.0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0.1, 0.2, 3.0, 1], "view_projection_matrix": [float(i) for i in range(16)]}
    for k in drop:
        m.pop(k)
    return m


def _wire(m) -> bytes:
    body = m if isinstance(m, bytes) else json.dumps(m).encode()
    return len(body).to_bytes(4, "little") + body


CAM, PAUSE, HOLD = _wire(_message()), _wire(_message(train=False)), _wire(_message(keep_alive=True))
RELEASE_LAST = _wire(_message(keep_alive=False))
ZERO, ZERO_TRAIN = _wire({"resolution_x": 0, "resolution_y": 0}), _wire({"resolution_x": 0, "resolution_y": 0, "train": True})
MALFORMED, MISSING = _wire(b"{not json"), _wire(_message(train=True, keep_alive=False, fov_x=None))
TRUNCATED = (500).to_bytes(4, "little") + b'{"resolution'

# name -> connections, each (iteration from which it waits, request bytes sent before the peer shuts its side down)
SCENARIOS = {
    "no viewer": [],
    "train each iteration": [(1, [CAM] * 4)],
    "train false pauses": [(1, [PAUSE, PAUSE, CAM, CAM, PAUSE, CAM, CAM])],
    "keep_alive before the last iteration": [(1, [HOLD, HOLD, HOLD, HOLD, HOLD, RELEASE_LAST])],
    "keep_alive at the last, then a disconnect": [(1, [CAM, CAM, CAM, HOLD, HOLD])],
    "keep_alive at the last, then train false and a release": [(3, [HOLD, HOLD, PAUSE, RELEASE_LAST])],
    "zero resolution never releases": [(1, [ZERO, ZERO_TRAIN, CAM, ZERO, CAM, ZERO, ZERO])],
    "malformed request": [(1, [CAM, MALFORMED, CAM]), (3, [CAM, CAM])],
    "a request without a key": [(1, [MISSING, CAM])],
    "peer closes mid-request": [(2, [CAM, TRUNCATED])],
    "a viewer that connects late": [(3, [PAUSE, CAM, HOLD, RELEASE_LAST])],
    "a viewer that sends nothing": [(2, [])],
}


class FakeListener:
    """What `init` leaves: accept() hands out each scripted connection from its iteration on, else raises as a
    non-blocking socket with nobody waiting does."""

    def __init__(self, conns):
        self.conns, self.now = list(conns), 0

    def accept(self):
        if self.conns and self.conns[0][0] <= self.now:
            return self.conns.pop(0)[1], ("127.0.0.1", 50000)
        raise BlockingIOError(errno.EAGAIN, "no viewer waits")


def _connections(scenario):
    """(listener, client ends): every connection's requests are already sent, then the client shuts down its side."""
    conns, clients = [], []
    for at, requests in SCENARIOS[scenario]:
        a, b = socket.socketpair()
        a.sendall(b"".join(requests))
        a.shutdown(socket.SHUT_WR)
        conns.append((at, b))
        clients.append(a)
    return FakeListener(conns), clients


def _drain(clients):
    out = []
    for a in clients:
        a.setblocking(False)
        buf = bytearray()
        while True:
            try:
                k = a.recv(1 << 16)
            except BlockingIOError:
                break
            except ConnectionResetError:    # the server closed with requests left unread
                buf += b"<reset>"
                break
            if not k:
                break
            buf += k
        a.close()
        out.append(bytes(buf))
    return out


class Reference:
    """renderer/gaussian_renderer/network_gui.py's module state and functions, restated with `listener` given; the camera is
    built on the host (the reference moves its matrices to the GPU, which the control flow does not see)."""

    def __init__(self, listener):
        self.listener, self.conn, self.addr = listener, None, None

    def try_connect(self):
        try:
            self.conn, self.addr = self.listener.accept()
            self.conn.settimeout(None)
        except Exception:
            pass

    def read(self):
        messageLength = self.conn.recv(4)
        messageLength = int.from_bytes(messageLength, 'little')
        message = self.conn.recv(messageLength)
        return json.loads(message.decode("utf-8"))

    def send(self, message_bytes, verify):
        if message_bytes != None:  # noqa: E711 (as written)
            self.conn.sendall(message_bytes)
        self.conn.sendall(len(verify).to_bytes(4, 'little'))
        self.conn.sendall(bytes(verify, 'ascii'))

    def receive(self):
        message = self.read()
        width = message["resolution_x"]
        height = message["resolution_y"]
        if width != 0 and height != 0:
            try:
                do_training = bool(message["train"])
                fovy = message["fov_y"]
                fovx = message["fov_x"]
                znear = message["z_near"]
                zfar = message["z_far"]
                do_shs_python = bool(message["shs_python"])
                do_rot_scale_python = bool(message["rot_scale_python"])
                keep_alive = bool(message["keep_alive"])
                scaling_modifier = message["scaling_modifier"]
                world_view_transform = torch.reshape(torch.tensor(message["view_matrix"]), (4, 4))
                world_view_transform[:, 1] = -world_view_transform[:, 1]
                world_view_transform[:, 2] = -world_view_transform[:, 2]
                full_proj_transform = torch.reshape(torch.tensor(message["view_projection_matrix"]), (4, 4))
                full_proj_transform[:, 1] = -full_proj_transform[:, 1]
                custom_cam = network_gui.MiniCam(width, height, fovy, fovx, znear, zfar, world_view_transform, full_proj_transform)
            except Exception as e:
                traceback.format_exc()
                raise e
            return custom_cam, do_training, do_shs_python, do_rot_scale_python, keep_alive, scaling_modifier
        else:
            return None, None, None, None, None, None


def _reference_trace(scenario, draw=_frame):
    """train.py:65-79 as written, per iteration: (frames sent, released by a request, connection dropped)."""
    listener, clients = _connections(scenario)
    network_gui_ = Reference(listener)
    trace = []
    for iteration in range(1, ITERATIONS + 1):
        listener.now = iteration
        frames, released, dropped = 0, False, False
        if network_gui_.conn == None:  # noqa: E711
            network_gui_.try_connect()
        while network_gui_.conn != None:  # noqa: E711
            try:
                net_image_bytes = None
                custom_cam, do_training, _, _, keep_alive, scaling_modifer = network_gui_.receive()
                if custom_cam != None:  # noqa: E711
                    net_image_bytes = memoryview(draw(custom_cam, scaling_modifer))
                network_gui_.send(net_image_bytes, VERIFY)
                frames += custom_cam is not None
                if do_training and ((iteration < int(ITERATIONS)) or not keep_alive):
                    released = True
                    break
            except Exception:
                network_gui_.conn = None
                dropped = True
        trace.append((frames, released, dropped))
    return trace, _drain(clients)


def _native_trace(scenario, draw=_frame):
    listener, clients = _connections(scenario)
    conn, trace, log = None, [], []
    for iteration in range(1, ITERATIONS + 1):
        listener.now = iteration
        if conn is None:
            conn = network_gui.try_connect(listener, log=log.append)
        had = conn is not None
        conn, frames = network_gui.serve_iteration(conn, draw, VERIFY.encode(), iteration, ITERATIONS, log=log.append)
        trace.append((frames, conn is not None and had, had and conn is None))
    return trace, _drain(clients)


@pytest.fixture(autouse=True)
def no_network(monkeypatch):
    real = socket.socket

    def local_only(family=-1, type=-1, proto=-1, fileno=None):
        if fileno is None or family != socket.AF_UNIX:
            raise AssertionError("network socket opened")
        return real(family, type, proto, fileno)

    monkeypatch.setattr(socket, "socket", local_only)
    monkeypatch.setattr(socket, "create_connection", lambda *a, **k: pytest.fail("network connection attempted"))


@pytest.mark.parametrize("scenario", list(SCENARIOS))
def test_serve_iteration_traces_train_py(scenario):
    want, want_replies = _reference_trace(scenario)
    got, got_replies = _native_trace(scenario)
    assert got == want, scenario
    assert got_replies == want_replies, scenario


def test_traces_of_the_scripted_behaviour():
    """What the restatement is expected to do, spelled out for the cases the issue names."""
    t = lambda s: _native_trace(s)[0]
    assert t("no viewer") == [(0, False, False)] * 4
    assert t("train each iteration") == [(1, True, False)] * 4
    assert t("train false pauses") == [(3, True, False), (1, True, False), (2, True, False), (1, True, False)]
    assert t("keep_alive before the last iteration") == [(1, True, False)] * 3 + [(3, True, False)]
    assert t("keep_alive at the last, then a disconnect") == [(1, True, False)] * 3 + [(2, False, True)]
    assert t("zero resolution never releases") == [(1, True, False), (1, True, False), (0, False, True), (0, False, False)]
    assert t("malformed request") == [(1, True, False), (0, False, True), (1, True, False), (1, True, False)]
    assert t("a request without a key") == [(0, False, True)] + [(0, False, False)] * 3
    assert t("peer closes mid-request") == [(0, False, False), (1, True, False), (0, False, True), (0, False, False)]
    assert t("a viewer that connects late") == [(0, False, False)] * 2 + [(2, True, False), (2, True, False)]


def test_a_failing_frame_drops_the_connection_and_training_goes_on():
    def broken(cam, s):
        raise RuntimeError("the frame failed")

    want, _ = _reference_trace("train each iteration", broken)
    got, _ = _native_trace("train each iteration", broken)
    assert got == want == [(0, False, True)] + [(0, False, False)] * 3


# ------------------------------------------------------------------------------------------------ cli.train's listener

class FakeSocket:
    """A TCP socket that records what is done to it; port 6010 is taken."""
    made = []

    def __init__(self, family=-1, type=-1, proto=-1, fileno=None):
        assert family == socket.AF_INET and type == socket.SOCK_STREAM
        self.calls, self.closed = [], False
        FakeSocket.made.append(self)

    def setsockopt(self, *a):
        self.calls.append(("setsockopt",) + a)

    def bind(self, addr):
        self.calls.append(("bind", addr))
        if addr[1] == 6010:
            raise OSError(errno.EADDRINUSE, "Address already in use")
        self.addr = (addr[0], addr[1] or 43210)

    def listen(self, *a):
        self.calls.append(("listen",))

    def settimeout(self, t):
        self.calls.append(("settimeout", t))

    def getsockname(self):
        return self.addr

    def accept(self):
        raise BlockingIOError(errno.EAGAIN, "no viewer waits")

    def close(self):
        self.closed = True


@pytest.fixture
def fake_sockets(monkeypatch):
    FakeSocket.made = []
    monkeypatch.setattr(socket, "socket", FakeSocket)
    return FakeSocket.made


def test_viewer_flags_parse_outside_every_group():
    a = cli_train.parse_args(["-s", "scene", "--viewer", "--ip", "0.0.0.0", "--port", "0"])
    assert (a.viewer, a.ip, a.port) == (True, "0.0.0.0", 0)
    b = cli_train.parse_args(["-s", "scene"])
    assert (b.viewer, b.ip, b.port) == (False, "127.0.0.1", 6009)
    assert options.cfg_args_string(a) == options.cfg_args_string(b) and "viewer" not in options.cfg_args_string(a)


def _training(tmp_path, argv, monkeypatch, setup=None):
    args = cli_train.parse_args(["-s", str(tmp_path / "scene"), "-m", str(tmp_path / "out"), "--quiet"] + argv)
    run = cli_train.Training(args, device="cpu")
    seen = {}

    def fake_setup():
        seen["out existed at setup"] = os.path.isdir(args.model_path)
        if setup is not None:
            setup()
        return run

    monkeypatch.setattr(run, "_setup", fake_setup)
    monkeypatch.setattr(cli_train, "open_summary_writer", lambda path, log: None)
    monkeypatch.setattr(run, "viewer_frames", lambda: "frames")
    return run, seen


def test_no_socket_without_the_flag(tmp_path, monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a socket was created without --viewer")

    monkeypatch.setattr(socket, "socket", refuse)
    run, seen = _training(tmp_path, ["--ip", "0.0.0.0", "--port", "0"], monkeypatch)
    assert run.prepare() is run and run.viewer is None and seen["out existed at setup"]


def test_listener_bound_before_the_output_folder_and_closed_by_run(tmp_path, monkeypatch, fake_sockets):
    out = tmp_path / "out"
    run, _ = _training(tmp_path, ["--viewer", "--port", "0"], monkeypatch)
    orig_bind = FakeSocket.bind

    def bind(self, addr):
        assert not out.exists(), "the listener is bound before the output folder is written"
        orig_bind(self, addr)

    monkeypatch.setattr(FakeSocket, "bind", bind)
    run.prepare()
    (s,) = fake_sockets
    assert ("bind", ("127.0.0.1", 0)) in s.calls and ("settimeout", 0) in s.calls and ("listen",) in s.calls
    assert run.viewer.address == ("127.0.0.1", 43210) and run.viewer.draw == "frames"
    assert run.viewer.verify == os.path.abspath(str(tmp_path / "scene")).encode()
    monkeypatch.setattr(run, "_loop", lambda: (_ for _ in ()).throw(RuntimeError("a failed iteration")))
    with pytest.raises(RuntimeError):
        run.run()
    assert s.closed


def test_listener_closed_when_setup_fails(tmp_path, monkeypatch, fake_sockets):
    def fail():
        raise ValueError("a bad scene")

    run, _ = _training(tmp_path, ["--viewer"], monkeypatch, setup=fail)
    with pytest.raises(ValueError):
        run.prepare()
    assert [s.closed for s in fake_sockets] == [True]


def test_busy_port_is_an_error_naming_the_address(tmp_path, monkeypatch, fake_sockets, capsys):
    run, _ = _training(tmp_path, ["--viewer", "--port", "6010"], monkeypatch)
    with pytest.raises(network_gui.AddressError, match="127.0.0.1:6010"):
        run.prepare()
    assert not (tmp_path / "out").exists() and [s.closed for s in fake_sockets] == [True]
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    with pytest.raises(SystemExit) as e:
        cli_train.main(["-s", str(tmp_path / "scene"), "-m", str(tmp_path / "out"), "--viewer", "--port", "6010", "--quiet"])
    assert "127.0.0.1:6010" in str(e.value.code) and "in use" in str(e.value.code)

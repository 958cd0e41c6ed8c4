"""The SIBR remote viewer's wire protocol: renderer/gaussian_renderer/network_gui.py restated, host side only.

A viewer connects over TCP and sends requests; each is a 4-byte little-endian length followed by that many bytes of
UTF-8 JSON.  A request with a non-zero `resolution_x` and `resolution_y` carries a camera, which `parse` turns into the
reference's MiniCam:

    world_view_transform = reshape(view_matrix, 4x4) with columns 1 and 2 negated
    full_proj_transform  = reshape(view_projection_matrix, 4x4) with column 1 negated
    camera_center        = inverse(world_view_transform)[3][:3]

both float32, plus `tanfovx` / `tanfovy` = tan(fov * 0.5) as render() computes them.  The reply is the image (uint8
[H,W,3], row-major), only when the request carries a camera, then a 4-byte little-endian length and the verify string
(the model's source_path).  A request with a zero resolution gets the verify string alone.

`serve` runs one session on an already-connected socket-like object; gms_b200.cli.view owns the listener and the frames.

The training side (train.py:65-79, `cli.train --viewer`): `listen` binds the listener once, non-blocking as `init` leaves
it; at the top of every iteration `TrainingViewer.poll` accepts a waiting viewer when none is connected (`try_connect`,
at most one) and then runs `serve_iteration`, the reference's loop for that iteration: while the viewer stays connected,
read a request, draw its camera when it has one, send the reply, and release the iteration only when the request says
`train` and (iteration < iterations or not `keep_alive`).  A zero-resolution request gets the verify string and does not
release the iteration (the reference's `do_training` is None there); so the last iteration is held for as long as the
viewer asks to keep it alive.  Any error -- a malformed request, a dropped peer, a failed frame -- drops the connection,
and training continues.

Deliberate differences from the reference:
  * `read` waits for exactly the announced number of bytes; the reference calls recv once and can act on a short read
    of a large request.  A request longer than MAX_REQUEST bytes is refused.
  * the camera centre is inverted on the host, in float32 as the reference's torch.inverse does it on the device, so a
    served frame needs no host synchronisation to build its camera.
  * the verify string is sent as UTF-8 (the reference's ASCII for an ASCII path; the reference cannot answer at all when
    the path is not ASCII).
  * `shs_python` and `rot_scale_python` only move the same computation into Python in the reference, so they are parsed
    and ignored; `train` and `keep_alive` steer a training loop (serve_iteration) and are ignored by `serve`.
  * a dropped connection is closed at once; the reference drops its reference to it and leaves the close to the
    garbage collector.
A request that is not valid JSON, lacks a key the reference reads, or has a negative or non-integer resolution ends its
session, as the reference's `conn = None` does, and so does a peer that goes away; the listener then waits for the next
viewer."""
from __future__ import annotations

import json
import math
import socket
import traceback
from dataclasses import dataclass
from typing import Callable, Optional

import torch

HOST, PORT = "127.0.0.1", 6009
MAX_REQUEST = 1 << 20       # a request is a few hundred bytes of JSON


class MiniCam:
    """scene/cameras.py MiniCam with the tan(fov / 2) the renderers read.  Every camera is the same view to a renderer's
    capacity prediction (uid 0), so a served frame is sized from the previous frame at its image size."""
    uid = 0

    def __init__(self, width: int, height: int, fovy: float, fovx: float, znear: float, zfar: float,
                 world_view_transform: torch.Tensor, full_proj_transform: torch.Tensor,
                 camera_center: Optional[torch.Tensor] = None):
        self.image_width, self.image_height = width, height
        self.FoVy, self.FoVx, self.znear, self.zfar = fovy, fovx, znear, zfar
        self.world_view_transform, self.full_proj_transform = world_view_transform, full_proj_transform
        self.camera_center = torch.inverse(world_view_transform)[3][:3] if camera_center is None else camera_center
        self.tanfovx, self.tanfovy = math.tan(fovx * 0.5), math.tan(fovy * 0.5)

    def packed(self) -> torch.Tensor:
        """float32 [35]: world_view_transform, full_proj_transform (row-major) and camera_center."""
        return torch.cat([self.world_view_transform.reshape(-1), self.full_proj_transform.reshape(-1),
                          self.camera_center.reshape(-1)])

    def on(self, packed: torch.Tensor) -> "MiniCam":
        """This camera with its tensors as views of `packed` (float32 [35] holding packed(), e.g. on the device)."""
        return MiniCam(self.image_width, self.image_height, self.FoVy, self.FoVx, self.znear, self.zfar,
                       packed[0:16].view(4, 4), packed[16:32].view(4, 4), packed[32:35])


@dataclass
class Request:
    """One parsed request: receive()'s tuple.  camera is None (and the rest unset) for a zero-resolution request."""
    camera: Optional[MiniCam] = None
    train: Optional[bool] = None
    shs_python: Optional[bool] = None
    rot_scale_python: Optional[bool] = None
    keep_alive: Optional[bool] = None
    scaling_modifier: Optional[float] = None


class ProtocolError(ValueError):
    """A request the protocol cannot answer; it ends the session."""


def recv_exact(conn, n: int) -> bytearray:
    """Exactly n bytes from conn; ConnectionError if the peer closes first."""
    buf = bytearray(n)
    view, got = memoryview(buf), 0
    while got < n:
        k = conn.recv_into(view[got:], n - got)
        if k == 0:
            raise ConnectionError(f"peer closed after {got} of {n} bytes")
        got += k
    return buf


def read(conn) -> dict:
    """network_gui.read: one length-prefixed JSON request."""
    n = int.from_bytes(recv_exact(conn, 4), "little")
    if n > MAX_REQUEST:
        raise ProtocolError(f"request of {n} bytes (at most {MAX_REQUEST})")
    try:
        return json.loads(recv_exact(conn, n).decode("utf-8"))
    except (UnicodeDecodeError, json.JSONDecodeError) as e:
        raise ProtocolError(f"request is not UTF-8 JSON: {e}") from None


def send(conn, image, verify: bytes) -> None:
    """network_gui.send: the image bytes (when not None), then the length-prefixed verify string."""
    if image is not None:
        conn.sendall(image)
    conn.sendall(len(verify).to_bytes(4, "little") + verify)


def _matrix(values) -> torch.Tensor:
    m = torch.tensor(values, dtype=torch.float32)
    if m.numel() != 16:
        raise ProtocolError(f"a camera matrix needs 16 values; got {m.numel()}")
    return m.reshape(4, 4)


def parse(message: dict) -> Request:
    """network_gui.receive on one decoded request, on the host."""
    try:
        width, height = message["resolution_x"], message["resolution_y"]
        if type(width) is not int or type(height) is not int:
            raise ProtocolError(f"resolution must be two integers; got {width!r} x {height!r}")
        if width == 0 or height == 0:
            return Request()
        if width < 0 or height < 0:
            raise ProtocolError(f"negative resolution {width} x {height}")
        train = bool(message["train"])
        fovy, fovx = float(message["fov_y"]), float(message["fov_x"])
        znear, zfar = float(message["z_near"]), float(message["z_far"])
        shs_python, rot_scale_python = bool(message["shs_python"]), bool(message["rot_scale_python"])
        keep_alive = bool(message["keep_alive"])
        scaling_modifier = float(message["scaling_modifier"])
        world_view = _matrix(message["view_matrix"])
        world_view[:, 1] = -world_view[:, 1]
        world_view[:, 2] = -world_view[:, 2]
        full_proj = _matrix(message["view_projection_matrix"])
        full_proj[:, 1] = -full_proj[:, 1]
        cam = MiniCam(width, height, fovy, fovx, znear, zfar, world_view, full_proj)
    except ProtocolError:
        raise
    except (KeyError, TypeError, ValueError, RuntimeError) as e:
        raise ProtocolError(f"malformed camera request: {type(e).__name__}: {e}") from None
    return Request(cam, train, shs_python, rot_scale_python, keep_alive, scaling_modifier)


def serve(conn, draw: Callable[[MiniCam, float], object], verify: bytes, log: Callable[[str], None] = print) -> int:
    """Answers the requests of one connected viewer until it disconnects or sends a request the protocol cannot answer,
    then closes conn.  draw(camera, scaling_modifier) returns the frame's bytes (uint8 [H,W,3]); they are sent before
    the next request is read.  Returns the number of frames served."""
    frames = 0
    try:
        while True:
            try:
                req = parse(read(conn))
                image = None if req.camera is None else draw(req.camera, req.scaling_modifier)
                send(conn, image, verify)
            except OSError:         # the peer went away (ConnectionError included)
                log(f"viewer disconnected after {frames} frames")
                return frames
            except Exception:       # the reference drops the connection on any error (train.py:78-79)
                log(f"closing the session after {frames} frames:\n{traceback.format_exc()}")
                return frames
            frames += req.camera is not None
    finally:
        conn.close()


def request(conn, message: dict) -> tuple:
    """The viewer's side of one exchange: sends `message`, returns (image bytes or None, verify bytes), as bytearrays."""
    body = json.dumps(message).encode("utf-8")
    conn.sendall(len(body).to_bytes(4, "little") + body)
    w, h = message["resolution_x"], message["resolution_y"]
    image = recv_exact(conn, w * h * 3) if w and h else None
    return image, recv_exact(conn, int.from_bytes(recv_exact(conn, 4), "little"))


class AddressError(OSError):
    """The listener's address cannot be bound."""


def listen(ip: str, port: int) -> socket.socket:
    """network_gui.init: a TCP listener bound to (ip, port) and listening, with settimeout(0) so that accept never waits.
    Port 0 binds a free port (getsockname() names it).  An address that cannot be bound -- a busy port, an address of no
    interface -- raises AddressError naming it."""
    listener = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
    try:
        listener.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
        listener.bind((ip, port))
        listener.listen()
        listener.settimeout(0)
    except OSError as e:
        listener.close()
        raise AddressError(f"cannot listen for the remote viewer on {ip}:{port}: {e.strerror or e}") from None
    return listener


def try_connect(listener, log: Callable[[str], None] = print):
    """network_gui.try_connect: the connection of a viewer waiting on `listener` (blocking from now on), or None when no
    viewer waits."""
    try:
        conn, addr = listener.accept()
    except OSError:         # BlockingIOError: nobody waits
        return None
    log(f"\nConnected by {addr}")
    conn.settimeout(None)
    return conn


def serve_iteration(conn, draw: Callable[[MiniCam, float], object], verify: bytes, iteration: int, iterations: int,
                    log: Callable[[str], None] = print) -> tuple:
    """train.py:66-79 at one iteration: answers the viewer on `conn` (None: no viewer, return at once) until a request
    releases the iteration -- `train` and (iteration < iterations or not `keep_alive`) -- or the connection drops, which
    closes it.  draw(camera, scaling_modifier) returns a frame's bytes, as for `serve`.  Returns (conn, or None once
    dropped; the number of frames sent)."""
    frames = 0
    while conn is not None:
        try:
            req = parse(read(conn))
            image = None if req.camera is None else draw(req.camera, req.scaling_modifier)
            send(conn, image, verify)
            frames += req.camera is not None
            if req.train and (iteration < iterations or not req.keep_alive):
                break
        except Exception as e:      # train.py:78-79: conn = None, and training goes on
            if isinstance(e, OSError):
                log(f"viewer disconnected at iteration {iteration}")
            else:
                log(f"closing the viewer's connection at iteration {iteration}:\n{traceback.format_exc()}")
            conn.close()
            conn = None
    return conn, frames


class TrainingViewer:
    """The viewer of a training run: the listener `listen` binds, at most one connection, and poll() for the top of
    every iteration.  `draw` (set once the model exists) and `verify` are serve_iteration's.  `frames` counts the frames
    sent over the run."""

    def __init__(self, ip: str, port: int, verify: bytes, log: Callable[[str], None] = print):
        self.listener = listen(ip, port)
        self.address = self.listener.getsockname()[:2]
        self.verify, self.log = verify, log
        self.conn, self.draw, self.frames = None, None, 0

    def poll(self, iteration: int, iterations: int) -> None:
        """train.py:65-79: try_connect when no viewer is connected, then serve_iteration."""
        if self.conn is None:
            self.conn = try_connect(self.listener, self.log)
        self.conn, n = serve_iteration(self.conn, self.draw, self.verify, iteration, iterations, self.log)
        self.frames += n

    def close(self) -> None:
        if self.conn is not None:
            self.conn.close()
            self.conn = None
        self.listener.close()

"""Generate viewer.npz: the reference's remote-viewer protocol (renderer/gaussian_renderer/network_gui.py) on the CPU.

    python tests/golden/make_viewer_golden.py        (needs /root/reference)

network_gui's read / send / receive and scene/cameras.py's MiniCam are taken out of the reference's sources with `ast`
and executed on their own (the module's import of the scene package and its listener are left out).  Their `conn` is a
recording connection that hands out one request per test case; `.cuda()` is the identity, so every tensor stays on the
CPU.  Each reply is what train.py:67-75 sends: the image bytes of `(torch.clamp(img, 0, 1) * 255).byte().permute(1, 2,
0).contiguous()` for a seeded image (values outside [0, 1] included), when the request carries a camera, then the
verify string.

Stored per case `<c>`: `<c>/request` (the bytes the viewer sends, length prefix included), `<c>/has_camera`,
`<c>/reply` (every byte send() wrote) and `<c>/image` (the image part of it); for a camera also `<c>/world_view`,
`<c>/full_proj`, `<c>/camera_center` (float32), `<c>/size` (width, height), `<c>/fov` (fovy, fovx), `<c>/z` (znear,
zfar), `<c>/flags` (train, shs_python, rot_scale_python, keep_alive) and `<c>/scaling_modifier`.  `verify` is the
source path."""
import ast
import json
import os
import traceback

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
VERIFY = "/data/nerf_synthetic/lego"


def _source(path, names):
    tree = ast.parse(open(path).read(), path)
    body = [n for n in tree.body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and n.name in names]
    assert sorted(n.name for n in body) == sorted(names), path
    return compile(ast.Module(body=body, type_ignores=[]), path, "exec")


class RecordingConnection:
    def __init__(self, data: bytes):
        self.data, self.sent = data, bytearray()

    def recv(self, n):
        out, self.data = self.data[:n], self.data[n:]
        return out

    def sendall(self, b):
        self.sent += bytes(b)


def _view_matrix(rng):
    """A world-to-view transform in the viewer's layout: rotation in the upper 3x3, translation in the last row."""
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    m = np.eye(4)
    m[:3, :3] = q * np.sign(np.linalg.det(q))
    m[3, :3] = rng.normal(size=3) * 3.0
    return m


def _projection(fovx, fovy, znear, zfar):
    t, r = np.tan(fovy / 2) * znear, np.tan(fovx / 2) * znear
    p = np.zeros((4, 4))
    p[0, 0], p[1, 1] = znear / r, znear / t
    p[2, 2], p[2, 3] = zfar / (zfar - znear), 1.0
    p[3, 2] = -(zfar * znear) / (zfar - znear)
    return p


def _camera_message(rng, w, h, fovy, scaling_modifier, flags):
    fovx = 2 * np.arctan(np.tan(fovy / 2) * w / h)
    view = _view_matrix(rng)
    return {"resolution_x": w, "resolution_y": h, "train": flags[0], "fov_y": fovy, "fov_x": float(fovx),
            "z_near": 0.01, "z_far": 100.0, "shs_python": flags[1], "rot_scale_python": flags[2], "keep_alive": flags[3],
            "scaling_modifier": scaling_modifier, "view_matrix": view.reshape(-1).tolist(),
            "view_projection_matrix": (view @ _projection(fovx, fovy, 0.01, 100.0)).reshape(-1).tolist()}


def cases():
    rng = np.random.default_rng(7)
    first = _camera_message(rng, 7, 5, 0.8575560450553894, 1.0, (False, False, False, False))
    return (("camera", first),
            ("flags", _camera_message(rng, 4, 9, 1.2, 0.37, (True, True, True, True))),
            ("ints", dict(_camera_message(rng, 3, 2, 0.6, 2, (1, 0, 1, 0)), z_near=1, z_far=50)),
            ("zero", {"resolution_x": 0, "resolution_y": 0}),
            ("zero_width", dict(first, resolution_x=0)))


def main():
    ns = {"torch": torch, "json": json, "traceback": traceback}
    exec(_source(os.path.join(REF, "scene/cameras.py"), ["MiniCam"]), ns)
    exec(_source(os.path.join(REF, "renderer/gaussian_renderer/network_gui.py"), ["read", "send", "receive"]), ns)
    torch.Tensor.cuda = lambda self, *a, **k: self
    out = {"verify": np.frombuffer(VERIFY.encode("ascii"), np.uint8)}
    gen = torch.Generator().manual_seed(3)
    for name, msg in cases():
        body = json.dumps(msg).encode("utf-8")
        request = len(body).to_bytes(4, "little") + body
        ns["conn"] = conn = RecordingConnection(request)
        cam, train, shs, rot, keep, sm = ns["receive"]()
        assert conn.data == b""
        image = None
        if cam is not None:
            img = torch.rand(3, cam.image_height, cam.image_width, generator=gen) * 1.6 - 0.3
            image = memoryview((torch.clamp(img, min=0, max=1.0) * 255).byte().permute(1, 2, 0).contiguous().cpu().numpy())
        ns["send"](image, VERIFY)
        out[f"{name}/request"] = np.frombuffer(request, np.uint8)
        out[f"{name}/has_camera"] = np.array(cam is not None)
        out[f"{name}/reply"] = np.frombuffer(bytes(conn.sent), np.uint8)
        out[f"{name}/image"] = np.frombuffer(b"" if image is None else bytes(image), np.uint8)
        if cam is not None:
            out[f"{name}/world_view"] = cam.world_view_transform.numpy()
            out[f"{name}/full_proj"] = cam.full_proj_transform.numpy()
            out[f"{name}/camera_center"] = cam.camera_center.numpy()
            out[f"{name}/size"] = np.array([cam.image_width, cam.image_height])
            out[f"{name}/fov"] = np.array([cam.FoVy, cam.FoVx])
            out[f"{name}/z"] = np.array([cam.znear, cam.zfar], np.float64)
            out[f"{name}/flags"] = np.array([train, shs, rot, keep])
            out[f"{name}/scaling_modifier"] = np.array(sm, np.float64)
    np.savez(os.path.join(HERE, "viewer.npz"), **out)


if __name__ == "__main__":
    main()

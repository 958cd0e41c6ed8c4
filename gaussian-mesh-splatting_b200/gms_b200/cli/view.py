"""python -m gms_b200.cli.view -m <model> [--iteration N] [--gs_type T] [--ip 127.0.0.1] [--port 6009] [-w]
[--antialiasing]: serves a trained model to the SIBR remote viewer over the reference's network_gui protocol
(gms_b200.network_gui), on the native renderers.

The model directory's cfg_args is merged with the command line as get_combined_args does; --gs_type defaults to the one
cfg_args names.  The checkpoint is loaded by cli.render's load_model (gs_mesh, gs_flat, gs, gs_points, gs_multi_mesh, and
gs_flame at its checkpoint pose); no dataset image is read.  The verify string is the model's source_path.  One viewer is
served at a time; when it disconnects, or sends a request the protocol cannot answer, the program waits for the next.

A served frame (Frames) is one render on the model's native renderer, one kernel that turns the float image into the
bytes of the reference's `(torch.clamp(img, 0, 1) * 255).byte().permute(1, 2, 0).contiguous()` (gms_image_clamp_u8),
one copy into pinned host memory and one host synchronisation, for that copy; the socket sends straight from the pinned
buffer.  There is one renderer per image size, and each renders sync-free at the binning capacity its previous frame
predicts; a frame that overflowed it is drawn again at its true N before it is sent."""
from __future__ import annotations

import collections
import os
import socket
from argparse import ArgumentParser

import torch

from .. import io_image, network_gui
from . import render


def build_parser() -> ArgumentParser:
    p = render.script_parser()
    p.add_argument("--iteration", default=-1, type=int)
    p.add_argument("--gs_type", type=str, default=None)
    p.add_argument("--ip", type=str, default=network_gui.HOST)
    p.add_argument("--port", type=int, default=network_gui.PORT)
    return p


class Frames:
    """draw(camera, scaling_modifier) for network_gui.serve and serve_iteration: the frame's uint8 [H,W,3] bytes, in a
    pinned host buffer that the next call at the same size overwrites.

    The renderers read the model's tensors at every frame, so a model that changes between frames (a training run's,
    updated in place) is drawn as it is at the call.  A renderer sized for another Gaussian count than the model's (after
    densification) is replaced before it draws.  `refresh`, when given, is called before each frame to bring the model
    up to date (cli.train's gs_flame pose)."""
    SIZES = 4       # renderers kept, least recently used dropped first: resizing a viewer window asks for many sizes

    def __init__(self, model, renderer_cls, bg: torch.Tensor, antialiasing: bool = False, refresh=None):
        self.model, self.renderer_cls, self.bg, self.antialiasing = model, renderer_cls, bg, bool(antialiasing)
        self.refresh = refresh
        self.dev = bg.device
        self.sizes = collections.OrderedDict()     # (W, H) -> (renderer, device bytes [H,W,3], pinned host bytes [H,W,3])
        self._cam_host = torch.empty(35, dtype=torch.float32).pin_memory()
        self._cam_dev = torch.empty(35, dtype=torch.float32, device=self.dev)

    def _slot(self, width: int, height: int):
        key = (width, height)
        slot = self.sizes.get(key)
        if slot is None or slot[0].stale:
            slot = (self.renderer_cls(self.model, width, height),
                    torch.empty(height, width, 3, dtype=torch.uint8, device=self.dev),
                    torch.empty(height, width, 3, dtype=torch.uint8).pin_memory())
            self.sizes[key] = slot
            while len(self.sizes) > self.SIZES:
                self.sizes.popitem(last=False)
        self.sizes.move_to_end(key)
        return slot

    def __call__(self, cam: network_gui.MiniCam, scaling_modifier: float) -> memoryview:
        if self.refresh is not None:
            self.refresh()
        r, dev_u8, host_u8 = self._slot(int(cam.image_width), int(cam.image_height))
        self._cam_host.copy_(cam.packed())      # the previous frame's upload finished before its read-back
        self._cam_dev.copy_(self._cam_host, non_blocking=True)
        cam = cam.on(self._cam_dev)
        overflows = r.overflows
        r.render(cam, self.bg, scale_modifier=scaling_modifier, antialiasing=self.antialiasing)
        self._read_back(r, dev_u8, host_u8)
        n = r.last_num_rendered                 # harvests this frame's (N, overflow flag)
        if r.overflows != overflows:
            r._render(cam, self.bg, scaling_modifier, self.antialiasing, capacity=max(n, 1))
            self._read_back(r, dev_u8, host_u8)
        return memoryview(host_u8.numpy()).cast("B")

    def _read_back(self, r, dev_u8: torch.Tensor, host_u8: torch.Tensor) -> None:
        io_image.clamp_u8(r.image, out=dev_u8)
        host_u8.copy_(dev_u8, non_blocking=True)
        torch.cuda.current_stream(self.dev).synchronize()


def load(argv=None):
    """(args, Frames, verify bytes) of the command line: the merged arguments, the loaded model and its source path."""
    parser = build_parser()
    args = render.combined_args(parser, argv)
    args.gs_type = getattr(args, "gs_type", None)
    if args.gs_type is None:
        parser.error("--gs_type is not given and the model's cfg_args names none")
    if args.gs_type not in render.GS_TYPES:
        parser.error(f"--gs_type {args.gs_type} is not supported (supported: {', '.join(render.GS_TYPES)})")
    dev = render.device(parser, args, "view")
    iteration, ply = render.checkpoint(args.model_path, args.iteration)
    print(f"Loading {ply}")
    model, renderer_cls = render.load_model(args.gs_type, ply, args.sh_degree, dev)
    frames = Frames(model, renderer_cls, render.background(bool(args.white_background), dev), args.antialiasing)
    verify = os.path.abspath(args.source_path) if args.source_path else ""
    return args, frames, verify.encode("utf-8")


def main(argv=None) -> None:
    args, frames, verify = load(argv)
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as listener:
        listener.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
        listener.bind((args.ip, args.port))
        listener.listen()
        print(f"Serving {args.model_path} ({args.gs_type}) to the remote viewer on {args.ip}:{args.port}", flush=True)
        with torch.no_grad():
            while True:
                conn, addr = listener.accept()
                print(f"Connected by {addr}", flush=True)
                network_gui.serve(conn, frames, verify, log=lambda s: print(s, flush=True))


if __name__ == "__main__":
    main()

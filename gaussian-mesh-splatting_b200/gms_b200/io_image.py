"""GPU image sink / source (SURVEY.md section 8(f) rank 4).

Sink: replaces `torchvision.utils.save_image(rendering, path)` as the reference's render scripts call it once per frame
(scripts/render_time_animated.py:86-87, scripts/render.py, scripts/render_points_time_animated.py) -- there: four
full-size ATen passes (mul, add, clamp, permute+to(uint8)) on the device, a synchronous 24.9 MB fp32-equivalent transfer,
and PIL's PNG encoder on the calling thread, all serialised with the next frame's rendering.  Here:

  * ONE kernel (gms_image_quantize) writes the bytes exactly as the encoder wants them (PNG scanlines incl. the filter
    byte, or plain interleaved RGB), on the caller's stream;
  * the 6.2 MB (1080p) result goes to a ring of pinned host buffers with an asynchronous copy; an event marks it ready;
  * a small pool of host threads waits for the event, deflates (zlib releases the GIL) and writes the file, while the GPU
    renders the following frames.  `ImageSink.write()` never blocks on the GPU unless the ring is full.

Formats: "png" (byte-identical pixels to save_image's: same rounding), "ppm" (P6, no compression), "raw" (all frames
appended to ONE rawvideo file, rgb24 -- `ffmpeg -f rawvideo -pix_fmt rgb24 -s WxH -i frames.rgb ...`).

Source: `load_image_u8` / `to_device_float` keep ground-truth images 8-bit on the host (as the dataset PNGs are) and turn them into
the float [3,H,W] tensor the loss consumes with one kernel (gms_image_dequantize; ToTensor semantics,
utils/general_utils.py:105-112).
"""
from __future__ import annotations

import os
import queue
import struct
import threading
import zlib
from typing import Optional

import numpy as np
import torch

from . import _lib

_PNG_SIG = b"\x89PNG\r\n\x1a\n"


def _chunk(tag: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)


def encode_png(scanlines: bytes, width: int, height: int, channels: int = 3, level: int = 1) -> bytes:
    """`scanlines`: height rows of (1 filter byte + width*channels bytes), 8 bits per sample -> a complete PNG file."""
    color_type = {1: 0, 3: 2, 4: 6}[channels]
    ihdr = struct.pack(">IIBBBBB", width, height, 8, color_type, 0, 0, 0)
    return _PNG_SIG + _chunk(b"IHDR", ihdr) + _chunk(b"IDAT", zlib.compress(scanlines, level)) + _chunk(b"IEND", b"")


def decode_png(data: bytes) -> np.ndarray:
    """Minimal decoder for the PNGs this module writes (8-bit, non-interlaced, any filter type) -> uint8 [H,W,C]; used by the
    tests and by load_image_u8 when PIL is unavailable."""
    if data[:8] != _PNG_SIG:
        raise ValueError("not a PNG file")
    pos, idat, W = 8, [], None
    while pos < len(data):
        (n,), tag = struct.unpack(">I", data[pos:pos + 4]), data[pos + 4:pos + 8]
        body = data[pos + 8:pos + 8 + n]
        if tag == b"IHDR":
            W, H, depth, ctype, _, _, interlace = struct.unpack(">IIBBBBB", body)
            if depth != 8 or interlace != 0 or ctype not in (0, 2, 6):
                raise ValueError("unsupported PNG variant")
            C = {0: 1, 2: 3, 6: 4}[ctype]
        elif tag == b"IDAT":
            idat.append(body)
        elif tag == b"IEND":
            break
        pos += 12 + n
    raw = np.frombuffer(zlib.decompress(b"".join(idat)), np.uint8).reshape(H, 1 + W * C)
    out = np.zeros((H, W * C), np.uint8)
    prev = np.zeros(W * C, np.int32)
    for y in range(H):
        f, line = int(raw[y, 0]), raw[y, 1:].astype(np.int32)
        if f == 0:
            cur = line
        elif f == 2:
            cur = (line + prev) & 255
        else:   # Sub / Average / Paeth need the running left neighbour: plain loop (only foreign files get here)
            cur = np.zeros(W * C, np.int32)
            for i in range(W * C):
                a = cur[i - C] if i >= C else 0
                b, c = prev[i], (prev[i - C] if i >= C else 0)
                if f == 1:
                    p = a
                elif f == 3:
                    p = (a + b) // 2
                else:
                    pa, pb, pc = abs(b - c), abs(a - c), abs(a + b - 2 * c)
                    p = a if (pa <= pb and pa <= pc) else (b if pb <= pc else c)
                cur[i] = (line[i] + p) & 255
        out[y] = cur
        prev = cur
    return out.reshape(H, W, C)


def quantize(image: torch.Tensor, out: Optional[torch.Tensor] = None, row_prefix: int = 0) -> torch.Tensor:
    """float [C,H,W] CUDA -> uint8 [H, row_prefix + W*C] on the current stream (save_image's rounding)."""
    import ctypes as C
    if not image.is_cuda:
        raise RuntimeError("io_image.quantize: CUDA tensor required (no CPU path in the product)")
    img = image.detach()
    if img.dtype != torch.float32 or not img.is_contiguous():
        img = img.float().contiguous()
    Cn, H, W = img.shape
    if out is None:
        out = torch.empty((H, row_prefix + W * Cn), dtype=torch.uint8, device=img.device)
    with torch.cuda.device(img.device):
        _lib.check(_lib.lib().gms_image_quantize(img.data_ptr(), out.data_ptr(), Cn, H, W, int(row_prefix),
                                                 torch.cuda.current_stream(img.device).cuda_stream), "gms_image_quantize")
    return out


def clamp_u8(image: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """float32 [C,H,W] CUDA -> uint8 [H,W,C] = (clamp(image, 0, 1) * 255).byte().permute(1, 2, 0), bit for bit, in one
    kernel on the current stream (gms_image_clamp_u8: truncates where quantize rounds)."""
    if not (image.is_cuda and image.dtype == torch.float32 and image.is_contiguous() and image.dim() == 3):
        raise RuntimeError("io_image.clamp_u8: contiguous float32 [C,H,W] CUDA tensor required")
    Cn, H, W = image.shape
    if out is None:
        out = torch.empty((H, W, Cn), dtype=torch.uint8, device=image.device)
    if not (out.dtype == torch.uint8 and out.is_contiguous() and tuple(out.shape) == (H, W, Cn) and out.device == image.device):
        raise RuntimeError(f"io_image.clamp_u8: out must be a contiguous uint8 [{H},{W},{Cn}] tensor on {image.device}")
    with torch.cuda.device(image.device):
        _lib.check(_lib.lib().gms_image_clamp_u8(image.data_ptr(), out.data_ptr(), Cn, H, W,
                                                 torch.cuda.current_stream(image.device).cuda_stream), "gms_image_clamp_u8")
    return out


def to_device_float(image_u8: torch.Tensor, out: Optional[torch.Tensor] = None, hwc: bool = True) -> torch.Tensor:
    """uint8 CUDA image ([H,W,C] if hwc else [C,H,W]) -> float [C,H,W] = byte / 255, one kernel on the current stream."""
    if not image_u8.is_cuda or image_u8.dtype != torch.uint8:
        raise RuntimeError("io_image.to_device_float: uint8 CUDA tensor required")
    src = image_u8.contiguous()
    H, W, Cn = (src.shape if hwc else (src.shape[1], src.shape[2], src.shape[0]))
    if out is None:
        out = torch.empty((Cn, H, W), dtype=torch.float32, device=src.device)
    with torch.cuda.device(src.device):
        _lib.check(_lib.lib().gms_image_dequantize(src.data_ptr(), 1 if hwc else 0, out.data_ptr(), Cn, H, W,
                                                   torch.cuda.current_stream(src.device).cuda_stream), "gms_image_dequantize")
    return out


class GroundTruthBuffer:
    """The float [3,H,W] ground truth the loss and metric kernels read, from 8-bit [H,W,3] images (dataset.load_scene's
    resident views): byte / 255 into ONE reused device buffer per frame or renderer, in stream order.

    up_to: height x width is the largest image; a smaller [h,w,3] image lands in the buffer's first 3*h*w floats as a
    contiguous [3,h,w] tensor.  `buf` is the last image's tensor."""

    def __init__(self, height: int, width: int, device, up_to: bool = False):
        self.H, self.W, self.dev, self.up_to = int(height), int(width), torch.device(device), bool(up_to)
        self.buf = None
        self._store = None

    def __call__(self, gt_u8: torch.Tensor, who: str) -> torch.Tensor:
        shape = tuple(gt_u8.shape)
        fits = len(shape) == 3 and shape[2] == 3 and (shape[0] <= self.H and shape[1] <= self.W if self.up_to
                                                      else shape[:2] == (self.H, self.W))
        if not fits:
            want = f"at most [{self.H},{self.W},3]" if self.up_to else f"[{self.H},{self.W},3]"
            raise ValueError(f"{who}: uint8 ground truth must be {want}; got {shape}")
        if self._store is None:
            self._store = torch.empty(3 * self.H * self.W, dtype=torch.float32, device=self.dev)
        self.buf = self._store[:3 * shape[0] * shape[1]].view(3, shape[0], shape[1])
        return to_device_float(gt_u8.to(self.dev, non_blocking=True), out=self.buf, hwc=True)


def load_image_u8(path: str) -> torch.Tensor:
    """PNG / PPM file -> pinned uint8 [H,W,C] host tensor (the data-loader side of the 8-bit ground-truth path)."""
    data = open(path, "rb").read()
    if data[:8] == _PNG_SIG:
        arr = decode_png(data)
    elif data[:2] == b"P6":
        parts = data.split(maxsplit=4)
        W, H = int(parts[1]), int(parts[2])
        arr = np.frombuffer(parts[4][:W * H * 3], np.uint8).reshape(H, W, 3)
    else:
        raise ValueError(f"{path}: unsupported image format")
    t = torch.from_numpy(np.array(arr, dtype=np.uint8, order="C"))      # (owning, writable copy)
    return t.pin_memory() if torch.cuda.is_available() else t


class ImageSink:
    """Asynchronous image writer for a fixed frame size.

        sink = ImageSink(H, W, fmt="png")
        for idx, view in enumerate(views):
            rendering = render(...)["render"]
            sink.write(rendering, os.path.join(render_path, f"{idx:05d}.png"))   # returns at once
        sink.close()                                                              # waits for the files
    """

    def __init__(self, height: int, width: int, fmt: str = "png", channels: int = 3, slots: Optional[int] = None, workers: Optional[int] = None,
                 compress_level: int = 1, device="cuda", raw_path: Optional[str] = None):
        if workers is None:     # deflate is the slow part of a PNG (zlib releases the GIL): spread it over the host cores
            workers = max(2, min(16, (os.cpu_count() or 4) // 4)) if fmt == "png" else 2
        if slots is None:
            slots = workers + 2
        if fmt not in ("png", "ppm", "raw"):
            raise ValueError("fmt must be 'png', 'ppm' or 'raw'")
        self.H, self.W, self.C, self.fmt, self.level = int(height), int(width), int(channels), fmt, int(compress_level)
        self.prefix = 1 if fmt == "png" else 0
        self.dev = torch.device(device)
        row = self.prefix + self.W * self.C
        self._dev_bufs = [torch.empty((self.H, row), dtype=torch.uint8, device=self.dev) for _ in range(slots)]
        self._host_bufs = [torch.empty((self.H, row), dtype=torch.uint8).pin_memory() for _ in range(slots)]
        self._events = [torch.cuda.Event() for _ in range(slots)]
        self._free = queue.Queue()
        for i in range(slots):
            self._free.put(i)
        self._jobs = queue.Queue()
        self._errors = []
        self._raw_lock = threading.Lock()
        self._raw_next, self._raw_pending, self._seq = 0, {}, 0
        self._raw_file = None
        if fmt == "raw":
            if not raw_path:
                raise ValueError("fmt='raw' needs raw_path (one file receives every frame)")
            workers = max(1, workers)
            self._raw_file = open(raw_path, "wb")
        self._threads = [threading.Thread(target=self._worker, daemon=True) for _ in range(max(1, workers))]
        for t in self._threads:
            t.start()
        self.frames = 0

    def write(self, image: torch.Tensor, path: Optional[str] = None) -> None:
        """Queue one float [C,H,W] CUDA image.  Blocks only while all ring slots are still being encoded."""
        if tuple(image.shape) != (self.C, self.H, self.W):
            raise ValueError(f"ImageSink sized for {(self.C, self.H, self.W)}, got {tuple(image.shape)}")
        if self.fmt != "raw" and not path:
            raise ValueError("a file path is required")
        slot = self._free.get()
        stream = torch.cuda.current_stream(self.dev)
        quantize(image, self._dev_bufs[slot], self.prefix)
        self._host_bufs[slot].copy_(self._dev_bufs[slot], non_blocking=True)
        self._events[slot].record(stream)
        self._jobs.put((slot, path, self._seq))
        self._seq += 1
        self.frames += 1

    def _worker(self):
        while True:
            job = self._jobs.get()
            if job is None:
                return
            slot, path, seq = job
            try:
                self._events[slot].synchronize()
                buf = self._host_bufs[slot].numpy()
                if self.fmt == "png":
                    data = encode_png(buf.tobytes(), self.W, self.H, self.C, self.level)
                elif self.fmt == "ppm":
                    data = b"P6\n%d %d\n255\n" % (self.W, self.H) + buf.tobytes()
                else:
                    data = buf.tobytes()
                if self.fmt == "raw":
                    with self._raw_lock:        # frames leave in submission order whatever thread finishes first
                        self._raw_pending[seq] = data
                        while self._raw_next in self._raw_pending:
                            self._raw_file.write(self._raw_pending.pop(self._raw_next))
                            self._raw_next += 1
                else:
                    d = os.path.dirname(os.path.abspath(path))
                    os.makedirs(d, exist_ok=True)
                    with open(path, "wb") as f:
                        f.write(data)
            except Exception as e:  # surfaced by close()
                self._errors.append(e)
            finally:
                self._free.put(slot)

    def close(self) -> None:
        for _ in self._threads:
            self._jobs.put(None)
        for t in self._threads:
            t.join()
        if self._raw_file is not None:
            self._raw_file.close()
        if self._errors:
            raise RuntimeError(f"ImageSink: {len(self._errors)} frame(s) failed: {self._errors[0]!r}")

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def save_image(image: torch.Tensor, path: str) -> None:
    """Synchronous one-off with torchvision.utils.save_image's call shape (single [C,H,W] image)."""
    fmt = "ppm" if path.lower().endswith(".ppm") else "png"
    with ImageSink(image.shape[1], image.shape[2], fmt=fmt, channels=image.shape[0], slots=1, workers=1, device=image.device) as s:
        s.write(image, path)

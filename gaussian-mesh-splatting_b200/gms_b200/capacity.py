"""Per-view binning capacity of the sync-free frames (NativeFrame for training, NativeRenderer for rendering), and the
host side every one-call frame shares: its argument checks and its launch.

A sync-free frame does not read N (the number of tile duplicates) back before it bins: the binning region is sized for a
PREDICTED capacity, N stays on the device and the range kernel mirrors (N, overflow flag) into a ring of mapped pinned host
slots that the host polls WITHOUT synchronising.  The prediction is per view: 1.08x the N this camera had at its last visit
(more when it moved a lot between its last two visits) + 64k; a camera seen for the first time gets 1.25x the largest N
seen so far + 256k.  A frame whose N exceeds its capacity renders the background; the host notices when it harvests that
frame's slot, counts it in `overflows`, and the camera's next visit is sized from the true N."""
from __future__ import annotations

import collections
import ctypes as C

import torch


def check_float32(t: torch.Tensor, what: str, dev) -> None:
    """Raw pointers go straight to CUDA kernels: refuse a tensor that is not a contiguous float32 one on `dev`."""
    if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.device == dev):
        raise RuntimeError(f"{what} must be a contiguous float32 CUDA tensor on {dev}")


def recorded_event(ev, dev) -> torch.cuda.Event:
    """`ev`, or (when None) a new event recorded once on the current stream of `dev`, which creates its cudaEvent_t."""
    if ev is None:
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(dev))
    return ev


def grow_only_alloc(dev):
    """(scratch dict, allocation callback) for the library's scratch regions: grow-only, persistent across frames, so
    there is no allocator traffic in steady state.  `scratch["requested"]` holds the byte count of the latest request per
    region."""
    from . import _lib
    scratch = {"requested": {}}

    def _alloc(user, which, nbytes):
        scratch["requested"][int(which)] = int(nbytes)
        t = scratch.get(int(which))
        if t is None or t.numel() < nbytes:
            try:
                t = torch.empty(int(nbytes * 1.25) + (1 << 20), dtype=torch.uint8, device=dev)
            except Exception:
                return 0
            scratch[int(which)] = t
        return t.data_ptr()

    return scratch, _lib.ALLOC_FN(_alloc)      # the closure captures `scratch`/`dev` only (no reference cycle through its owner)


class SyncFreeCapacity:
    RING = 64       # mapped (N, flag) slots = frames the host may run ahead of the device before it waits

    def _init_capacity(self, sync_free: bool = True) -> None:
        self.n_rendered = C.c_int64(0)
        self.sync_free = bool(sync_free)
        self.capacity = 0                       # duplicates the most recent frame's binning region was sized for (0: not known yet)
        self.capacity_override = None           # tests: force the next frames' capacity
        self.n_host = torch.zeros(self.RING, 2, dtype=torch.int32).pin_memory()   # slot i: (N, overflow flag) of an in-flight frame
        self._n_np = self.n_host.numpy()
        self._pending = collections.deque()     # (slot, view key, capacity) of frames whose N has not been harvested yet
        self._view_n = {}                       # view key -> (N at the last visit, N at the visit before)
        self._n_max, self._n_last, self._frame_no = 0, 0, 0
        self.overflows = 0
        self._epoch, self._view_epoch = 0, {}     # frames of a view learn N once per epoch after _forget_views (epoch > 0)

    @property
    def last_num_rendered(self) -> int:
        """N of the most recent frame whose range kernel has run (no synchronisation: may lag behind the queue)."""
        if self.sync_free and self.capacity > 0:
            self._harvest()
            return self._n_last
        return int(self.n_rendered.value)

    def _harvest(self) -> None:
        """Collect (N, overflow) of the frames the device has finished binning; their slots become reusable."""
        while self._pending:
            slot, key, cap = self._pending[0]
            n = int(self._n_np[slot, 0])
            if n < 0:                       # that frame's k_tile_ranges has not run yet
                break
            self._pending.popleft()
            self._note(key, n)
            if n > cap:
                self.overflows += 1

    def _note(self, key, n: int) -> None:
        prev = self._view_n.get(key)
        self._view_n[key] = (n, prev[0] if prev else 0)
        self._n_max, self._n_last = max(self._n_max, n), n

    def _predict_capacity(self, key) -> int:
        if self.capacity_override is not None:
            return int(self.capacity_override)
        known = self._view_n.get(key)
        if known is None:
            return int(self._n_max * 1.25) + (1 << 18)
        n1, n0 = known
        drift = abs(n1 - n0) / max(n1, 1) if n0 else 0.0
        return int(n1 * (1.0 + max(0.08, 3.0 * drift))) + (1 << 16)

    @staticmethod
    def _view_key(cam):
        key = getattr(cam, "uid", None)
        return id(cam) if key is None else key

    def _sync_free_slot(self, key, dev) -> int:
        """Capacity and ring slot of the next sync-free frame of view `key`: sets self.capacity, returns the address of the
        frame's mapped (N, flag) pair."""
        self._harvest()
        if len(self._pending) >= self.RING - 1:         # the host is a whole ring ahead of the device: wait for the oldest frames
            torch.cuda.current_stream(dev).synchronize()
            self._harvest()
        slot = self._frame_no % self.RING
        self._frame_no += 1
        self.capacity = self._predict_capacity(key)
        self._n_np[slot, 0], self._n_np[slot, 1] = -1, 0
        self._pending.append((slot, key, self.capacity))
        return self.n_host.data_ptr() + 8 * slot

    def _learned_first(self, key) -> None:
        """After the one synchronising frame: its N sizes the next ones."""
        n = max(int(self.n_rendered.value), 0)
        self._note(key, n)
        self.capacity = n

    def _forget_views(self) -> None:
        """The frame changed (its Gaussian count or its workspace size): every view's next frame learns its N with one
        read-back."""
        self._harvest()
        self._epoch += 1
        self._view_n.clear()
        self._n_max = 0

    up_to = False       # True: self.W x self.H is the largest view; smaller views run at their own size (training frames)

    def _check_view(self, cam, bg, where: str = None, gt=None, gt_fits=None) -> None:
        """The camera, background (and ground truth) of a frame are float32 on the frame's device, at its image size (up_to:
        at most its image size); gt_fits(W, H), when given, tells whether the ground truth is the camera's W x H.  `where`
        names the caller in the messages (default: the class)."""
        owner = type(self).__name__
        where = where or owner
        for t, what in (() if gt is None else ((gt, "gt"),)) + ((bg, "bg"), (cam.world_view_transform, "camera matrices"),
                                                               (cam.full_proj_transform, "camera matrices"), (cam.camera_center, "camera centre")):
            if not t.is_cuda or t.device != self.dev or t.dtype != torch.float32:
                raise RuntimeError(f"{where}: {what} must be float32 on {self.dev}")
        W, H = int(cam.image_width), int(cam.image_height)
        fits = W <= self.W and H <= self.H if self.up_to else (W, H) == (self.W, self.H)
        if not fits or (gt_fits is not None and not gt_fits(W, H)):
            sized = f"for views up to {self.W}x{self.H}" if self.up_to else f"for {self.W}x{self.H}"
            raise ValueError(f"{owner} was sized {sized}; got a {cam.image_width}x{cam.image_height} camera")

    def _launch(self, fn: str, a, cam, bg, scale_modifier: float = 1.0, antialiasing: bool = False, capacity: int = None,
                n_host: int = None, debug: bool = False) -> bool:
        """Fills the settings, workspace, num_rendered and capacity fields every one-call frame's args struct shares and
        calls `fn` on the current stream.  With `capacity` (and the mapped (N, flag) address `n_host`) the frame is sync-free
        at that capacity.  Otherwise the frame is synchronising when it has to learn N (the first frame, or the view's first
        frame since _forget_views) or the frames are not sync-free, and sync-free on the next ring slot at the view's
        predicted capacity else.  The image size is the camera's.  debug: the reference's pipe.debug (settings.debug: every
        launch waited for and checked by name, the binning check on the frame's own buffers).  Returns whether the frame
        learned N."""
        from . import _lib
        s = a.settings
        s.image_height, s.image_width, s.tanfovx, s.tanfovy = int(cam.image_height), int(cam.image_width), cam.tanfovx, cam.tanfovy
        s.bg, s.scale_modifier = bg.data_ptr(), float(scale_modifier)
        s.viewmatrix, s.projmatrix, s.campos = cam.world_view_transform.data_ptr(), cam.full_proj_transform.data_ptr(), cam.camera_center.data_ptr()
        s.sh_degree, s.prefiltered, s.debug, s.antialiasing = self.model.active_sh_degree, 0, int(bool(debug)), int(bool(antialiasing))
        a.workspace, a.workspace_bytes = self.ws.data_ptr(), self.ws.numel()
        a.num_rendered = C.pointer(self.n_rendered)
        learn = False
        if capacity is None:
            key = self._view_key(cam)
            relearn = self._epoch > 0 and self._view_epoch.get(key) != self._epoch
            learn = self.sync_free and (self.capacity == 0 or relearn)
            if self.sync_free and not learn:
                n_host = self._sync_free_slot(key, self.dev)
                capacity = self.capacity
        a.binning_capacity, a.n_host_mapped = int(capacity or 0), n_host
        with torch.cuda.device(self.dev):
            _lib.check(getattr(_lib.lib(), fn)(C.byref(a), self._cb, None, torch.cuda.current_stream(self.dev).cuda_stream), fn)
        if learn:           # the synchronising frame told us N
            self._learned_first(key)
            self._view_epoch[key] = self._epoch
        return learn

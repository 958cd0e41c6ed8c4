"""FlatAdam -- the reference's Adam (gaussian_mesh_model.py:171-183, train.py:146-148) as ONE kernel launch.

All learnable tensors, their gradients and both Adam moments live in four flat fp32 buffers; `param.data` and
`param.grad` are views into them.  One launch of gms_adam_step updates everything, applies the per-group learning rates
(vertices / alpha / f_dc / f_rest / opacity / scaling, arguments_games/__init__.py:17-30) and zeroes the gradient in the
same pass.  The flat gradient buffer is also what the data-parallel all-reduce sends (trainer.py)."""
from __future__ import annotations

import ctypes as C
import math
from typing import List, Sequence, Tuple

import torch

from . import _lib

# name -> learning rate (OptimizationParamsMesh, arguments_games/__init__.py:17-30)
REFERENCE_LRS = dict(vertices=0.0, alpha=0.001, f_dc=0.0025, f_rest=0.0025 / 20.0, opacity=0.05, scaling=0.005)


class FlatAdam:
    def __init__(self, groups: Sequence[dict], betas=(0.9, 0.999), eps: float = 1e-15, world: int = 1, rank: int = 0, kernel=None,
                 sh_factored: bool = False):
        """groups: dicts with `param` and either `lr`, or (`lr0`, `lr1`, `inner`, `period`) for the packed SH tensor.
        world > 1: SHARDED optimizer (ZeRO-1 style).  The gradient exchange is a reduce-scatter, every rank keeps Adam
        moments for and updates only its 1/world slice of the flat buffer, and an all-gather brings the updated
        parameters back -- the same bytes on NVLink as an all-reduce, but the 28 B/parameter Adam pass shrinks by `world`."""
        self.groups = list(groups)
        self.world, self.rank = int(world), int(rank)
        # sh_factored: the LAST group is the packed SH tensor [P,16,3] and its gradient arrives as factors (step(sh=...)):
        # the optimizer is then REPLICATED (full moments on every rank), the exchange is an all-reduce of the other groups'
        # gradients (32 B/Gaussian) plus an all-gather of the colour gradients (12 B/Gaussian/rank), and no parameter
        # all-gather follows.  Dense mode (default): sharded optimizer, reduce-scatter + all-gather of everything.
        self.sh_factored = bool(sh_factored)
        if self.sh_factored and not ("period" in self.groups[-1] and self.groups[-1]["param"].dim() == 3):
            raise ValueError("sh_factored needs the packed SH tensor as the last group (mesh_model_groups(features_last=True))")
        params = [g["param"] for g in self.groups]
        dev = params[0].device
        pad = lambda k: (k + 63) // 64 * 64     # every segment starts 256-byte aligned (the kernels use 128-bit accesses)
        n = sum(pad(p.numel()) for p in params)
        n = (n + 64 * self.world - 1) // (64 * self.world) * (64 * self.world)     # equal, 256-byte aligned shards
        self.n = n
        self.shard = n // self.world
        self.p = torch.zeros(n, dtype=torch.float32, device=dev)
        self.g = torch.zeros(n, dtype=torch.float32, device=dev)
        nm = n if self.sh_factored else self.shard
        self.m = torch.zeros(nm, dtype=torch.float32, device=dev)      # moments: this rank's slice only (dense mode)
        self.v = torch.zeros(nm, dtype=torch.float32, device=dev)
        self.g_shard = torch.zeros(self.shard, dtype=torch.float32, device=dev) if self.world > 1 else None
        off = 0
        self.ends = []
        for p in params:
            k = p.numel()
            self.p[off:off + k].copy_(p.detach().reshape(-1))
            p.data = self.p[off:off + k].view(p.shape)
            p.grad = self.g[off:off + k].view(p.shape)
            off += pad(k)
            self.ends.append(off)
        if not self.groups or len(self._segments()[0]) > 8:
            raise ValueError("FlatAdam: gms_adam_step takes at most 8 segments of distinct hyper-parameters")
        self.betas, self.eps = betas, eps
        # Adam step count per group (torch.optim.Adam keeps one per parameter): a group whose update is skipped -- the
        # reference's reset_opacity replaces the opacity parameter by one without a gradient -- lags the others from then on
        self.steps = [0] * len(self.groups)
        self._kernel = kernel or self._cuda_kernel       # `kernel`: test hook (a callable taking the _adam_desc dict)
        self._comm = None                                # side stream of the factored exchange (created on first use)

    @property
    def t(self) -> int:
        """The step count, when every group has the same one (every mesh training path); else the largest."""
        return max(self.steps)

    @t.setter
    def t(self, value: int) -> None:
        self.steps = [int(value)] * len(self.groups)

    def group_index(self, name: str) -> int:
        return next(i for i, g in enumerate(self.groups) if g.get("name") == name)

    def _launch_runs(self, groups, zero_grad, zero_end):
        """One gms_adam_step per run of consecutive groups in `groups` with equal step counts, each over its flat sub-range
        (p/g/m/v at the run's first element, `offset` = its flat index; the segment table stays the whole buffer's)."""
        if self.world != 1:
            raise ValueError("per-group step counts need a single-GPU FlatAdam")
        runs = []
        for i in groups:
            if runs and runs[-1][-1] == i - 1 and self.steps[i] == self.steps[runs[-1][0]]:
                runs[-1].append(i)
            else:
                runs.append([i])
        for r in runs:
            off, end = (self.ends[r[0] - 1] if r[0] else 0), self.ends[r[-1]]
            d = self._adam_desc(end - off, off, self.p[off:], self.g[off:], zero_grad, zero_end)
            d.update(m=self.m[off:], v=self.v[off:], step=self.steps[r[0]])
            self._kernel(d)

    def _step_groups(self, groups, zero_end, skip):
        """Advances and updates `groups` minus the names in `skip`.  Returns False when that is every group with equal counts
        (the caller then issues its single launch)."""
        skipped = [self.group_index(n) for n in skip]
        active = [i for i in groups if i not in skipped]
        for i in active:
            self.steps[i] += 1
        for i in skipped:           # the frame's gradient of a skipped group is discarded
            self.g[(self.ends[i - 1] if i else 0):self.ends[i]].zero_()
        if not skipped and len({self.steps[i] for i in groups}) == 1:
            return False
        self._launch_runs(active, 1 if zero_end is None else 2, 0 if zero_end is None else zero_end)
        return True

    def resize(self, shapes, fill) -> None:
        """Re-homes the flat buffers for new group shapes (a densification changes every group's row count).
        fill(old, new) writes the new rows: `old` / `new` map "p", "m", "v" to per-group views of the old / new buffers in
        the group's shape.  param.data and .grad become views of the new buffers, the gradient is zero, the step counts stay."""
        if self.world != 1:
            raise ValueError("FlatAdam.resize needs a single-GPU optimizer")
        pad = lambda k: (k + 63) // 64 * 64
        ends, off = [], 0
        for sh in shapes:
            off += pad(math.prod(sh))
            ends.append(off)
        n = (off + 63) // 64 * 64
        dev = self.p.device
        new = {k: torch.zeros(n, dtype=torch.float32, device=dev) for k in ("p", "m", "v")}

        def views(bufs, ends_, shapes_):
            return {k: [b[(ends_[i - 1] if i else 0):(ends_[i - 1] if i else 0) + math.prod(sh)].view(sh) for i, sh in enumerate(shapes_)]
                    for k, b in bufs.items()}

        old_shapes = [tuple(g["param"].shape) for g in self.groups]
        fill(views({"p": self.p, "m": self.m, "v": self.v}, self.ends, old_shapes), views(new, ends, shapes))
        self.p, self.m, self.v = new["p"], new["m"], new["v"]
        self.g = torch.zeros(n, dtype=torch.float32, device=dev)
        self.n = self.shard = n
        self.ends = ends
        for i, (g, sh) in enumerate(zip(self.groups, shapes)):
            o = ends[i - 1] if i else 0
            k = math.prod(sh)
            g["param"].data = self.p[o:o + k].view(sh)
            g["param"].grad = self.g[o:o + k].view(sh)

    @property
    def flat_grad(self) -> torch.Tensor:
        return self.g

    def zero_grad(self):
        self.g.zero_()

    # ---- the three stages of a step; `step()` strings them together (tests drive them under gloo with a stub kernel)
    def _exchange_gradient(self):
        """world > 1: average the flat gradient over the ranks and return (this rank's slice of it, parameter slice, flat
        offset).  NCCL: one reduce-scatter that averages inside the collective (exact for power-of-two world sizes).
        Backends without reduce-scatter / AVG (gloo: the CPU tests): all-reduce(SUM), scale, slice."""
        import torch.distributed as dist
        off = self.rank * self.shard
        p_local = self.p[off:off + self.shard]
        if self.world <= 1:
            return self.g, self.p, 0
        if dist.get_backend() == "nccl":
            dist.reduce_scatter_tensor(self.g_shard, self.g, op=dist.ReduceOp.AVG)
        else:
            dist.all_reduce(self.g, op=dist.ReduceOp.SUM)
            self.g_shard.copy_(self.g[off:off + self.shard]).mul_(1.0 / self.world)
        return self.g_shard, p_local, off

    def _segments(self):
        """(seg_end, lr0, lr1, inner, period) of gms_adam_step: one segment per group.  With more than 8 groups (gs_flame has
        ten), neighbouring groups with the same hyper-parameters share one segment; Adam is element-wise, so the update is
        the same."""
        hp = [(float(g_.get("lr0", g_.get("lr", 0.0))), float(g_.get("lr1", g_.get("lr", 0.0))), int(g_.get("inner", 1)),
               int(g_.get("period", 0))) for g_ in self.groups]
        ends = list(self.ends)
        if len(self.groups) > 8:
            keep = [i for i in range(len(hp)) if i == len(hp) - 1 or hp[i] != hp[i + 1]]
            hp, ends = [hp[i] for i in keep], [ends[i] for i in keep]
        return [ends] + [[h[k] for h in hp] for k in range(4)]

    def _adam_desc(self, n, offset, p, g, zero_grad, zero_end):
        """Everything gms_adam_step needs, as plain Python (the stub kernel of the CPU tests reads the same dict)."""
        seg_end, lr0, lr1, inner, period = self._segments()
        return dict(n=int(n), offset=int(offset), p=p, g=g, m=self.m, v=self.v, seg_end=seg_end, lr0=lr0, lr1=lr1, inner=inner,
                    period=period, beta1=self.betas[0], beta2=self.betas[1], eps=self.eps, step=self.t, zero_grad=int(zero_grad),
                    zero_end=int(zero_end))

    def _cuda_kernel(self, d):
        a = _lib.AdamArgs()
        a.n, a.offset = d["n"], d["offset"]
        a.p, a.g, a.m, a.v = d["p"].data_ptr(), d["g"].data_ptr(), d["m"].data_ptr(), d["v"].data_ptr()
        a.nseg = len(d["seg_end"])
        for i in range(a.nseg):
            a.seg_end[i], a.lr0[i], a.lr1[i], a.inner[i], a.period[i] = d["seg_end"][i], d["lr0"][i], d["lr1"][i], d["inner"][i], d["period"][i]
        a.beta1, a.beta2, a.eps, a.step, a.zero_grad, a.zero_end = d["beta1"], d["beta2"], d["eps"], d["step"], d["zero_grad"], d["zero_end"]
        dev = d["p"].device
        if not d["p"].is_cuda:
            raise RuntimeError("FlatAdam: CUDA tensors required (no CPU path in the product)")
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gms_adam_step(C.byref(a), torch.cuda.current_stream(dev).cuda_stream), "gms_adam_step")

    def _publish_parameters(self, p_local, zero_end):
        import torch.distributed as dist
        if self.world > 1:
            dist.all_gather_into_tensor(self.p, p_local)
            (self.g if zero_end is None else self.g[:int(zero_end)]).zero_()

    def _step_factored(self, zero_end, sh):
        """sh = dict(xyz=<device pointer>, exchange=<[R, slot] float tensor: slot r = colour gradients + camera centre of rank r's frame>,
        degree=<active SH degree>)."""
        import torch.distributed as dist
        prefix = self.ends[-2]                       # everything but the SH group
        ex = sh["exchange"]
        gathered = reduced = None
        if self.world > 1:
            dev = self.p.device
            avg = dist.get_backend() == "nccl"

            def reduce_rest():
                if avg:
                    dist.all_reduce(self.g[:prefix], op=dist.ReduceOp.AVG)
                else:
                    dist.all_reduce(self.g[:prefix], op=dist.ReduceOp.SUM); self.g[:prefix].mul_(1.0 / self.world)

            if self.g.is_cuda:
                # Both collectives run from a side stream: the all-gather of the colour gradients starts right after the
                # preprocess backward (event recorded inside gms_train_frame) and overlaps the opacity / expansion backward; the
                # all-reduce of the other gradients starts when the frame is complete and overlaps k_adam_sh, which needs the
                # gather only.  k_adam (the non-SH parameters) waits for the all-reduce.
                main = torch.cuda.current_stream(dev)
                if self._comm is None:
                    self._comm = torch.cuda.Stream(dev)
                comm = self._comm
                comm.wait_event(sh["event"] if sh.get("event") is not None else main.record_event())
                with torch.cuda.stream(comm):
                    dist.all_gather_into_tensor(ex.view(-1), ex[self.rank])
                    gathered = comm.record_event()
                comm.wait_event(main.record_event())
                with torch.cuda.stream(comm):
                    reduce_rest()
                    reduced = comm.record_event()
            else:
                dist.all_gather_into_tensor(ex.view(-1), ex[self.rank])
                reduce_rest()
        if gathered is not None:
            torch.cuda.current_stream(self.p.device).wait_event(gathered)
        self._adam_sh(sh)
        if reduced is not None:
            torch.cuda.current_stream(self.p.device).wait_event(reduced)
        self.step_rest(zero_end, _advance=False)

    def step_rest(self, zero_end=None, skip=(), _advance=True):
        """Adam on every group but the SH group (one launch, gradient zeroed as in step()).  skip: names of groups that take
        no step (their step count does not advance, their gradient is discarded); with unequal counts, one launch per run."""
        if _advance and self._step_groups(range(len(self.groups) - 1), zero_end, skip):
            return
        d = self._adam_desc(self.ends[-2], 0, self.p, self.g, 1 if zero_end is None else 2, 0 if zero_end is None else zero_end)
        for k in ("seg_end", "lr0", "lr1", "inner", "period"):
            d[k] = d[k][:-1]
        d["step"] = self.steps[0]
        self._kernel(d)

    def begin_fused_sh_step(self) -> "_lib.ShAdam":
        """Single-GPU factored optimizer: the next frame applies the SH group's Adam step itself, inside its preprocess backward
        (gms_train_frame with this gms_sh_adam descriptor: the parameter rows are read once and no colour gradient goes
        through memory).  Advances the SH group's step count; step_rest() then updates the other groups."""
        if not self.sh_factored or self.world != 1:
            raise ValueError("the fused SH step needs a single-GPU FlatAdam built with sh_factored=True")
        self.steps[-1] += 1
        gsh = self.groups[-1]
        off = self.ends[-2]
        a = _lib.ShAdam()
        a.m, a.v = self.m[off:].data_ptr(), self.v[off:].data_ptr()
        a.lr_dc, a.lr_rest = float(gsh["lr0"]), float(gsh["lr1"])
        a.beta1, a.beta2, a.eps, a.step = self.betas[0], self.betas[1], self.eps, self.steps[-1]
        return a

    def _adam_sh(self, sh):
        ex = sh["exchange"]
        gsh = self.groups[-1]
        f = gsh["param"]
        off = self.ends[-2]
        a = _lib.AdamShArgs()
        a.P, a.M, a.sh_degree, a.R = f.shape[0], f.shape[1], int(sh["degree"]), ex.shape[0]
        a.xyz, a.exchange, a.slot_floats, a.grad_scale = int(sh["xyz"]), ex.data_ptr(), ex.shape[1], 1.0 / ex.shape[0]
        a.p, a.m, a.v = f.data_ptr(), self.m[off:].data_ptr(), self.v[off:].data_ptr()
        a.lr_dc, a.lr_rest = float(gsh["lr0"]), float(gsh["lr1"])
        a.beta1, a.beta2, a.eps, a.step = self.betas[0], self.betas[1], self.eps, self.steps[-1]
        dev = f.device
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gms_adam_sh_factored(C.byref(a), torch.cuda.current_stream(dev).cuda_stream), "gms_adam_sh_factored")

    def step(self, zero_end=None, sh=None, skip=()):
        """sh given (sh_factored optimizers): see _step_factored.  Otherwise:
        world == 1: one launch over the whole flat buffer (gradient zeroed in the same pass).
        world > 1: reduce-scatter(mean) -> Adam on the local slice -> all-gather of the parameters; the full gradient
        buffer is re-zeroed with one memset.
        zero_end: when the producer of the gradients OVERWRITES everything at flat indices >= zero_end each frame
        (gms_train_frame: all but the atomically accumulated vertex gradients), only [0, zero_end) is zeroed.
        skip: names of groups that take no step this time (single GPU, dense mode); while every group's step count is the
        same, the step is the one launch above, otherwise one launch per run of equal counts."""
        if skip or len(set(self.steps)) != 1:
            if self.sh_factored or not self._step_groups(range(len(self.groups)), zero_end, skip):
                raise ValueError("skipped groups / unequal step counts need a single-GPU FlatAdam in dense mode")
            return
        self.t += 1
        if self.sh_factored:
            if sh is None:
                raise ValueError("this FlatAdam was built with sh_factored=True: step() needs the SH gradient factors (sh=...)")
            return self._step_factored(zero_end, sh)
        g, p_local, off = self._exchange_gradient()
        if self.world > 1:
            d = self._adam_desc(self.shard, off, p_local, g, 0, 0)          # g_shard is overwritten by the next exchange
        else:
            d = self._adam_desc(self.n, 0, self.p, self.g, 1 if zero_end is None else 2, 0 if zero_end is None else zero_end)
        self._kernel(d)
        self._publish_parameters(p_local, zero_end)

    def zero_grad_partial(self, zero_end=None):
        (self.g if zero_end is None else self.g[:int(zero_end)]).zero_()


def mesh_model_groups(model, lrs=REFERENCE_LRS, features_last: bool = False) -> List[dict]:
    """Parameter groups of a MeshGaussianModel with the reference's learning rates; the reference's order (vertices, alpha,
    f_dc, f_rest, opacity, scaling -- gaussian_mesh_model.py:174-181), or with the packed SH tensor moved to the end
    (features_last: what FlatAdam(sh_factored=True) needs; the order of Adam groups has no numerical meaning)."""
    g = [dict(param=model.vertices, lr=lrs["vertices"], name="vertices"), dict(param=model._alpha, lr=lrs["alpha"], name="alpha")]
    feats = []
    if model._features is not None:
        M = model._features.shape[1]
        feats.append(dict(param=model._features, lr0=lrs["f_dc"], lr1=lrs["f_rest"], inner=3, period=M, name="features"))
    else:
        feats += [dict(param=model._features_dc, lr=lrs["f_dc"], name="f_dc"), dict(param=model._features_rest, lr=lrs["f_rest"], name="f_rest")]
    rest = [dict(param=model._opacity, lr=lrs["opacity"], name="opacity"), dict(param=model._scale, lr=lrs["scaling"], name="scaling")]
    return g + (rest + feats if features_last else feats + rest)


def free_model_groups(model, xyz_lr: float, feature_lr: float = 0.0025, opacity_lr: float = 0.05, scaling_lr: float = 0.005,
                      rotation_lr: float = 0.001) -> List[dict]:
    """Parameter groups of a FreeGaussianModel (gs / gs_flat) with the reference's learning rates (GaussianModel.training_setup,
    scene/gaussian_model.py:149-167; arguments/__init__.py:72-91): xyz (its lr follows the schedule), scaling, rotation,
    opacity, and the packed SH tensor last (f_dc at feature_lr, f_rest at feature_lr / 20), as FlatAdam(sh_factored=True)
    needs it.  Opacity is the last group before the SH tensor: once a lone opacity reset has made its step count lag, the
    other groups still form one run of equal counts, so the step takes two gms_adam_step launches instead of three."""
    M = model._features.shape[1]
    return [dict(param=model._xyz, lr=xyz_lr, name="xyz"), dict(param=model._scaling, lr=scaling_lr, name="scaling"),
            dict(param=model._rotation, lr=rotation_lr, name="rotation"), dict(param=model._opacity, lr=opacity_lr, name="opacity"),
            dict(param=model._features, lr0=feature_lr, lr1=feature_lr / 20.0, inner=3, period=M, name="features")]

"""CPU: FlatAdam's per-group step counts under a stub kernel.  While every group has the same count a step is the one launch
over the whole flat buffer it always was; a skipped group (the reference's lone reset_opacity) does not advance, and from
then on a step is one launch per run of consecutive groups with equal counts, over that run's flat sub-range."""
import torch
from torch import nn

from gms_b200.optim import FlatAdam


def _opt(calls, sizes=(30, 70, 5, 64, 100)):
    ps = [nn.Parameter(torch.randn(n)) for n in sizes]
    names = ["xyz", "opacity", "scaling", "rotation", "features"]
    return FlatAdam([dict(param=p, lr=0.1 * (i + 1), name=n) for i, (p, n) in enumerate(zip(ps, names))], kernel=calls.append), ps


def test_equal_counts_give_the_single_launch():
    calls = []
    opt, _ = _opt(calls)
    for t in (1, 2):
        opt.step()
        d = calls[-1]
        assert (d["n"], d["offset"], d["step"]) == (opt.n, 0, t) and d["p"] is opt.p and d["g"] is opt.g
    assert len(calls) == 2 and opt.steps == [2] * 5 and opt.t == 2


def test_skipped_group_splits_the_launch_by_runs():
    calls = []
    opt, ps = _opt(calls)
    opt.step()
    opt.g.fill_(1.0)
    opt.step(skip=("opacity",))
    assert opt.steps == [2, 1, 2, 2, 2]
    d_xyz, d_rest = calls[1:]
    assert (d_xyz["offset"], d_xyz["n"], d_xyz["step"]) == (0, opt.ends[0], 2)
    assert (d_rest["offset"], d_rest["n"], d_rest["step"]) == (opt.ends[1], opt.ends[4] - opt.ends[1], 2)
    assert d_rest["p"].data_ptr() == opt.p[opt.ends[1]:].data_ptr() and d_rest["m"].data_ptr() == opt.m[opt.ends[1]:].data_ptr()
    assert not opt.g[opt.ends[0]:opt.ends[1]].any()          # the skipped group's gradient is discarded
    calls.clear()
    opt.step()
    assert opt.steps == [3, 2, 3, 3, 3]
    assert [(d["offset"], d["step"]) for d in calls] == [(0, 3), (opt.ends[0], 2), (opt.ends[1], 3)]


def test_resize_rehomes_buffers_and_keeps_counts():
    calls = []
    opt, ps = _opt(calls, sizes=(6, 2, 4, 8, 32))
    opt.step()
    shapes = [(9,), (3,), (6,), (12,), (48,)]

    def fill(old, new):
        for k in ("p", "m", "v"):
            for o, n in zip(old[k], new[k]):
                n[:o.shape[0]] = o + (1 if k == "p" else 0)

    old_p = [p.detach().clone() for p in ps]
    opt.resize(shapes, fill)
    assert opt.steps == [1] * 5
    for p, o, sh in zip(ps, old_p, shapes):
        assert tuple(p.shape) == sh and torch.equal(p.data[:o.shape[0]], o + 1) and not p.grad.any()
        assert p.data.data_ptr() >= opt.p.data_ptr() and p.grad.data_ptr() >= opt.g.data_ptr()

"""CPU: the ATen restatement of densify_and_prune (densify_oracle.py), the xyz learning-rate schedule and the scene extent
against the reference's own outputs (tests/golden/densify.npz, make_densify_golden.py): masks, counts and row order bit
for bit."""
import types

import numpy as np
import pytest
import torch

import densify_oracle as D
from gms_b200 import scenes
from gms_b200.trainer import FreeOptimizationParams, expon_lr

EXTENT = 4.0
CASES = [(k, s) for k in ("gs", "gs_flat") for s in ("none", "20")]


@pytest.fixture(scope="module")
def gold(golden_dir):
    return dict(np.load(f"{golden_dir}/densify.npz"))


def _case(gold, tag):
    st = {k[len(tag) + 3:]: torch.from_numpy(v) for k, v in gold.items() if k.startswith(tag + "in_")}
    return st, torch.from_numpy(gold[tag + "accum"]), torch.from_numpy(gold[tag + "denom"]), torch.from_numpy(gold[tag + "normals"])


@pytest.mark.parametrize("kind,size", CASES)
def test_densify_matches_the_reference_bit_for_bit(gold, kind, size):
    tag = f"{kind}_{size}_"
    st, accum, denom, normals = _case(gold, tag)
    out, masks, counts = D.densify(st, accum, denom, normals, EXTENT, size_prune=size != "none")
    assert counts[0] == gold[tag + "out_xyz"].shape[0]
    for k, v in out.items():
        np.testing.assert_array_equal(v.numpy(), gold[tag + "out_" + k], err_msg=k)
    # every class occurs in the fixture
    assert masks["clone"].any() and masks["split"].any() and (denom == 0).any()
    assert masks["prune"].any() and (size == "none" or masks["prune_children"].any())


def test_reference_accum_is_reset_after_densification(gold):
    # densification_postfix resets the statistics (and max_radii2D) to zeros: nothing carries over
    for kind, size in CASES:
        assert not gold[f"{kind}_{size}_out_accum"].any()


def test_add_stats_restates_the_reference():
    P = 50
    g = torch.Generator().manual_seed(0)
    a, d = torch.zeros(P), torch.zeros(P)
    for _ in range(3):
        grad = torch.randn(P, 3, generator=g)
        radii = torch.randint(0, 3, (P,), generator=g)
        a2, d2 = D.add_stats(a, d, grad, radii)
        vis = radii > 0
        ref_a = a.clone()[:, None]
        ref_a[vis] += torch.norm(grad[vis, :2], dim=-1, keepdim=True)
        assert torch.equal(a2, ref_a[:, 0]) and torch.equal(d2[vis], d[vis] + 1) and torch.equal(d2[~vis], d[~vis])
        a, d = a2, d2


def test_xyz_schedule_matches_get_expon_lr_func(gold):
    o = FreeOptimizationParams()
    got = [expon_lr(int(i), o.position_lr_init * EXTENT, o.position_lr_final * EXTENT, lr_delay_mult=o.position_lr_delay_mult,
                    max_steps=o.position_lr_max_steps) for i in gold["lr_iters"]]
    np.testing.assert_array_equal(np.array(got), gold["lr_xyz"])


def test_camera_extent_matches_getNerfppNorm(gold):
    cams = []
    for R, T in zip(gold["cam_R"], gold["cam_T"]):
        W2C = np.eye(4)
        W2C[:3, :3], W2C[:3, 3] = R.T, T
        cams.append(types.SimpleNamespace(camera_center=np.linalg.inv(W2C.astype(np.float32))[:3, 3]))   # getWorld2View2 is float32
    assert scenes.camera_extent(cams) == float(gold["cam_radius"])


def test_reset_opacity_restatement(gold):
    op = torch.from_numpy(gold["reset_in_opacity"])
    x = torch.min(torch.sigmoid(op), torch.ones_like(op) * 0.01)
    np.testing.assert_array_equal(torch.log(x / (1 - x)).numpy(), gold["reset_mid_opacity"])
    assert not gold["reset_mid_m_opacity"].any() and not gold["reset_mid_v_opacity"].any()
    # the lone reset skipped the opacity group once: its step count lags by one
    assert list(gold["reset_steps"]) == [3, 3, 3, 2, 3, 3]

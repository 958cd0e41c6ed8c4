"""Softmax barycentric weights (gs_flame) on the meshes of tests/expansion_cases.py, and their float64 reference.

The same per-element comparison rule as expansion_cases.py (its module docstring), with two changes for the softmax:
  - the reference is tests/flame_reference.softmax_expand through autograd (float64, and float32 for err32);
  - cond of dL/d_alpha_j is alpha_j (G_j + sum_i alpha_i G_i), G_j = sum_c |dL/dxyz_c t_jc|: the softmax backward
    alpha_j (g_j - sum_i alpha_i g_i) is scaled by sum_i |alpha_i g_i|, not by its (possibly cancelling) value.
Logits: N(0, 2) with exact ties in 5 % of the rows, a dominant logit (+/- 1e3 apart) in 5 %, and rows far above the
range expf can take without the max subtraction (all three near 1e3)."""
from __future__ import annotations

import numpy as np
import torch

import expansion_cases as ec
import flame_reference as fr

K_VALUES = (1, 3, 7, 40, 100, 128)


def softmax_logits(rs, F, K):
    a = (2.0 * rs.randn(F, K, 3)).astype(np.float32)
    u = rs.rand(F, K)
    a[u < 0.05] = np.float32(rs.randn())                                       # three equal logits
    dom = (u >= 0.05) & (u < 0.10)
    a[dom, 0] += np.float32(1e3)                                               # one weight is 1, the others underflow to 0
    a[(u >= 0.10) & (u < 0.15)] += np.float32(1e3)                             # overflow without the max subtraction
    a[(u >= 0.15) & (u < 0.17), 1] = np.float32(-1e3)
    s = (0.8 + 0.8 * rs.randn(F * K, 1)).astype(np.float32)
    s[rs.rand(F * K) < 0.03] = 0.0
    return a, s


def build_cases():
    """(mesh name, K) for every mesh of expansion_cases.build_cases() and every K of K_VALUES, with softmax logits."""
    rs = np.random.RandomState(77)
    cases = []
    for base in ec.build_cases():
        for K in K_VALUES:
            a, s = softmax_logits(rs, base.F, K)
            c = ec.Case(f"{base.name}-K{K}", base.vertices, base.faces, a, s, seed=len(cases), max_ambiguous=base.max_ambiguous / base.F)
            c.animated = base.animated
            cases.append(c)
    return cases


def oracle_run(case, dtype):
    v = torch.tensor(case.vertices, dtype=dtype, requires_grad=True)
    a = torch.tensor(case.alpha_raw, dtype=dtype, requires_grad=True)
    s = torch.tensor(case.scale_raw, dtype=dtype, requires_grad=True)
    xyz, sl, rr, alpha, tri = fr.softmax_expand(v, torch.tensor(case.faces), a, s, ec.EPS)
    tri.retain_grad()
    ec._loss((xyz, sl, rr), case.up).backward()
    d = lambda t: t.detach().numpy().astype(np.float64)
    out = dict(alpha=d(alpha), xyz=d(xyz), scaling_log=d(sl), rotation_raw=d(rr), scaling_act=d(torch.exp(sl)),
               rotation_act=d(torch.nn.functional.normalize(rr)), dL_dalpha_raw=d(a.grad), dL_dscale_raw=d(s.grad),
               dL_dtriangles=d(tri.grad).reshape(-1, 9), dL_dvertices=d(v.grad))
    out["_rows"] = ec.oexp.face_frames(tri.detach(), ec.EPS)[0]
    t = tri.detach()
    al = alpha.detach()
    out["_cond_xyz"] = d(torch.matmul(al, t.abs()).reshape(-1, 3))
    G = torch.einsum("fkc,fjc->fkj", torch.as_tensor(case.up["dL_dxyz"]).to(dtype).reshape(case.F, case.K, 3).abs(), t.abs())
    out["_cond_alpha"] = d(al * (G + (al * G).sum(-1, keepdim=True)))
    return out


class Reference(ec.Reference):
    def __init__(self, case):
        orig = ec.oracle_run
        ec.oracle_run = oracle_run
        try:
            super().__init__(case)
        finally:
            ec.oracle_run = orig

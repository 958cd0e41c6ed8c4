"""A synthetic FLAME-shaped driver for the gs_flame tests (TEST-ONLY; the library only ever calls a driver).

FLAME (games/flame_splatting/FLAME/FLAME.py) is linear blend skinning of a template head: shape and expression blend
shapes (here n_shape + n_exp = 150 columns of a 400-column basis, as FLAME's 300 shape + 100 expression), 36 pose
features (the rotation matrices of joints 1..4 minus the identity) times pose blend shapes, five joints (global, neck, jaw,
two eyes) regressed from the shaped template, and a kinematic chain.  This driver has the same structure and call
signature on a closed UV sphere (V = 2 + rings * segments, F = 2 * segments * rings): random but fixed bases, so every
FLAME parameter moves the mesh smoothly and has a gradient.  Returns (vertices [1,V,3], landmarks = None)."""
from __future__ import annotations

import numpy as np
import torch

PARENTS = (-1, 0, 1, 1, 1)        # global -> neck -> (jaw, left eye, right eye)


def uv_sphere(rings: int, segments: int):
    """A closed sphere: two poles and `rings` rings of `segments` vertices; F = 2 * segments * rings."""
    th = np.pi * (np.arange(rings) + 1) / (rings + 1)
    ph = 2 * np.pi * np.arange(segments) / segments
    ring = np.stack([np.outer(np.sin(th), np.cos(ph)), np.outer(np.sin(th), np.sin(ph)), np.outer(np.cos(th), np.ones_like(ph))], -1)
    v = np.concatenate([[[0, 0, 1]], ring.reshape(-1, 3), [[0, 0, -1]]])
    idx = lambda r, s: 1 + r * segments + (s % segments)
    f = [[0, idx(0, s), idx(0, s + 1)] for s in range(segments)]
    for r in range(rings - 1):
        for s in range(segments):
            f += [[idx(r, s), idx(r + 1, s), idx(r + 1, s + 1)], [idx(r, s), idx(r + 1, s + 1), idx(r, s + 1)]]
    last = len(v) - 1
    f += [[last, idx(rings - 1, s + 1), idx(rings - 1, s)] for s in range(segments)]
    return v, np.asarray(f, np.int64)


def rodrigues(rv: torch.Tensor) -> torch.Tensor:
    """Axis-angle [N,3] -> rotation matrices [N,3,3] (FLAME's lbs.batch_rodrigues, with its +1e-8 in the angle)."""
    angle = torch.norm(rv + 1e-8, dim=1, keepdim=True)
    k = rv / angle
    c, s = torch.cos(angle)[:, :, None], torch.sin(angle)[:, :, None]
    z = torch.zeros_like(k[:, :1])
    K = torch.cat([z, -k[:, 2:3], k[:, 1:2], k[:, 2:3], z, -k[:, 0:1], -k[:, 1:2], k[:, 0:1], z], 1).view(-1, 3, 3)
    eye = torch.eye(3, dtype=rv.dtype, device=rv.device)[None]
    return eye + s * K + (1 - c) * torch.bmm(K, K)


class SyntheticFlame(torch.nn.Module):
    def __init__(self, rings: int = 71, segments: int = 70, n_shape: int = 100, n_exp: int = 50, seed: int = 0, scale: float = 0.1):
        super().__init__()
        rs = np.random.RandomState(seed)
        v, f = uv_sphere(rings, segments)
        V = v.shape[0]
        v = v * np.array([0.8, 1.0, 0.9]) * scale
        self.faces = f
        t = lambda a: torch.tensor(np.asarray(a), dtype=torch.float32)
        self.register_buffer("v_template", t(v))
        basis = rs.randn(V, 3, 400) * scale * 0.01                    # FLAME: 300 shape + 100 expression columns
        self.register_buffer("shapedirs", t(np.concatenate([basis[..., :n_shape], basis[..., 300:300 + n_exp]], -1)))
        self.register_buffer("posedirs", t(rs.randn(36, V * 3) * scale * 0.01))
        w = np.exp(-4 * ((v[:, None, :] / scale - rs.randn(1, 5, 3) * 0.5) ** 2).sum(-1))
        self.register_buffer("lbs_weights", t(w / w.sum(1, keepdims=True)))
        jr = rs.rand(5, V) ** 8
        self.register_buffer("J_regressor", t(jr / jr.sum(1, keepdims=True)))

    def forward(self, shape_params, expression_params, pose_params, neck_pose, transl):
        betas = torch.cat([shape_params, expression_params], 1)                              # [1,150]
        v = self.v_template + torch.einsum("vcb,b->vc", self.shapedirs, betas[0])
        J = self.J_regressor @ v                                                            # [5,3]
        eyes = torch.zeros(1, 6, dtype=pose_params.dtype, device=pose_params.device)
        full = torch.cat([pose_params[:, :3], neck_pose, pose_params[:, 3:], eyes], 1).view(5, 3)
        R = rodrigues(full)                                                                 # [5,3,3]
        feat = (R[1:] - torch.eye(3, dtype=R.dtype, device=R.device)).reshape(1, 36)
        v = v + (feat @ self.posedirs).view(-1, 3)
        G = []
        for j, p in enumerate(PARENTS):
            rel = J[j] - (J[p] if p >= 0 else 0)
            T = torch.cat([torch.cat([R[j], rel[:, None]], 1), torch.tensor([[0, 0, 0, 1.0]], dtype=R.dtype, device=R.device)], 0)
            G.append(T if p < 0 else G[p] @ T)
        G = torch.stack(G)                                                                  # [5,4,4]
        Gr = G[:, :3, :3]
        Gt = G[:, :3, 3] - torch.einsum("jab,jb->ja", Gr, J)                                # remove the rest joint position
        A_r = torch.einsum("vj,jab->vab", self.lbs_weights, Gr)
        A_t = self.lbs_weights @ Gt
        out = torch.einsum("vab,vb->va", A_r, v) + A_t + transl
        return out[None], None

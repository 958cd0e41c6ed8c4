"""FLAME's vertex model restated in float64 (TEST-ONLY): smplx.lbs.lbs as FLAME.forward calls it
(games/flame_splatting/FLAME/FLAME.py:204-248), plus transform_vertices_function
(games/flame_splatting/scene/dataset_readers.py:40-45).  Written op for op from smplx's lbs, batch_rodrigues and
batch_rigid_transform, through torch so that autograd gives every gradient.  Works in any dtype."""
from __future__ import annotations

import torch


def rodrigues(rv):
    """smplx.lbs.batch_rodrigues: [N,3] -> [N,3,3], with its +1e-8 inside the norm."""
    angle = torch.norm(rv + 1e-8, dim=1, keepdim=True)
    k = rv / angle
    c, s = torch.cos(angle)[:, :, None], torch.sin(angle)[:, :, None]
    z = torch.zeros_like(k[:, :1])
    K = torch.cat([z, -k[:, 2:3], k[:, 1:2], k[:, 2:3], z, -k[:, 0:1], -k[:, 1:2], k[:, 0:1], z], 1).view(-1, 3, 3)
    return torch.eye(3, dtype=rv.dtype, device=rv.device)[None] + s * K + (1 - c) * torch.bmm(K, K)


def joints(full_pose, J, parents):
    """Rodrigues, the pose feature and batch_rigid_transform: full_pose [5,3], J [5,3] -> (R [5,3,3], feat [36], A [5,3,4])."""
    R = rodrigues(full_pose)
    eye = torch.eye(3, dtype=R.dtype, device=R.device)
    feat = (R[1:] - eye).reshape(-1)
    G = []
    for j, p in enumerate(parents):
        rel = J[j] - (J[p] if p >= 0 else 0)
        T = torch.cat([torch.cat([R[j], rel[:, None]], 1), torch.tensor([[0, 0, 0, 1.0]], dtype=R.dtype, device=R.device)], 0)
        G.append(T if p < 0 else G[p] @ T)
    G = torch.stack(G)
    A = torch.cat([G[:, :3, :3], (G[:, :3, 3] - torch.einsum("jab,jb->ja", G[:, :3, :3], J))[:, :, None]], 2)
    return R, feat, A


def full_pose(pose, neck):
    """[pose[:3], neck, pose[3:], eye_pose = 0] as five axis-angles."""
    z = torch.zeros(6, dtype=pose.dtype, device=pose.device)
    return torch.cat([pose.reshape(-1)[:3], neck.reshape(-1), pose.reshape(-1)[3:], z]).view(5, 3)


def lbs(buf, shape, expression, pose, neck, transl):
    """FLAME.forward's vertices [V,3] (landmarks left out).  `buf`: v_template [V,3], shapedirs [V,3,B] already packed to
    the active columns (shape first), posedirs [36,3V], J_regressor [5,V], lbs_weights [V,5], parents."""
    betas = torch.cat([shape.reshape(-1), expression.reshape(-1)])
    vs = buf["v_template"] + torch.einsum("vcb,b->vc", buf["shapedirs"], betas)
    J = buf["J_regressor"] @ vs
    _, feat, A = joints(full_pose(pose, neck), J, buf["parents"])
    vp = vs + (feat @ buf["posedirs"]).view(-1, 3)
    T = torch.einsum("vj,jab->vab", buf["lbs_weights"], A)
    return torch.einsum("vab,vb->va", T[:, :, :3], vp) + T[:, :, 3] + transl.reshape(1, 3)


def transform(v, enlargement):
    """transform_vertices_function: (x, -z, y) * enlargement."""
    return torch.stack((v[:, 0], -v[:, 2], v[:, 1]), 1) * enlargement


def packed(shapedirs, n_shape, n_exp):
    """FLAME's [V,3,400] basis -> its active columns [V,3,n_shape + n_exp]; a basis already that wide is returned as is."""
    if shapedirs.shape[2] == n_shape + n_exp:
        return shapedirs
    return torch.cat([shapedirs[:, :, :n_shape], shapedirs[:, :, 300:300 + n_exp]], 2)

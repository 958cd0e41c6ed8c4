"""gs_flame references for the tests and tools (TEST-ONLY).

softmax_expand: the reference's GaussianFlameModel.update_alpha + _calc_xyz + prepare_scaling_rot
(games/flame_splatting/scene/gaussian_flame_model.py:108-206) in any dtype, through autograd: alpha = softmax(_alpha, 2),
then the mesh expansion of oracle/expansion.py.

AtenFlameArm: one reference training iteration of gs_flame the way the reference computes it -- the driver, the ATen
softmax expansion above, the activations, the library's shim rasterizer and fused loss, and torch.optim.Adam over the
reference's eleven groups (f_dc and f_rest separate)."""
from __future__ import annotations

import torch

from oracle import expansion as oexp


def softmax_expand(vertices, faces, _alpha, _scales, eps=1e-8):
    """-> xyz [P,3], _scaling [P,3] (log), _rotation [P,4] (raw), alpha [F,K,3], triangles [F,3,3]."""
    alpha = torch.softmax(_alpha, dim=2)
    triangles = vertices[faces]
    xyz = torch.matmul(alpha, triangles).reshape(-1, 3)
    _scaling, _rotation = oexp.prepare_scaling_rot(triangles, _scales, _alpha.shape[1], eps)
    return xyz, _scaling, _rotation, alpha, triangles


class AtenFlameArm:
    NAMES = ("_flame_shape", "_flame_exp", "_flame_pose", "_flame_neck_pose", "_flame_trans", "_vertices_enlargement")

    def __init__(self, model, bg, opt=None):
        """A copy of `model`'s parameters (FlameGaussianModel) trained the reference's way."""
        from gms_b200.trainer import FlameOptimizationParams
        o = opt or FlameOptimizationParams()
        self.model, self.bg, self.o = model, bg, o
        P = lambda t: torch.nn.Parameter(t.detach().clone())
        self.p = {n: P(getattr(model, n)) for n in self.NAMES + ("_alpha", "_scales", "_opacity")}
        self.p["_features_dc"] = P(model._features[:, :1])
        self.p["_features_rest"] = P(model._features[:, 1:])
        lr = dict(_flame_shape=o.flame_shape_lr, _flame_exp=o.flame_exp_lr, _flame_pose=o.flame_pose_lr,
                  _flame_neck_pose=o.flame_neck_pose_lr, _flame_trans=o.flame_trans_lr, _vertices_enlargement=o.vertices_enlargement_lr,
                  _alpha=o.alpha_lr, _features_dc=o.feature_lr, _features_rest=o.feature_lr / 20.0, _opacity=o.opacity_lr,
                  _scales=o.scaling_lr)
        self.adam = torch.optim.Adam([{"params": [self.p[n]], "lr": lr[n], "name": n} for n in lr], lr=0.0, eps=1e-15)
        self.active_sh_degree = model.active_sh_degree

    def vertices(self):
        from gms_b200.model import flame_transform_vertices
        p = self.p
        v, _ = self.model.driver(shape_params=p["_flame_shape"], expression_params=p["_flame_exp"], pose_params=p["_flame_pose"],
                                 neck_pose=p["_flame_neck_pose"], transl=p["_flame_trans"])
        return flame_transform_vertices(v, p["_vertices_enlargement"])

    def loss(self, cam, gt):
        from gms_b200.losses import fused_training_loss
        return fused_training_loss(self.render(cam), gt, self.o.lambda_dssim)

    def render(self, cam):
        import diff_gaussian_rasterization as dgr
        p = self.p
        xyz, sl, rr, _, _ = softmax_expand(self.vertices(), self.model.faces, p["_alpha"], p["_scales"], self.model.eps_s0)
        rs = dgr.GaussianRasterizationSettings(
            image_height=int(cam.image_height), image_width=int(cam.image_width), tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
            bg=self.bg, scale_modifier=1.0, viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform,
            sh_degree=self.active_sh_degree, campos=cam.camera_center, prefiltered=False, debug=False, antialiasing=False)
        means2D = torch.zeros_like(xyz, requires_grad=True)
        image, _, _ = dgr.GaussianRasterizer(raster_settings=rs)(
            means3D=xyz, means2D=means2D, opacities=torch.sigmoid(p["_opacity"]),
            shs=torch.cat((p["_features_dc"], p["_features_rest"]), 1), scales=torch.exp(sl),
            rotations=torch.nn.functional.normalize(rr))
        return image

    def step(self, cam, gt, optimizer_step=True):
        loss = self.loss(cam, gt)
        loss.backward()
        if optimizer_step:
            self.adam.step()
            self.adam.zero_grad(set_to_none=True)
        return loss.detach()

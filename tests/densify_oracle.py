"""ATen restatement of the reference's densification for free Gaussians (gs / gs_flat), pinned to tests/golden/densify.npz.

    add_densification_stats   scene/gaussian_model.py:416-418
    densify_and_prune         scene/gaussian_model.py:360-414, games/flat_splatting/scene/flat_gaussian_model.py:62-88

A state is a dict of tensors: xyz [P,3], scaling [P,C] (C = 3 gs, 2 gs_flat), rotation [P,4], opacity [P,1], features [P,M,3],
and for each of those names an Adam moment pair m_<name> / v_<name>.  The reference's clone -> split -> prune sequence
amounts to: keep the rows that are not split, append the clones, append split copy 0 of every split row, then copy 1, and
drop every row of that list that fails the prune.  Clones never split (their padded gradient is 0), and max_radii2D is all
zeros by the time the prune reads it, so only the world-size test can prune by size.  normals [P,2,3] holds the standard-normal
draws of copy 0 / copy 1 of each row (only split rows are read)."""
import torch

NAMES = ("xyz", "scaling", "rotation", "opacity", "features")


def add_stats(accum, denom, dmeans2d, radii):
    """accum / denom [P] after one frame: |dL/dmean2D.xy| and +1 where radii > 0."""
    vis = radii > 0
    accum = accum.clone()
    denom = denom.clone()
    accum[vis] += torch.norm(dmeans2d[vis, :2], dim=-1)
    denom[vis] += 1
    return accum, denom


def get_scaling(scaling, eps=1e-8):
    s = torch.exp(scaling)
    if scaling.shape[1] == 3:
        return s
    return torch.cat([torch.ones(s.shape[0], 1, dtype=s.dtype, device=s.device) * eps, s], dim=1)


def rotation_matrix(r):
    """Unit-quaternion (w, x, y, z) rotation matrices of normalise(r), [P,3,3]."""
    n = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / n[:, None]
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], dim=1)
    return R.view(-1, 3, 3)


def plan(state, accum, denom, extent, grad_threshold=0.0002, min_opacity=0.005, percent_dense=0.01, size_prune=False, eps=1e-8):
    """Masks over the P source rows: clone, split, prune (the row and its clone), prune_children."""
    g = accum / denom
    g[g.isnan()] = 0.0
    smax = torch.max(get_scaling(state["scaling"], eps), dim=1).values
    hot = g >= grad_threshold
    clone = hot & (smax <= percent_dense * extent)
    split = hot & (smax > percent_dense * extent)
    transparent = (torch.sigmoid(state["opacity"]) < min_opacity).squeeze(1)
    child_scaling = child_log_scale(state["scaling"], eps)
    prune, prune_children = transparent.clone(), transparent.clone()
    if size_prune:
        prune |= smax > 0.1 * extent
        prune_children |= torch.max(get_scaling(child_scaling, eps), dim=1).values > 0.1 * extent
    return dict(clone=clone, split=split, prune=prune, prune_children=prune_children & split)


def child_log_scale(scaling, eps=1e-8):
    c = torch.log(get_scaling(scaling, eps) / (0.8 * 2))
    return c if scaling.shape[1] == 3 else c[:, [1, 2]]


def densify(state, accum, denom, normals, extent, size_prune=False, eps=1e-8, **kw):
    """-> (new state, masks, counts [new P, kept originals, surviving clones, surviving split pairs, pruned rows])."""
    mk = plan(state, accum, denom, extent, size_prune=size_prune, eps=eps, **kw)
    clone, split, prune, prune_c = mk["clone"], mk["split"], mk["prune"], mk["prune_children"]
    keep = ~split & ~prune
    clone_keep = clone & ~prune
    split_keep = split & ~prune_c
    std = get_scaling(state["scaling"], eps)[split_keep]
    R = rotation_matrix(state["rotation"][split_keep])
    xyz0 = state["xyz"][split_keep]
    child_s = child_log_scale(state["scaling"], eps)[split_keep]
    out = {}
    for n in NAMES:
        p = state[n]
        children = [p[split_keep]] * 2
        if n == "xyz":
            children = [torch.bmm(R, (normals[split_keep, c] * std).unsqueeze(-1)).squeeze(-1) + xyz0 for c in range(2)]
        elif n == "scaling":
            children = [child_s, child_s]
        out[n] = torch.cat([p[keep], p[clone_keep]] + children)
        for mom in ("m_", "v_"):
            q = state[mom + n]
            z = torch.zeros((int(clone_keep.sum()) + 2 * int(split_keep.sum()),) + tuple(q.shape[1:]), dtype=q.dtype, device=q.device)
            out[mom + n] = torch.cat([q[keep], z])
    pruned = int((~split & prune).sum()) + int((clone & prune).sum()) + 2 * int((split & prune_c).sum())
    counts = [out["xyz"].shape[0], int(keep.sum()), int(clone_keep.sum()), int(split_keep.sum()), pruned]
    return out, mk, counts

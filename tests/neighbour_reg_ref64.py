"""Float64 reference of the neighbour regularisers (include/mgs_rasterizer.h, mgs_neighbour_reg) in torch autograd on the
CPU: padded and out-of-range slots masked, torch's own F.normalize, norm and abs giving the gradient conventions, and the
restatement of INTEGRATION.md section 17 verbatim, which the reference equals on lists without padding."""
import torch
import torch.nn.functional as F


def qmul(a, b):
    ar, ax, ay, az = a.unbind(-1)
    br, bx, by, bz = b.unbind(-1)
    return torch.stack([ar * br - ax * bx - ay * by - az * bz, ar * bx + ax * br + ay * bz - az * by,
                        ar * by - ax * bz + ay * br + az * bx, ar * bz + ax * by - ay * bx + az * br], -1)


def qrot(q):
    r, x, y, z = q.unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).view(*q.shape[:-1], 3, 3)


def _masked_norm(v, valid):
    # torch.norm's gradient at 0 is 0; invalid slots get a zero vector, so they add nothing and pass no gradient
    return torch.where(valid[..., None], v, torch.zeros_like(v)).norm(dim=-1)


def neighbour_reg_ref64(xyz, rot, xyz_next, rot_next, index, weight):
    """the definition: (rigid, rotation, isometry) as 0-dim tensors in the inputs' dtype (pass float64), differentiable in
    xyz, rot, xyz_next and rot_next"""
    P, k = index.shape
    if P == 0:
        z = xyz.sum() * 0
        return z, z.clone(), z.clone()
    valid = (index >= 0) & (index < P)
    j = torch.where(valid, index, torch.zeros_like(index))
    w = torch.where(valid, weight.to(xyz.dtype), torch.zeros_like(weight, dtype=xyz.dtype))
    q, qn = F.normalize(rot, dim=-1), F.normalize(rot_next, dim=-1)
    rel = qmul(qn, q * q.new_tensor([1.0, -1.0, -1.0, -1.0]))
    off, off_next = xyz[j] - xyz[:, None], xyz_next[j] - xyz_next[:, None]
    d = off_next - (qrot(rel)[:, None] @ off[..., None]).squeeze(-1)
    rigid = (w * _masked_norm(d, valid)).sum() / (P * k)
    rotation = (w * _masked_norm(rel[j] - rel[:, None], valid)).sum() / (P * k)
    iso = _masked_norm(off_next, valid) - _masked_norm(off, valid)
    isometry = (w * torch.where(valid, iso, torch.zeros_like(iso)).abs()).sum() / (P * k)
    return rigid, rotation, isometry


def integration_restatement(xyz, rot, xyz_next, rot_next, j, w):
    """INTEGRATION.md section 17's code, verbatim (lists without padding)"""
    q, qn = F.normalize(rot, dim=-1), F.normalize(rot_next, dim=-1)
    q_inv = q * q.new_tensor([1.0, -1.0, -1.0, -1.0])
    rel = qmul(qn, q_inv)
    off, off_next = xyz[j] - xyz[:, None], xyz_next[j] - xyz_next[:, None]
    rigid = (w[..., None] * (off_next - (qrot(rel)[:, None] @ off[..., None]).squeeze(-1))).norm(dim=-1).mean()
    rotation = (w[..., None] * (rel[j] - rel[:, None])).norm(dim=-1).mean()
    isometry = (w * (off_next.norm(dim=-1) - off.norm(dim=-1)).abs()).mean()
    return rigid, rotation, isometry

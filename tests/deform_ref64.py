"""Float64 reference of the control-graph deformation (include/mgs_rasterizer.h, mgs_deform; INTEGRATION.md section 20) in
torch autograd on the CPU: padded and out-of-range slots masked, torch's own F.normalize and torch.where giving the gradient
conventions.  It is the definition the kernels are checked against."""
import torch
import torch.nn.functional as F

from neighbour_reg_ref64 import qmul, qrot


def deform_ref64(xyz, rot, node_xyz, node_rot, node_t, index, weight):
    """the definition: (xyz' [P,3], rot' [P,4]) in the inputs' dtype (pass float64), differentiable in xyz, rot, node_xyz,
    node_rot, node_t and weight; with no nodes the cloud is returned as it is"""
    N = node_xyz.shape[0]
    if N == 0:
        return xyz, rot
    valid = (index >= 0) & (index < N)
    j = index.clamp(0, max(N - 1, 0))
    w = torch.where(valid, weight, torch.zeros_like(weight))
    q = F.normalize(node_rot, dim=-1)
    q = torch.where(q[:, :1] < 0, -q, q)
    R = qrot(q)                                                            # [N,3,3]
    c = node_xyz + node_t - (R @ node_xyz[..., None]).squeeze(-1)          # [N,3]
    moved = (R[j] @ xyz[:, None, :, None]).squeeze(-1) + c[j]              # [P,k,3]
    xyz_out = xyz + (w[..., None] * (moved - xyz[:, None])).sum(1)
    e = xyz.new_tensor([1.0, 0.0, 0.0, 0.0])
    rot_out = qmul(F.normalize(e + (w[..., None] * (q[j] - e)).sum(1), dim=-1), rot)
    return xyz_out, rot_out

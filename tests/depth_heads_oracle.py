"""numpy oracle of the depth and mask loss heads (DESIGN row f7) -- TEST INFRASTRUCTURE ONLY.

The contract, per view, from the depth plane D [H,W] (sum z_k alpha_k T_k) and the alpha plane A = 1 - final_T [H,W],
N = H * W (INTEGRATION.md §4 taken per view):
  depth  valid = (g > 0) & (A > 0.5), a constant;  d = D / A;  n = sum valid
         loss_depth = sum_valid |d - g| / n, and 0 (no gradient) when n = 0
  mask   loss_mask = mean_px BCE(clamp(A, EPS, 1 - EPS), m) exactly as torch.nn.functional.binary_cross_entropy defines it
         (logs clamped at -100, backward denominator max(a (1 - a), 1e-12)); the clamp passes the gradient only inside
         [EPS, 1 - EPS], as ATen's clamp does
The cotangent planes are those the forward blend's epilogue writes, unscaled: cot_depth = d|d - g|/dD, cot_alpha_depth =
d|d - g|/dA on valid pixels (0 elsewhere), cot_alpha_mask = d loss_mask / dA.  The losses' gradients are then
dL/dD = cot_depth / max(n, 1) and dL/dA = cot_alpha_depth / max(n, 1) + cot_alpha_mask.
Evaluated in float32 with the kernel's operation order, so that the planes can be compared element by element.
"""
import numpy as np

EPS = np.float32(1e-4)
EPS_HI = np.float32(1 - 1e-4)   # torch.clamp(A, 1e-4, 1 - 1e-4) on float32
ALPHA_MIN = np.float32(0.5)


def depth_head(D, A, g):
    """-> (loss, n, cot_depth, cot_alpha_depth) of one view"""
    D, A, g = (np.asarray(x, np.float32) for x in (D, A, g))
    valid = (g > 0) & (A > ALPHA_MIN)
    with np.errstate(divide="ignore", invalid="ignore"):
        d = np.where(valid, D / np.where(valid, A, np.float32(1)), np.float32(0)).astype(np.float32)
    s = np.sign(d - g).astype(np.float32)
    n = int(valid.sum())
    err = np.where(valid, np.abs(d - g), np.float32(0))
    loss = float(err.astype(np.float64).sum() / max(n, 1))
    safeA = np.where(valid, A, np.float32(1))
    cot_d = np.where(valid, s / safeA, np.float32(0)).astype(np.float32)
    cot_a = np.where(valid, -s * (d / safeA), np.float32(0)).astype(np.float32)
    return loss, n, cot_d, cot_a


def mask_head(A, m):
    """-> (loss, cot_alpha_mask) of one view"""
    A, m = np.asarray(A, np.float32), np.asarray(m, np.float32)
    N = A.size
    a = np.minimum(np.maximum(A, EPS), EPS_HI)
    la = np.maximum(np.log(a), np.float32(-100))
    l1a = np.maximum(np.log1p(-a), np.float32(-100))
    bce = (m - np.float32(1)) * l1a - m * la
    inside = (A >= EPS) & (A <= EPS_HI)
    grad = np.where(inside, (a - m) / np.maximum((np.float32(1) - a) * a, np.float32(1e-12)), np.float32(0))
    return float(bce.astype(np.float64).sum() / N), (grad * np.float32(1.0 / N)).astype(np.float32)


def gradients(D, A, g=None, m=None):
    """dL/dD and dL/dA of loss_depth + loss_mask (either head may be absent) from the cotangent planes"""
    dD = np.zeros(np.shape(D), np.float64)
    dA = np.zeros(np.shape(A), np.float64)
    if g is not None:
        _, n, cd, ca = depth_head(D, A, g)
        dD += cd / max(n, 1)
        dA += ca / max(n, 1)
    if m is not None:
        dA += mask_head(A, m)[1]
    return dD, dA

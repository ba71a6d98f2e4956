"""CPU oracle (numpy) of ManiGaussian's two rendering loss heads -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import this.  It restates
  l2_loss(network_output, gt)     = ((network_output - gt) ** 2).mean()                       agents/manigaussian_bc/loss.py:12-13
  cosine_loss(network_output, gt) = 1 - F.cosine_similarity(network_output, gt, dim=-1).mean()  loss.py:18-23
(F.cosine_similarity: x.y / (max(|x|, 1e-8) * max(|y|, 1e-8)), ATen) as NeuralRenderer.forward applies them to one rendered
view (neural_rendering.py:300-318), and their derivatives w.r.t. the network output.  Pinned: tests/golden/loss_heads.npz holds
outputs of the REFERENCE's own functions (lifted from loss.py with ast, run under torch autograd on the CPU by
tests/golden/make_loss_golden.py); tests/test_loss_cpu.py checks this file against them.
Images are planar like the rasterizer's outputs: render [3,H,W], embed [F,H,W].
"""
import numpy as np

EPS = 1e-8


def l2_head(render, gt):
    """-> (loss, dloss/drender)"""
    d = render.astype(np.float64) - gt.astype(np.float64)
    return float((d ** 2).mean()), (2.0 * d / d.size)


def cosine_head(embed, gt):
    """-> (loss, dloss/dembed); channel axis 0"""
    x, y = embed.astype(np.float64), gt.astype(np.float64)
    N = x[0].size
    nx, ny = np.sqrt((x * x).sum(0)), np.sqrt((y * y).sum(0))
    cx, cy = np.maximum(nx, EPS), np.maximum(ny, EPS)
    cos = (x * y).sum(0) / (cx * cy)
    # d cos / dx = y / (cx cy) - cos x / (nx cx) for nx > 0, as ATen's cosine_similarity backward (continuous at nx = eps:
    # below it the clamped norm is a constant, but nx still depends on x); 0 at x = 0
    k = np.where(nx > 0, cos / np.where(nx > 0, nx * cx, 1.0), 0.0)
    dcos = y / (cx * cy) - k * x
    return float(1.0 - cos.mean()), (-dcos / N)

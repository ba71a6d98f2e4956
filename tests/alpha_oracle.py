"""Expected values of the alpha plane (accumulated opacity 1 - final_T) from the unmodified C oracle (oracle/gs_oracle.c).

Forward: alpha = 1 - final_T of the oracle's forward.
Backward: d alpha / d a_k = T_final / (1 - a_k), which is exactly the form of the background term of dL/da_k.  So the
gradient of sum(alpha * h) is the oracle's backward of a render with zero colours, no features, background (1, 0, 0) and
colour cotangent (-h, 0, 0): per pair it evaluates dL/da_k = -T_final (1 * -h) / (1 - a_k) and nothing else.  The chain to
the per-Gaussian parameters is linear in the blend-stage gradients, so a backward with colour / feature cotangents and an
alpha cotangent is the sum of the oracle's two backwards.  tests/test_alpha_cpu.py checks this construction against
central differences of the oracle's own 1 - final_T.
"""
import numpy as np

from oracle import gs_oracle as O

# gradients an alpha cotangent reaches (through means2D, conic and opacity); the colour, SH and feature gradients do not
GEOMETRY = ("dL_dmeans2D", "dL_dconic", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dscales", "dL_drotations")


def forward(*args, **kw):
    """gs_oracle.forward() plus "alpha" [H,W] = 1 - final_T."""
    fw = O.forward(*args, **kw)
    fw["alpha"] = (np.float32(1) - fw["final_T"]).reshape(fw["H"], fw["W"])
    return fw


def backward(fw, dL_dcolor, dL_dfeature, means3D, viewmatrix, projmatrix, campos, tanfovx, tanfovy, bg, dL_dalpha=None, **kw):
    """gs_oracle.backward() with an optional alpha cotangent dL_dalpha [H,W]; keyword arguments as gs_oracle.backward."""
    g = O.backward(fw, dL_dcolor, dL_dfeature, means3D, viewmatrix, projmatrix, campos, tanfovx, tanfovy, bg, **kw)
    if dL_dalpha is None:
        return g
    P, H, W = fw["P"], fw["H"], fw["W"]
    ct = np.zeros((3, H, W), np.float32)
    ct[0] = -np.asarray(dL_dalpha, np.float32)
    trick = dict(kw, shs=None, sh_degree=0, colors_precomp=np.zeros((P, 3), np.float32), feature=None)
    a = O.backward(dict(fw, F=0, M=0), ct, None, means3D, viewmatrix, projmatrix, campos, tanfovx, tanfovy,
                   np.array([1.0, 0.0, 0.0], np.float32), **trick)
    for k in GEOMETRY:
        g[k] = g[k] + a[k].reshape(g[k].shape)
    return g

"""Float64 numpy restatement of the L1 + SSIM loss (include/mgs_rasterizer.h, mgs_view_ssim; DESIGN row f9): the values,
the per-pixel partials of S the forward kernel stores, and the gradient with respect to the rendered image.  Held to torch
float64 autograd of the reference's expression by tests/test_ssim_cpu.py; the GPU tests hold the kernels to it."""
import numpy as np

R = 5  # window radius: 11 taps
C1, C2 = 0.01 ** 2, 0.03 ** 2


def gauss1d():
    w = np.exp(-((np.arange(2 * R + 1) - R) ** 2) / 4.5)
    return w / w.sum()


def conv(p):
    """zero-padded 'same' convolution of every [H,W] plane of p [..., H, W] by the 11x11 window (separable, symmetric)"""
    w = gauss1d()
    H, W = p.shape[-2:]
    q = np.pad(p, [(0, 0)] * (p.ndim - 2) + [(R, R), (R, R)])
    h = sum(w[k] * q[..., :, k:k + W] for k in range(2 * R + 1))
    return sum(w[k] * h[..., k:k + H, :] for k in range(2 * R + 1))


def ssim_map(x, g):
    """S and its three partials {dS/dmu_x, dS/dE[x^2], dS/dE[xg]} per entry of x, g [..., H, W]"""
    x, g = np.asarray(x, np.float64), np.asarray(g, np.float64)
    mx, mg = conv(x), conv(g)
    sxx, sgg, sxg = conv(x * x) - mx * mx, conv(g * g) - mg * mg, conv(x * g) - mx * mg
    A, B = 2 * mx * mg + C1, 2 * sxg + C2
    C, D = mx * mx + mg * mg + C1, sxx + sgg + C2
    S = A * B / (C * D)
    d_mu = 2 * mg * (B - A) / (C * D) - 2 * mx * S * (1 / C - 1 / D)
    return S, d_mu, -S / D, 2 * A / (C * D)


def losses(x, g):
    """(loss_l1, ssim) of one image x, g [C,H,W]: means over its C H W entries"""
    x, g = np.asarray(x, np.float64), np.asarray(g, np.float64)
    return np.abs(x - g).mean(), ssim_map(x, g)[0].mean()


def terms(x, g):
    """the forward kernel's ssim_terms of one image [C,H,W]: [3 partials x C channels, H, W]"""
    return np.concatenate(ssim_map(x, g)[1:], 0)


def grad(x, g, g_l1=1.0, g_ssim=1.0):
    """g_l1 d loss_l1 / dx + g_ssim d ssim / dx for one image [C,H,W] (sign(0) = 0)"""
    x, g = np.asarray(x, np.float64), np.asarray(g, np.float64)
    N = x.size
    _, d_mu, d_e2, d_exg = ssim_map(x, g)
    d_ssim = (conv(d_mu) + 2 * x * conv(d_e2) + g * conv(d_exg)) / N
    return g_l1 * np.sign(x - g) / N + g_ssim * d_ssim

"""Float64 restatement of the median-contributor rule (include/mgs_rasterizer.h, mgs_view_median).

Given a pixel's pairs in list order, their alphas and its contributor mask (the forward's decisions), the transmittance before
contributor k is T_k = prod over the earlier contributors j of (1 - a_j).  The median contributor is the last contributor with
T_k > 0.5; -1 where the pixel has no contributor.  Vectorised over pixels: [n, L] arrays, exclusive cumulative products.
"""
import numpy as np

U = 2.0 ** -24


def incoming_T(alpha, mask):
    """[n, L] transmittance before every pair (the product over the earlier contributors)"""
    om = np.where(mask, 1.0 - alpha, 1.0)
    cp = np.cumprod(om, axis=1)
    return np.concatenate([np.ones((cp.shape[0], 1)), cp[:, :-1]], axis=1)


def median(alpha, mask, threshold=0.5):
    """[n] list index of each pixel's median contributor under `threshold` (T_k > threshold), -1 without a contributor"""
    cand = mask & (incoming_T(alpha, mask) > threshold)
    L = mask.shape[1]
    last = L - 1 - np.argmax(cand[:, ::-1], axis=1)
    return np.where(cand.any(1), last, -1)


def median_band(alpha, mask, ea, band=4.0):
    """(earliest, latest) [n] median index the fp32 recurrence can give: the rule at the thresholds 0.5 +- the first-order bound of
    the fp32 running product (2 + ea a / (1 - a) units u per contributor, ea the relative error of the fp32 alpha in u)"""
    rel = np.cumsum(np.where(mask, 2.0 + ea * alpha / (1.0 - alpha), 0.0), axis=1) * U * band
    T = incoming_T(alpha, mask)
    tol = np.concatenate([np.zeros((T.shape[0], 1)), rel[:, :-1]], axis=1) * T + 4 * U
    lo = np.where(mask & (T > 0.5 + tol), np.arange(mask.shape[1])[None, :], -1).max(1)
    hi = np.where(mask & (T > 0.5 - tol), np.arange(mask.shape[1])[None, :], -1).max(1)
    return lo, hi

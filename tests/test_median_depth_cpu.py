"""The median-depth plane without a GPU: the float64 rule and the C ABI's argument checks.

* tests/median_ref64.py, the vectorised float64 statement of the rule (last contributor whose incoming T > 0.5), agrees with a
  pixel-by-pixel walk on random small scenes with random contributor masks, picks the pixel's last contributor where T never
  falls to 0.5, -1 where there is no contributor, and its fp32 band always contains the exact choice.
* A median-depth output or cotangent without median_id returns MGS_ERR_INVALID_ARG
  before anything is enqueued (no device is touched: the pointers are never dereferenced).
"""
import ctypes

import numpy as np
import pytest

import util  # noqa: F401  (sys.path)
import median_ref64 as M
from manigaussian_b200 import _binding


def _walk(alpha, mask):
    """the rule, one pixel at a time: walk the contributors front to back"""
    out = []
    for a, m in zip(alpha, mask):
        T, med = 1.0, -1
        for k in range(len(a)):
            if not m[k]:
                continue
            if T > 0.5:
                med = k
            T *= 1.0 - a[k]
        out.append(med)
    return np.array(out)


@pytest.mark.parametrize("seed", range(6))
def test_vectorised_rule_matches_a_walk(seed):
    rng = np.random.default_rng(seed)
    n, L = 300, int(rng.integers(1, 40))
    alpha = rng.uniform(1 / 255, 0.99, (n, L)) ** rng.uniform(0.3, 3)
    mask = rng.random((n, L)) < rng.uniform(0.05, 0.9)
    mask[:10] = False                         # pixels without a contributor
    alpha[10:20] = 0.01                       # pixels whose T never reaches 0.5
    got = M.median(alpha, mask)
    assert np.array_equal(got, _walk(alpha, mask))
    assert (got[:10] == -1).all()
    last = np.where(mask.any(1), mask.shape[1] - 1 - np.argmax(mask[:, ::-1], 1), -1)
    thin = mask[10:20].sum(1) < 60            # 0.99^k > 0.5 for k < 69
    assert np.array_equal(got[10:20][thin], last[10:20][thin])
    has = mask.any(1)
    assert mask[np.arange(n)[has], got[has]].all()  # the choice is a contributor
    lo, hi = M.median_band(alpha, mask, np.full_like(alpha, 3.0))
    assert ((lo <= got) & (got <= hi)).all()


def test_threshold_is_strict_and_crossing_pair_is_chosen():
    # T before the pairs: 1, 0.5, 0.25: the pair entering at exactly 0.5 is not the median; the one that brought T to 0.5 is
    alpha = np.array([[0.5, 0.5, 0.5]])
    mask = np.ones_like(alpha, bool)
    assert M.median(alpha, mask)[0] == 0
    # a non-contributing pair in between changes nothing
    alpha = np.array([[0.3, 0.9, 0.3, 0.3]])
    mask = np.array([[True, False, True, True]])
    assert M.median(alpha, mask)[0] == 2 and _walk(alpha, mask)[0] == 2


# --------------------------------------------------------------------------- the C ABI
def _view():
    views = (_binding.View * 1)()
    v = views[0]
    v.width, v.height, v.tan_fovx, v.tan_fovy = 8, 8, 0.5, 0.5
    for name in ("viewmatrix", "projmatrix", "cam_pos", "background", "geometry_state", "binning_state", "image_state",
                 "radii", "dL_dpix", "blend_scratch", "out_color"):
        setattr(v, name, 4096)
    v.binning_capacity = 1
    return views


def test_median_option_checks_its_arguments():
    L = _binding.lib()
    views = _view()
    clouds = (_binding.Cloud * 1)()
    c = clouds[0]
    c.P, c.means3D, c.colors_precomp, c.opacities, c.scales, c.rotations = 4, 4096, 4096, 4096, 4096, 4096
    c.dL_dmean3D, c.dL_dopacity = 4096, 4096
    offs = (ctypes.c_int * 2)(0, 1)
    for field in ("out_median_depth", "dL_dpix_median_depth"):
        med = (_binding.ViewMedian * 1)()
        setattr(med[0], field, 4096)  # without median_id
        med = _binding.RenderOptions(median=med)
        if field == "out_median_depth":
            rc = L.mgs_forward_views(1, views, med, 4, 0, 0, 0, 4096, None, 4096, None, 4096, 4096,
                                     1.0, 4096, None, 0, 0, None)
            assert rc == -1 and "median_id" in _binding.last_error()
            rc = L.mgs_forward_clouds(1, clouds, offs, views, med, 0, 0, 0, 1.0, 0, 0, None)
            assert rc == -1 and "median_id" in _binding.last_error()
        else:
            rc = L.mgs_backward_views(1, views, med, 4, 0, 0, 0, 4096, None, 4096, None, None,
                                      1.0, None, None, 4096, 4096, None, None, None, None, None, None, 0, 0, 3, 0, None)
            assert rc == -1 and "median_id" in _binding.last_error()
            rc = L.mgs_backward_clouds(1, clouds, offs, views, med, 0, 0, 0, 1.0, 0, 0, None)
            assert rc == -1 and "median_id" in _binding.last_error()
    # the other argument checks still come first
    med = _binding.RenderOptions(median=(_binding.ViewMedian * 1)(), antialiasing=2)
    rc = L.mgs_forward_views(1, views, med, 4, 0, 0, 0, 4096, None, 4096, None, 4096, 4096, 1.0,
                             4096, None, 0, 0, None)
    assert rc == -1 and "antialiasing" in _binding.last_error()

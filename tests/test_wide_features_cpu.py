"""CPU-side checks of the feature-width limit: every entry point that blends refuses F = MGS_MAX_FEATURE_CHANNELS + 1 with
MGS_ERR_UNSUPPORTED before it enqueues any device work (the pointers below are never dereferenced)."""
import ctypes
import os
import re

import util  # noqa: F401  (sys.path)
from manigaussian_b200 import _binding

MGS_ERR_UNSUPPORTED = -2


def _max_channels():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    return int(re.search(r"#define\s+MGS_MAX_FEATURE_CHANNELS\s+(\d+)", hdr).group(1))


def test_feature_width_limit_is_512_and_documented_in_python():
    assert _max_channels() == 512
    from manigaussian_b200 import rasterizer
    assert "0..512" in rasterizer.__doc__


def test_too_wide_features_are_refused_by_every_call_without_touching_a_gpu():
    L = _binding.lib()
    F = _max_channels() + 1
    fake = ctypes.c_void_p(4096)  # a non-NULL device address: the width check comes first, nothing reads it
    cb = _binding.ALLOC_FN(lambda u, n: 0)
    rc = L.mgs_forward(cb, None, cb, None, cb, None, 10, 1, 4, F, fake, 64, 64, fake, fake, None, fake, fake, fake, 1.0, fake,
                       None, fake, fake, fake, 0.3, 0.3, 0, fake, fake, None, fake, 0, None)
    assert rc == MGS_ERR_UNSUPPORTED, _binding.last_error()
    assert str(F - 1) in _binding.last_error()
    rc = L.mgs_backward(10, 1, 4, F, 100,                    # P D M F R
                        fake, 64, 64,                        # background width height
                        fake, fake, None, fake,              # means3D shs colors feature
                        fake, 1.0, fake, None,               # scales scale_modifier rotations cov3D_precomp
                        fake, fake, fake, 0.3, 0.3,          # viewmatrix projmatrix campos tan_fovx tan_fovy
                        fake, fake, fake, fake,              # radii geometry binning image
                        fake, fake, None,                    # dL_dpix dL_dpix_F dL_dpix_depth
                        fake, None, fake, fake, fake,        # dL_dmean2D dL_dconic dL_dopacity dL_dcolor dL_dfeature
                        fake, None, fake, fake, fake,        # dL_dmean3D dL_dcov3D dL_dsh dL_dscale dL_drot
                        fake, 0, 0, None)                    # scratch accumulate debug stream
    assert rc == MGS_ERR_UNSUPPORTED, _binding.last_error()
    views = (_binding.View * 1)()
    rc = L.mgs_forward_views(1, views, None, 10, 1, 4, F, fake, fake, None, fake, fake, fake, 1.0, fake, None, 0, 0, None)
    assert rc == MGS_ERR_UNSUPPORTED, _binding.last_error()
    rc = L.mgs_backward_views(1, views, None, 10, 1, 4, F, fake, fake, None, fake, fake, 1.0, fake, None,
                              fake, fake, None, fake, None, fake, fake, fake, 1, 0, 3, 0, None)
    assert rc == MGS_ERR_UNSUPPORTED, _binding.last_error()

"""The lift without a GPU: the C ABI's struct and argument checks, lift_views' input checks, and the float64 statement of
the lift as the transpose of the feature blend.

* mgs_view_lift is one pointer, as in include/mgs_rasterizer.h.
* Every argument error of mgs_lift_views returns its code and sets mgs_last_error before anything is enqueued (the pointers
  are never dereferenced, so no device is touched).
* gaussian_renderer.lift_views raises ValueError on mismatched shapes, dtypes and devices.
* On the four golden scenes, with the C oracle's decisions, blend_ref64's dL_dfeature with the map as the cotangent is the
  transpose of its feature image: <lifted(map), f> = <map, feature(f)> to 1e-12 relative, and with a ones map <weight, f>
  = <1, feature(f)>.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import blend_ref64 as R64
import util
from manigaussian_b200 import _binding
from test_blend_ref64_cpu import GOLDEN, _golden, oracle_state


def test_view_lift_layout_matches_the_header():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    body = re.search(r"typedef struct mgs_view_lift \{(.*?)\} mgs_view_lift;", hdr, re.S).group(1)
    fields = re.findall(r"\*\s*(\w+)\s*;", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert fields == [f[0] for f in _binding.ViewLift._fields_] == ["map"]
    assert ctypes.sizeof(_binding.ViewLift) == ctypes.sizeof(ctypes.c_void_p)
    assert "mgs_lift_views" in _binding.EXPORTED_SYMBOLS and hasattr(_binding.lib(), "mgs_lift_views")


def _views(V=1):
    views = (_binding.View * V)()
    for v in views:
        v.width, v.height, v.tan_fovx, v.tan_fovy = 8, 8, 0.5, 0.5
        for name in ("viewmatrix", "projmatrix", "cam_pos", "background", "geometry_state", "binning_state", "image_state",
                     "radii"):
            setattr(v, name, 4096)
        v.binning_capacity = 1
    return views


def _call(V=1, views=None, lift="ok", aa=0, P=4, C=3, colors=4096, out_lifted=4096, out_weight=4096):
    L = _binding.lib()
    views = _views(max(V, 1)) if views is None else views
    if lift == "ok":
        lift = (_binding.ViewLift * max(V, 1))()
        for i in range(max(V, 1)):
            lift[i].map = 4096
    return L.mgs_lift_views(V, views, lift, aa, None, None, None, None, P, 0, 0, C, 4096, None, colors, 4096, 4096, 1.0, 4096, None,
                            out_lifted, out_weight, 0, None)


@pytest.mark.parametrize("case,code,msg", [
    ("V0", -1, "at least one view"),
    ("C_neg", -2, "channel count"),
    ("C_513", -2, "channel count"),
    ("no_map", -1, "map"),
    ("no_lift", -1, "mgs_view_lift"),
    ("no_lifted", -1, "out_lifted"),
    ("no_weight", -1, "out_weight"),
    ("no_geometry", -1, "state buffers"),
    ("no_image", -1, "state buffers"),
    ("no_binning", -1, "state buffers"),
    ("no_colors", -1, "colours"),
    ("aa", -1, "antialiasing"),
])
def test_lift_argument_errors_return_their_code_without_touching_a_gpu(case, code, msg):
    views = _views()
    kw = {}
    if case == "V0":
        kw["V"] = 0
    elif case == "C_neg":
        kw["C"] = -1
    elif case == "C_513":
        kw["C"] = 513
    elif case == "no_map":
        lift = (_binding.ViewLift * 1)()
        kw["lift"] = lift
    elif case == "no_lift":
        kw["lift"] = None
    elif case == "no_lifted":
        kw["out_lifted"] = None
    elif case == "no_weight":
        kw["out_weight"] = None
    elif case.startswith("no_") and case[3:] in ("geometry", "image", "binning"):
        setattr(views[0], case[3:] + "_state", None)
    elif case == "no_colors":
        kw["colors"] = None
    elif case == "aa":
        kw["aa"] = 2
    rc = _call(views=views, **kw)
    assert rc == code and msg in _binding.last_error(), (rc, _binding.last_error())


def test_lift_of_weights_only_needs_no_map_or_lifted_output():
    # C = 0 with no lift array and no lifted output passes every argument check; with V = 0 the call still fails on V,
    # so no work is enqueued
    rc = _call(V=0, lift=None, C=0, out_lifted=None)
    assert rc == -1 and "at least one view" in _binding.last_error()


def _cloud_args(P=6):
    return dict(pts_xyz=torch.zeros(P, 3), rotations=torch.zeros(P, 4), scales=torch.zeros(P, 3), opacity=torch.zeros(P, 1))


def _settings(V=2, W=8, H=6):
    from manigaussian_b200.rasterizer import GaussianRasterizationSettings
    return [GaussianRasterizationSettings(H, W, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3),
                                          False, False, False) for _ in range(V)]


@pytest.mark.parametrize("case,match", [
    ("rotations_shape", "rotations: expected"),
    ("opacity_shape", "opacity: expected"),
    ("scales_dtype", "scales: expected float32"),
    ("maps_count", "one per view"),
    ("maps_shape", r"maps\[1\]: expected"),
    ("maps_ndim", "maps: expected"),
    ("maps_dtype", r"maps\[0\]: expected float32"),
    ("maps_width", "at most 512"),
    ("device", "CUDA tensor"),
])
def test_lift_views_rejects_mismatches(case, match):
    from manigaussian_b200 import gaussian_renderer as GR
    a = _cloud_args()
    views = _settings()
    maps = torch.zeros(2, 3, 6, 8)
    if case == "rotations_shape":
        a["rotations"] = torch.zeros(6, 3)
    elif case == "opacity_shape":
        a["opacity"] = torch.zeros(5, 1)
    elif case == "scales_dtype":
        a["scales"] = a["scales"].double()
    elif case == "maps_count":
        maps = maps[:1]
    elif case == "maps_shape":
        maps = [maps[0], torch.zeros(3, 6, 9)]
    elif case == "maps_ndim":
        maps = torch.zeros(3, 6, 8)
    elif case == "maps_dtype":
        maps = maps.half()
    elif case == "maps_width":
        maps = torch.zeros(2, 513, 6, 8)
    with pytest.raises(ValueError, match=match):
        GR.lift_views(views, a["pts_xyz"], a["rotations"], a["scales"], a["opacity"], maps)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_reference_lift_is_the_transpose_of_the_feature_blend(path):
    z, inp, fw, bw = _golden(path)
    st = oracle_state(inp, fw)
    T = st["ranges"].shape[0]
    masks = [R64.decide_fp32(st, t) for t in range(T)]
    W, H, P = inp["W"], inp["H"], fw["means2D"].shape[0]
    rng = np.random.default_rng(3)
    for C, ones in ((5, False), (1, True)):
        f = rng.normal(0, 1, (P, C))
        m = np.ones((C, H, W)) if ones else rng.normal(0, 1, (C, H, W))
        ref = R64.blend(dict(st, feature=f, g_feature=m), masks)
        lhs = float((ref["dL_dfeature"] * f).sum())
        rhs = float((m * ref["feature"]).sum())
        scale = float((np.abs(ref["dL_dfeature"]) * np.abs(f)).sum())
        assert scale > 0 and abs(lhs - rhs) <= 1e-12 * scale, (C, lhs, rhs)
        if ones:
            # weight = sum_p w_pg, and summed over the Gaussians it is the alpha plane's sum
            assert abs(ref["dL_dfeature"][:, 0].sum() - ref["alpha"].sum()) <= 1e-12 * ref["alpha"].sum()

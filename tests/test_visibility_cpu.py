"""Point visibility without a GPU: the float64 statement (tests/visibility_ref64.py) on the golden scenes, the C ABI's exports
and argument checks, and point_visibility's input checks.

* At every pixel centre, behind the scene, the reference's T is blend_ref64's final_T of the same state (float64 decisions)
  wherever neither has a borderline decision; in front of the scene it is 1.
* Along a ray T does not increase with the depth, for all four camera models.
* in_view at the -0.5 and W - 0.5 edges.
* Every argument error of mgs_visibility_views returns its code and sets mgs_last_error before anything is enqueued (the
  pointers are never dereferenced, so no device is touched).
"""
import os

import numpy as np
import pytest
import torch

import blend_ref64 as R64
import util
import visibility_ref64 as V64
from manigaussian_b200 import _binding
from test_blend_ref64_cpu import GOLDEN, _golden, oracle_state


def _state(path):
    z, inp, fw, bw = _golden(path)
    st = dict(oracle_state(inp, fw), depths=np.asarray(fw["depths"], np.float64))
    return inp, fw, st


def _pixel_centres(W, H):
    yy, xx = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    return np.stack([xx.ravel(), yy.ravel()], 1)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_reference_gives_final_T_behind_the_scene_and_one_in_front(path):
    inp, fw, st = _state(path)
    W, H = inp["W"], inp["H"]
    uv = _pixel_centres(W, H)
    inside = np.ones(len(uv), bool)
    T, border = V64.transmittance(st, uv, np.full(len(uv), np.inf), inside)
    nt = st["ranges"].shape[0]
    dec = [R64.decide(st, t) for t in range(nt)]
    ref = R64.blend(dict(st, feature=None), [d["mask"] for d in dec], backward=False)["final_T"].ravel()
    # pixels whose float64 decisions are all clear of the fp32 bands, in blend_ref64's and in this reference's terms
    clear = np.zeros((H, W), bool)
    for t, d in enumerate(dec):
        px, py, ins = R64.tile_pixels(W, H, t)
        clear[py[ins], px[ins]] = d["first_border"][ins] == d["mask"].shape[1]
    ok = clear.ravel() & ~border
    assert ok.mean() > 0.9
    assert np.abs(T[ok] - ref[ok]).max() <= 1e-12
    assert (T < 1).sum() > len(T) // 4  # the scene covers the image
    # the oracle's fp32 final_T agrees to its rounding
    assert np.abs(T[ok] - np.asarray(fw["final_T"], np.float64).ravel()[ok]).max() <= 1e-5
    front, _ = V64.transmittance(st, uv, np.full(len(uv), 0.1), inside)  # in front of the near plane's every Gaussian
    assert (front == 1.0).all()


def _model_view(inp, model):
    from test_planar_depth_gpu import _model_kw
    return _model_kw(inp, model)[1]


@pytest.mark.parametrize("model", ["pinhole", "ortho", "fisheye", "distorted"])
def test_transmittance_does_not_increase_along_a_ray(model):
    inp, fw, st = _state(GOLDEN[0])
    view = _model_view(inp, model)
    vm = np.asarray(view["viewmatrix"], np.float64).reshape(4, 4).T  # world -> view, column vectors
    c2w = np.linalg.inv(vm)
    rng = np.random.default_rng(1)
    dirs = np.concatenate([rng.uniform(-0.4, 0.4, (40, 2)), np.ones((40, 1))], 1)
    depths = np.linspace(0.3, 12.0, 60)
    for dvec in dirs:
        if model == "ortho":  # rays of an orthographic view are parallel to its z axis
            t = np.stack([np.full_like(depths, dvec[0]), np.full_like(depths, dvec[1]), depths], 1)
        else:
            t = depths[:, None] * dvec[None, :]
        world = t @ c2w[:3, :3].T + c2w[:3, 3]
        uv, d, ok = V64.project(world, view)
        inside = V64.in_view(uv, ok, inp["W"], inp["H"])
        if not inside.any():
            continue
        # the ray stays on one screen position (up to the projection's w + 1e-7, ~1e-7 / z px), and at that position T does
        # not increase with d
        u0 = uv[inside][0]
        assert np.abs(uv[inside] - u0).max() < 1e-4, (model, dvec)
        T, _ = V64.transmittance(st, np.broadcast_to(u0, uv.shape), d, inside)
        Tin = T[inside]
        assert np.all(np.diff(Tin) <= 0.0), (model, dvec, Tin)
        assert Tin[0] == 1.0 or d[inside][0] > st["depths"].min()
        assert np.allclose(d[ok], t[ok, 2], rtol=1e-12)


def test_in_view_edges():
    W, H = 40, 24
    e = 1e-9
    uv = np.array([[-0.5, 3.0], [-0.5 - e, 3.0], [W - 0.5, 3.0], [W - 0.5 - e, 3.0],
                   [3.0, -0.5], [3.0, -0.5 - e], [3.0, H - 0.5], [3.0, H - 0.5 - e], [np.nan, np.nan]])
    ok = np.array([True] * 8 + [False])
    assert V64.in_view(uv, ok, W, H).tolist() == [True, False, False, True, True, False, False, True, False]
    # the last pixel column and row of the image belong to the last tile
    assert V64.tile_of(uv[[3, 7]], W, H).tolist() == [((3 + 0) // 16) * 3 + 2, ((H - 1) // 16) * 3 + 0]


def test_symbols_are_declared_and_exported():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    L = _binding.lib()
    for sym in ("mgs_visibility_views", "mgs_visibility_scratch_bytes"):
        assert f"{sym}(" in hdr and sym in _binding.EXPORTED_SYMBOLS and hasattr(L, sym)
    a, b = L.mgs_visibility_scratch_bytes(1000, 128, 128), L.mgs_visibility_scratch_bytes(2000, 128, 128)
    assert b > a >= 1000 * (16 + 16)


def _views(V=1):
    views = (_binding.View * V)()
    for v in views:
        v.width, v.height, v.tan_fovx, v.tan_fovy = 8, 8, 0.5, 0.5
        for name in ("viewmatrix", "projmatrix", "cam_pos", "background", "geometry_state", "binning_state", "image_state",
                     "blend_scratch", "radii"):
            setattr(v, name, 4096)
        v.binning_capacity = 1
    return views


def _call(V=1, views=None, aa=0, ortho=None, fisheye=None, P=4, Q=3, points=4096, colors=4096, out_T=4096):
    L = _binding.lib()
    views = _views(max(V, 1)) if views is None else views
    return L.mgs_visibility_views(V, views, aa, None, ortho, fisheye, None, P, 0, 0, Q, points, 4096, None, colors, 4096, 4096, 1.0,
                                  4096, None, None, None, None, out_T, 0, None)


@pytest.mark.parametrize("case,code,msg", [
    ("V0", -1, "at least one view"),
    ("Q_neg", -1, "Q must be"),
    ("no_points", -1, "points"),
    ("no_T", -1, "out_T"),
    ("P0", -1, "P must be"),
    ("no_geometry", -1, "state buffers"),
    ("no_scratch", -1, "blend_scratch"),
    ("no_radii", -1, "radii"),
    ("no_colors", -1, "colours"),
    ("aa", -1, "antialiasing"),
    ("ortho", -1, "ortho"),
    ("fisheye", -1, "theta_max"),
])
def test_invalid_arguments_return_error_codes_without_touching_a_gpu(case, code, msg):
    views = _views()
    kw = {}
    if case == "V0":
        kw["V"] = 0
    elif case == "Q_neg":
        kw["Q"] = -1
    elif case == "no_points":
        kw["points"] = None
    elif case == "no_T":
        kw["out_T"] = None
    elif case == "P0":
        kw["P"] = 0
    elif case == "no_geometry":
        views[0].geometry_state = None
    elif case == "no_scratch":
        views[0].blend_scratch = None
    elif case == "no_radii":
        views[0].radii = None
    elif case == "no_colors":
        kw["colors"] = None
    elif case == "aa":
        kw["aa"] = 2
    elif case == "ortho":
        kw["ortho"] = (ctypes_int * 1)(2)
    elif case == "fisheye":
        fe = (_binding.ViewFisheye * 1)()
        fe[0].fisheye, fe[0].theta_max = 1, 2.0
        kw["fisheye"] = fe
    rc = _call(views=views, **kw)
    assert rc == code and msg in _binding.last_error(), (rc, _binding.last_error())


def test_zero_points_is_a_no_op():
    # every check passes and nothing is enqueued (the pointers are never dereferenced)
    assert _call(Q=0, points=None) == 0


ctypes_int = __import__("ctypes").c_int


def _cloud(P=6):
    return dict(pts_xyz=torch.zeros(P, 3), rotations=torch.zeros(P, 4), scales=torch.zeros(P, 3), opacity=torch.zeros(P, 1))


def _settings(V=2, W=8, H=6):
    from manigaussian_b200.rasterizer import GaussianRasterizationSettings
    return [GaussianRasterizationSettings(H, W, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3),
                                          False, False, False) for _ in range(V)]


@pytest.mark.parametrize("case,match", [
    ("rotations_shape", "rotations: expected"),
    ("opacity_shape", "opacity: expected"),
    ("scales_dtype", "scales: expected float32"),
    ("points_shape", r"points: expected \[Q,3\]"),
    ("points_dtype", "points: expected float32"),
    ("no_views", "at least one view"),
    ("device", "CUDA tensor"),
])
def test_point_visibility_rejects_mismatches(case, match):
    from manigaussian_b200 import gaussian_renderer as GR
    a = _cloud()
    views = _settings()
    pts = torch.zeros(5, 3)
    if case == "rotations_shape":
        a["rotations"] = torch.zeros(6, 3)
    elif case == "opacity_shape":
        a["opacity"] = torch.zeros(5, 1)
    elif case == "scales_dtype":
        a["scales"] = a["scales"].double()
    elif case == "points_shape":
        pts = torch.zeros(5, 2)
    elif case == "points_dtype":
        pts = pts.double()
    elif case == "no_views":
        views = []
    with pytest.raises(ValueError, match=match):
        GR.point_visibility(views, pts, a["pts_xyz"], a["rotations"], a["scales"], a["opacity"])

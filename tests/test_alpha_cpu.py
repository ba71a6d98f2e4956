"""The alpha plane (accumulated opacity 1 - final_T) without a GPU: the C ABI declares its struct and options field while
the existing view and cloud structs keep their layouts, and the alpha expectations built from the C oracle
(tests/alpha_oracle.py) are right: the plane against the reference's stored final_T, the gradient against central
differences of the oracle's own 1 - final_T."""
import ctypes
import glob
import json
import os
import re

import numpy as np
import pytest

import util
from manigaussian_b200 import _binding
import alpha_oracle as A

# mgs_view as C callers compiled against ABI 300 hold it: the alpha plane must not move a field
VIEW_FIELDS = ("viewmatrix", "projmatrix", "cam_pos", "background", "tan_fovx", "tan_fovy", "width", "height", "geometry_state",
               "binning_state", "image_state", "binning_capacity", "out_color", "out_feature", "out_depth", "radii", "status",
               "dL_dpix", "dL_dpix_F", "dL_dpix_depth", "blend_scratch", "dL_dmean2D", "stream", "target_color", "target_feature",
               "cot_color", "cot_feature", "loss_acc", "cot_scale")


def test_header_declares_the_alpha_struct_and_option():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    code = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    assert re.search(r"typedef struct mgs_view_alpha \{\s*float\* out_alpha;\s*const float\* dL_dpix_alpha;\s*\} mgs_view_alpha;", code)
    assert re.search(r"typedef struct mgs_render_options \{[^}]*const mgs_view_alpha\* alpha;", code)
    assert [f for f, _ in _binding.ViewAlpha._fields_] == ["out_alpha", "dL_dpix_alpha"]
    assert ctypes.sizeof(_binding.ViewAlpha) == 2 * ctypes.sizeof(ctypes.c_void_p)


def test_view_and_cloud_layouts_are_unchanged():
    assert tuple(f for f, _ in _binding.View._fields_) == VIEW_FIELDS
    ptr, i32, f32 = ctypes.sizeof(ctypes.c_void_p), 4, 4
    # 4 pointers, 2 floats + 2 ints, 3 pointers, 1 int (padded), 4 pointers, 1 pointer (status), 6 pointers, 6 pointers
    assert ctypes.sizeof(_binding.View) == 4 * ptr + 2 * f32 + 2 * i32 + 3 * ptr + ptr + 4 * ptr + ptr + 6 * ptr + 6 * ptr
    assert ctypes.sizeof(_binding.Cloud) == 17 * ptr


def test_alpha_option_checks_its_arguments_without_a_gpu():
    L = _binding.lib()
    views = (_binding.View * 1)()
    alpha = _binding.RenderOptions(alpha=(_binding.ViewAlpha * 1)())
    rc = L.mgs_forward_views(0, views, alpha, 10, 1, 4, 0, None, None, None, None, None, None, 1.0, None, None, 0, 0, None)
    assert rc < 0 and _binding.last_error()
    rc = L.mgs_backward_views(1, views, alpha, 0, 1, 4, 0, None, None, None, None, None, 1.0, None, None,
                              None, None, None, None, None, None, None, None, 1, 0, 3, 0, None)
    assert rc < 0
    offs = (ctypes.c_int * 2)(0, 1)
    clouds = (_binding.Cloud * 1)()
    assert L.mgs_forward_clouds(0, clouds, offs, views, alpha, 1, 4, 0, 1.0, 0, 0, None) < 0
    assert L.mgs_backward_clouds(1, clouds, offs, views, None, 1, 4, 0, 1.0, 0, 0, None) < 0  # P = 0


GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "g[0-9]*.npz")))


def _oracle(inp, dL_dcolor, dL_dfeature, dL_dalpha=None, backward=True):
    g, cam = inp["g"], inp["cam"]
    kw = dict(scales=g["scales"], rotations=g["rotations"], cov3D_precomp=g["cov3D_precomp"], shs=g["shs"], sh_degree=g["sh_degree"],
              colors_precomp=g["colors_precomp"], feature=g["feature"])
    fw = A.forward(g["means3D"], g["opacities"], cam["viewmatrix"], cam["projmatrix"], cam["campos"], inp["W"], inp["H"],
                   cam["tanfovx"], cam["tanfovy"], inp["bg"], **kw)
    if not backward:
        return fw, None
    bw = A.backward(fw, dL_dcolor, dL_dfeature, g["means3D"], cam["viewmatrix"], cam["projmatrix"], cam["campos"], cam["tanfovx"],
                    cam["tanfovy"], inp["bg"], dL_dalpha=dL_dalpha, **kw)
    return fw, bw


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_oracle_alpha_is_one_minus_final_T(path):
    z = np.load(path)
    kw = json.loads(bytes(z["recipe"]).decode())
    if "bg" in kw:
        kw["bg"] = tuple(kw["bg"])
    inp = util.make_inputs(**kw)
    fw, _ = _oracle(inp, None, None, backward=False)
    H, W = inp["H"], inp["W"]
    assert fw["alpha"].shape == (H, W) and fw["alpha"].dtype == np.float32
    assert np.array_equal(fw["alpha"], (np.float32(1) - fw["final_T"]).reshape(H, W))
    assert util.rel_l2(fw["alpha"], 1 - z["fw_final_T"].reshape(H, W)) < 1e-4
    assert fw["alpha"].min() >= 0 and fw["alpha"].max() <= np.float32(1) - np.float32(1e-4)


@pytest.mark.parametrize("F", [0, 4])
def test_alpha_cotangent_only_moves_the_geometry_gradients(F):
    """An alpha cotangent adds to the gradients of means, conics, opacities, scales and rotations only; a zero one adds
    nothing; and colour / SH / feature gradients are those of the backward without it."""
    inp = util.make_inputs(P=3000, W=70, H=45, F=F, seed=11, bg=(0.3, 0.6, 0.9))
    H, W, ct = inp["H"], inp["W"], inp["ct"]
    h = np.random.default_rng(3).standard_normal((H, W)).astype(np.float32)
    dfeat = ct["dL_dfeature"] if F else None
    _, g0 = _oracle(inp, ct["dL_dcolor"], dfeat)
    _, gz = _oracle(inp, ct["dL_dcolor"], dfeat, dL_dalpha=np.zeros((H, W), np.float32))
    _, gh = _oracle(inp, ct["dL_dcolor"], dfeat, dL_dalpha=h)
    for k in g0:
        assert np.array_equal(g0[k], gz[k]), k
    for k in ("dL_dcolors", "dL_dsh") + (("dL_dfeature",) if F else ()):
        assert np.array_equal(g0[k], gh[k]), k
    for k in ("dL_dmeans2D", "dL_dopacity", "dL_dmeans3D", "dL_dscales", "dL_drotations"):
        assert util.rel_l2(gh[k], g0[k]) > 1e-3, k


@pytest.mark.parametrize("field,gname", [("opacities", "dL_dopacity"), ("means3D", "dL_dmeans3D"), ("scales", "dL_dscales")])
def test_oracle_alpha_backward_matches_finite_differences(field, gname):
    """Few large, faint splats (the setting of test_oracle_cpu.test_backward_matches_finite_differences): the alpha
    gradient against central differences of sum(alpha * h), alpha = 1 - final_T of the oracle's forward."""
    inp = util.make_inputs(P=12, W=32, H=32, F=0, seed=5, scale0=0.06, sh_degree=2)
    inp["g"]["opacities"][:] = 0.35
    inp["g"]["scales"] = np.clip(inp["g"]["scales"], 0.04, 0.09).astype(np.float32)
    yy, xx = np.mgrid[0:32, 0:32].astype(np.float32) / 32
    h = (0.5 + xx * yy).astype(np.float32)
    zc = np.zeros((3, 32, 32), np.float32)
    _, bw = _oracle(inp, zc, None, dL_dalpha=h)
    g = bw[gname].reshape(inp["g"][field].shape).astype(np.float64)

    def loss(gg):
        fw, _ = _oracle(dict(inp, g=gg), None, None, backward=False)
        return float((fw["alpha"].astype(np.float64) * h).sum())

    rng = np.random.default_rng(0)
    base = inp["g"][field]
    num, ana = [], []
    for _ in range(10):
        idx = tuple(rng.integers(0, s) for s in base.shape)
        eps = 1e-3 if field == "scales" else 2e-3 * max(1.0, abs(float(base[idx])))
        a, b = base.copy(), base.copy()
        a[idx] += eps
        b[idx] -= eps
        num.append((loss(dict(inp["g"], **{field: a})) - loss(dict(inp["g"], **{field: b}))) / (float(a[idx]) - float(b[idx])))
        ana.append(g[idx])
    num, ana = np.array(num), np.array(ana)
    # the alpha >= 1/255 cut is a jump of 1/255 in alpha itself wherever a footprint edge crosses a pixel, which central
    # differences see and the analytic gradient does not: a few percent, also for the opacity
    tol = 0.10 if field in ("means3D", "scales") else 0.05
    assert np.linalg.norm(num - ana) <= tol * max(np.linalg.norm(ana), 1e-3), (field, num, ana)

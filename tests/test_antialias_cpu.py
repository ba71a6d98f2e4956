"""The anti-aliased projection without a GPU: the C ABI declares its switch in the render options and rejects an
out-of-range switch before enqueueing anything, the settings keep the reference's 13 fields with `antialiasing` as a 14th
argument, and the expectations of tests/aa_oracle.py (the unmodified C oracle plus a float64 compensation) are right: mode
on changes only the opacity the blend sees and keeps the oracle's own chain, the float64 screen covariance is the oracle's,
and the backward matches central differences of the anti-aliased forward, on both sides of the clamp."""
import ctypes as C
import glob
import json
import os
import re

import numpy as np
import pytest
import torch

import util
from manigaussian_b200 import _binding
import aa_oracle as A
from oracle import gs_oracle as O

AA_CALLS = ("mgs_forward_views", "mgs_backward_views", "mgs_forward_clouds", "mgs_backward_clouds")
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "g[0-9]*.npz")))
MGS_ERR_INVALID_ARG = -1


def test_header_declares_the_aa_option():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    code = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    assert re.search(r"typedef struct mgs_render_options \{[^}]*\bint antialiasing;", code)
    assert dict(_binding.RenderOptions._fields_)["antialiasing"] is C.c_int
    hm = re.search(r"#define\s+MGS_ERR_INVALID_ARG\s+\(?(-?\d+)\)?", hdr)
    assert hm and int(hm.group(1)) == MGS_ERR_INVALID_ARG


@pytest.mark.parametrize("value", [-1, 2, 7])
def test_out_of_range_aa_option_is_rejected_before_anything_runs(value):
    """Every other argument is valid-looking or NULL: the switch is checked first, so no stream or pointer is touched."""
    L = _binding.lib()
    views = (_binding.View * 1)()
    offs = (C.c_int * 2)(0, 1)
    clouds = (_binding.Cloud * 1)()
    clouds[0].P = 10
    opts = _binding.RenderOptions(antialiasing=value)
    rcs = [
        L.mgs_forward_views(1, views, opts, 10, 1, 4, 0, None, None, None, None, None, None, 1.0, None, None, 0, 0, None),
        L.mgs_backward_views(1, views, opts, 10, 1, 4, 0, None, None, None, None, None, 1.0, None, None,
                             None, None, None, None, None, None, None, None, 1, 0, 3, 0, None),
        L.mgs_forward_clouds(1, clouds, offs, views, opts, 1, 4, 0, 1.0, 0, 0, None),
        L.mgs_backward_clouds(1, clouds, offs, views, opts, 1, 4, 0, 1.0, 0, 0, None),
    ]
    for name, rc in zip(AA_CALLS, rcs):
        assert rc == MGS_ERR_INVALID_ARG, name
        assert "antialiasing" in _binding.last_error(), name


def test_settings_keep_the_reference_fields_and_default_off():
    from manigaussian_b200 import GaussianRasterizationSettings as S
    base = (8, 8, 0.3, 0.3, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 1, torch.zeros(3), False, False, False)
    st = S(*base)  # ManiGaussian's 13-argument construction
    assert st.antialiasing is False and len(st) == 13 and len(S._fields) == 13
    on = S(*base, True)
    assert on.antialiasing is True and tuple(on)[:13] == tuple(st)[:13] and len(on) == 13
    assert S(*base, antialiasing=True).antialiasing is True
    kw = S(**dict(zip(S._fields, base)))
    assert kw.antialiasing is False
    r = on._replace(image_height=16)
    assert r.antialiasing is True and r.image_height == 16
    assert on._replace(antialiasing=False).antialiasing is False
    assert "antialiasing=True" in repr(on)
    import copy
    assert copy.deepcopy(on).antialiasing is True


# ---------------------------------------------------------------------------------------------------------------- oracle
def _kw(g):
    return dict(scales=g["scales"], rotations=g["rotations"], cov3D_precomp=g["cov3D_precomp"], shs=g["shs"], sh_degree=g["sh_degree"],
                colors_precomp=g["colors_precomp"], feature=g["feature"])


def _golden_inputs(path):
    z = np.load(path)
    kw = json.loads(bytes(z["recipe"]).decode())
    if "bg" in kw:
        kw["bg"] = tuple(kw["bg"])
    return util.make_inputs(**kw)


def _args(inp):
    g, cam = inp["g"], inp["cam"]
    return (g["means3D"], g["opacities"], cam["viewmatrix"], cam["projmatrix"], cam["campos"], inp["W"], inp["H"], cam["tanfovx"],
            cam["tanfovy"], inp["bg"])


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_aa_oracle_changes_only_the_opacity_and_keeps_the_oracle_plumbing(path):
    """tests/aa_oracle.py on the four golden scenes: mode off is gs_oracle itself; mode on moves conic_opacity.w (and what the
    blend computes from it) only, and lowers it; its per-Gaussian backward with no opacity gradient (so no compensation term) is
    gs_oracle.backward's, bit for bit -- the injected conic gradient is the only way the mode enters the oracle's chain."""
    inp = _golden_inputs(path)
    g, cam, ct = inp["g"], inp["cam"], inp["ct"]
    off = O.forward(*_args(inp), **_kw(g))
    again = A.forward(*_args(inp), antialiasing=False, **_kw(g))
    for k in ("out_color", "final_T", "conic_opacity", "radii"):
        assert np.array_equal(off[k], again[k]), k
    on = A.forward(*_args(inp), **_kw(g))
    for k in ("radii", "means2D", "depths", "cov3D", "rgb", "clamped", "tiles_touched", "point_list", "point_list_keys", "ranges"):
        assert np.array_equal(off[k], on[k]), k
    assert np.array_equal(off["conic_opacity"][:, :3], on["conic_opacity"][:, :3])
    vis = off["radii"] > 0
    s = on["conic_opacity"][vis, 3] / off["conic_opacity"][vis, 3]
    assert s.min() > 0 and s.max() <= 1.0 + 1e-6 and s.min() < 0.999  # every splat loses energy, some visibly
    assert not np.array_equal(off["out_color"], on["out_color"])

    bargs = (g["means3D"], cam["viewmatrix"], cam["projmatrix"], cam["campos"], cam["tanfovx"], cam["tanfovy"])
    b_off = O.backward(off, ct["dL_dcolor"], ct["dL_dfeature"], *bargs, inp["bg"], **_kw(g))
    fw = dict(off, aa=on["aa"], opacities=on["opacities"])
    pre = A.preprocess_backward(fw, *bargs, b_off["dL_dmeans2D"], b_off["dL_dconic"], b_off["dL_dcolors"], np.zeros(inp["P"], np.float32),
                                **_kw(g))
    for k in ("dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales", "dL_drotations"):
        assert np.array_equal(pre[k], b_off[k]), k
    b_on = A.backward(on, ct["dL_dcolor"], ct["dL_dfeature"], *bargs, inp["bg"], **_kw(g))
    assert b_on["dL_dopacity"].shape == b_off["dL_dopacity"].shape and np.isfinite(b_on["dL_dmeans3D"]).all()


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_aa_oracle_screen_covariance_is_the_oracles(path):
    """The float64 screen-space covariance the compensation is computed from, dilated and inverted, is the C oracle's conic:
    within 4e-6 (1 + kappa1) of the conic's norm per Gaussian, kappa1 = (a c + b^2) / (a c - b^2) the cancellation of the
    oracle's fp32 determinant."""
    inp = _golden_inputs(path)
    g, cam = inp["g"], inp["cam"]
    fw = A.forward(*_args(inp), stages_only=True, **_kw(g))
    vis = fw["radii"] > 0
    a, b, c, d1 = (fw["aa"][k][vis] for k in ("a", "b", "c", "d1"))
    conic64 = np.stack([c / d1, -b / d1, a / d1], 1)
    got = fw["conic_opacity"][vis, :3].astype(np.float64)
    k1 = (a * c + b * b) / d1
    err = np.linalg.norm(got - conic64, axis=1) / np.linalg.norm(conic64, axis=1)
    assert np.all(err <= 4e-6 * (1 + k1)), float((err / (4e-6 * (1 + k1))).max())
    assert np.all(fw["aa"]["s"][vis] <= 1.0) and np.all(fw["aa"]["s"][vis] >= np.sqrt(2.5e-5))


# ------------------------------------------------------------------------------------------------------------- gradients
def _scene(precomp_cov=False):
    """Small and mid-sized splats (screen sigma of ~0.2-3 px) in front of a 48x40 camera, plus two needles: two scale axes
    of 1e-6 m, so that d0 / d1 sits far below the 2.5e-5 clamp."""
    inp = util.make_inputs(P=24, W=48, H=40, F=0, seed=21, precomp_colors=True, scale0=0.004)
    g = inp["g"]
    rng = np.random.default_rng(4)
    g["scales"] = np.exp(rng.uniform(np.log(4e-3), np.log(6e-2), (24, 3))).astype(np.float32)
    g["scales"][:2, :2] = 1e-6  # a line segment: its screen covariance has rank 1
    g["scales"][:2, 2] = 5e-2
    g["means3D"] = (np.asarray(util.scenes.SCENE_CENTER, np.float32) + rng.uniform(-0.12, 0.12, (24, 3))).astype(np.float32)
    g["opacities"] = rng.uniform(0.2, 0.9, (24, 1)).astype(np.float32)
    if precomp_cov:
        s, q = g["scales"].astype(np.float64), g["rotations"].astype(np.float64)
        r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        Rm = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                       2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                       2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)
        Sig = Rm @ (s[:, :, None] ** 2 * np.transpose(Rm, (0, 2, 1)))
        g["cov3D_precomp"] = np.stack([Sig[:, 0, 0], Sig[:, 0, 1], Sig[:, 0, 2], Sig[:, 1, 1], Sig[:, 1, 2], Sig[:, 2, 2]],
                                      -1).astype(np.float32)
        g["scales"], g["rotations"] = None, None
    return inp


def _weights(P):
    rng = np.random.default_rng(17)
    return rng.normal(0, 1, (P, 3)), rng.normal(0, 1, P)


def _stage_loss(inp, g):
    """L = sum_i wq_i . (conic xx, xy, yy)_i + wo_i o_eff_i over the oracle's AA projection: the per-Gaussian stage alone,
    smooth in every parameter (no alpha cut, no early termination), so central differences apply."""
    cam = inp["cam"]
    fw = A.forward(g["means3D"], g["opacities"], cam["viewmatrix"], cam["projmatrix"], cam["campos"], inp["W"], inp["H"], cam["tanfovx"],
                   cam["tanfovy"], inp["bg"], **_kw(g), stages_only=True)
    wq, wo = _weights(inp["P"])
    co = fw["conic_opacity"].astype(np.float64)
    return float((co[:, :3] * wq).sum() + (co[:, 3] * wo).sum()), fw


def _stage_grads(inp, antialiasing=True):
    """The AA oracle's per-Gaussian backward of _stage_loss: the blend-stage gradients are the loss weights (dL/dconic.y halved,
    the reference's convention), dL/do_eff = wo.  antialiasing=False: no opacity gradient, so no compensation term -- the
    oracle's own preprocess backward of the conic weights."""
    g, cam = inp["g"], inp["cam"]
    _, fw = _stage_loss(inp, g)
    P = inp["P"]
    wq, wo = _weights(P)
    vis = fw["radii"] > 0
    dconic = np.zeros((P, 4), np.float32)
    dconic[:, 0], dconic[:, 1], dconic[:, 3] = wq[:, 0], 0.5 * wq[:, 1], wq[:, 2]
    dconic[~vis] = 0
    zeros3 = np.zeros((P, 3), np.float32)
    g_eff = np.where(vis, wo, 0.0).astype(np.float32) if antialiasing else np.zeros(P, np.float32)
    out = A.preprocess_backward(fw, g["means3D"], cam["viewmatrix"], cam["projmatrix"], cam["campos"], cam["tanfovx"], cam["tanfovy"],
                                zeros3, dconic, zeros3, g_eff, **dict(_kw(g), shs=None, sh_degree=0))
    return out, fw


@pytest.mark.parametrize("field,gname,precomp", [("opacities", "dL_dopacity", False), ("means3D", "dL_dmeans3D", False),
                                                 ("scales", "dL_dscales", False), ("rotations", "dL_drotations", False),
                                                 ("cov3D_precomp", "dL_dcov3D", True)])
def test_oracle_aa_backward_matches_finite_differences(field, gname, precomp):
    inp = _scene(precomp)
    grads, fw = _stage_grads(inp)
    vis = fw["radii"] > 0
    assert vis.sum() >= 20
    # both sides of the clamp are present: the needles below it, the others above
    _, gfw = _stage_loss(inp, inp["g"])
    off = O.forward(inp["g"]["means3D"], inp["g"]["opacities"], inp["cam"]["viewmatrix"], inp["cam"]["projmatrix"], inp["cam"]["campos"],
                    inp["W"], inp["H"], inp["cam"]["tanfovx"], inp["cam"]["tanfovy"], inp["bg"], **_kw(inp["g"]), stages_only=True)
    s = gfw["conic_opacity"][vis, 3] / off["conic_opacity"][vis, 3]
    assert np.isclose(s.min(), np.sqrt(2.5e-5), rtol=1e-3) and 0.2 < np.median(s) < 0.98
    base = inp["g"][field]
    ana = grads[gname].reshape(base.shape).astype(np.float64)
    num = np.zeros_like(ana)
    for idx in np.ndindex(*base.shape):
        if not vis[idx[0]]:
            continue
        h = 1e-3 * max(abs(float(base[idx])), 1e-3 if field != "cov3D_precomp" else 1e-7)
        if field == "means3D":
            h = 1e-4
        a, b = base.copy(), base.copy()
        a[idx] += h
        b[idx] -= h
        la, _ = _stage_loss(inp, dict(inp["g"], **{field: a}))
        lb, _ = _stage_loss(inp, dict(inp["g"], **{field: b}))
        num[idx] = (la - lb) / (float(a[idx]) - float(b[idx]))
    # fp32 central differences: the loss is evaluated in fp32 (~1e-7 relative per conic entry, amplified by the conic's
    # 1/det^2 and d0's cancellation for thin splats) and divided by a ~1e-3 relative step, so ~1e-3 of the gradient's
    # norm is noise; 1 % leaves room for it and is far below what a wrong term (a factor of 2 on H01, a missing s, the
    # compensation's covariance term left out: 10-60 % here) produces
    # the needles' d0 is ~0: a covariance step moves it across the clamp's kink, where central differences do not apply
    rows = vis.copy()
    if field == "cov3D_precomp":
        rows[:2] = False
    err = np.linalg.norm((num - ana)[rows])
    assert err <= 0.01 * np.linalg.norm(ana[rows]), (field, err / np.linalg.norm(ana[rows]))
    # the needles (clamped) get dL/do = sqrt(2.5e-5) wo and no covariance term from the compensation: their geometry
    # gradients are those of the backward without the mode, bit for bit
    if field == "opacities":
        wo = _weights(inp["P"])[1]
        assert np.allclose(ana[:2, 0], np.sqrt(2.5e-5) * wo[:2], rtol=1e-5)
    else:
        plain, _ = _stage_grads(inp, antialiasing=False)
        assert np.array_equal(grads[gname][:2], plain[gname][:2])
        assert not np.allclose(grads[gname][2:][vis[2:]], plain[gname][2:][vis[2:]], rtol=1e-2)

"""The L1 + SSIM loss without a GPU: the float64 numpy oracle (tests/ssim_oracle.py) against torch float64 autograd of the
reference's expression (F.conv2d with the 2-D window, padding 5, groups = C), and the C ABI of the SSIM head (declarations,
exports, the ctypes layout of mgs_view_ssim, argument checks that return before any GPU work)."""
import ctypes
import math
import os
import re

import numpy as np
import pytest

import util
from manigaussian_b200 import _binding
import ssim_oracle as O

CALLS = ("mgs_ssim", "mgs_ssim_backward")
FIELDS = ("ssim_terms", "loss_acc", "cot_scale", "cot_color")


def _reference(x, g, g_l1, g_ssim):
    """the reference's l1_loss and _ssim (window 11, sigma 1.5, size_average) in float64 torch, and d(g_l1 l1 + g_ssim ssim)/dx"""
    import torch
    import torch.nn.functional as F
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    gt = torch.tensor(g, dtype=torch.float64)
    C = x.shape[0]
    gauss = torch.tensor([math.exp(-(i - 5) ** 2 / 4.5) for i in range(11)], dtype=torch.float64)
    gauss = gauss / gauss.sum()
    w = (gauss[:, None] @ gauss[None, :]).expand(C, 1, 11, 11).contiguous()
    a, b = xt.unsqueeze(0), gt.unsqueeze(0)
    mu1, mu2 = F.conv2d(a, w, padding=5, groups=C), F.conv2d(b, w, padding=5, groups=C)
    s1 = F.conv2d(a * a, w, padding=5, groups=C) - mu1 ** 2
    s2 = F.conv2d(b * b, w, padding=5, groups=C) - mu2 ** 2
    s12 = F.conv2d(a * b, w, padding=5, groups=C) - mu1 * mu2
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    smap = ((2 * mu1 * mu2 + c1) * (2 * s12 + c2)) / ((mu1 ** 2 + mu2 ** 2 + c1) * (s1 + s2 + c2))
    l1 = (xt - gt).abs().mean()
    ssim = smap.mean()
    (g_l1 * l1 + g_ssim * ssim).backward()
    return float(l1.detach()), float(ssim.detach()), xt.grad.numpy()


def _case(name):
    rng = np.random.default_rng(CASES.index(name))
    shapes = {"1x1": (1, 1), "5x7": (5, 7), "11x11": (11, 11), "37x61": (37, 61), "constant": (13, 17), "equal": (16, 16),
              "outside01": (19, 23), "sign0": (12, 20)}
    H, W = shapes[name]
    x, g = rng.uniform(0, 1, (3, H, W)), rng.uniform(0, 1, (3, H, W))
    if name == "constant":
        x, g = np.full((3, H, W), 0.3), np.full((3, H, W), 0.7)
    elif name == "equal":
        g = x.copy()
    elif name == "outside01":
        x, g = rng.uniform(-0.5, 1.8, (3, H, W)), rng.uniform(-0.2, 1.3, (3, H, W))
    elif name == "sign0":
        x[:, ::2] = g[:, ::2]  # every other row: x == g, where the L1 gradient is sign(0) = 0
    return x, g


CASES = ("1x1", "5x7", "11x11", "37x61", "constant", "equal", "outside01", "sign0")


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_torch_float64_autograd_of_the_reference(name):
    x, g = _case(name)
    g_l1, g_ssim = 0.8, -0.2  # the 3DGS objective: 0.8 l1 + 0.2 (1 - ssim)
    l1, ssim, dx = _reference(x, g, g_l1, g_ssim)
    o_l1, o_ssim = O.losses(x, g)
    assert abs(o_l1 - l1) <= 1e-12 * max(abs(l1), 1e-300)
    assert abs(o_ssim - ssim) <= 1e-12 * abs(ssim)
    got = O.grad(x, g, g_l1, g_ssim)
    scale = np.abs(dx).max()
    if name == "equal":
        assert ssim == pytest.approx(1.0, abs=1e-14)
        assert np.abs(got).max() <= 1e-13 and scale <= 1e-13  # a maximum of SSIM, and sign(0) = 0: no gradient at all
    else:
        assert np.linalg.norm(got - dx) <= 1e-12 * np.linalg.norm(dx)
    if name == "sign0":
        l1_only = O.grad(x, g, 1.0, 0.0)
        assert not l1_only[:, ::2].any() and l1_only[:, 1::2].all()


def test_oracle_terms_and_batches():
    """terms() is [3 x C, H, W] in (partial, channel) order, and a batch is a set of independent images"""
    x, g = _case("5x7")
    t = O.terms(x, g)
    S, d_mu, d_e2, d_exg = O.ssim_map(x, g)
    assert t.shape == (9, 5, 7)
    assert np.array_equal(t[0:3], d_mu) and np.array_equal(t[3:6], d_e2) and np.array_equal(t[6:9], d_exg)
    x2, g2 = np.stack([x, x[::-1]]), np.stack([g, g[::-1]])
    assert np.array_equal(O.ssim_map(x2, g2)[0][1], O.ssim_map(x[::-1], g[::-1])[0])


def test_header_declares_the_ssim_struct_option_and_calls():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    code = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    m = re.search(r"typedef struct mgs_view_ssim \{(.*?)\} mgs_view_ssim;", code, flags=re.S)
    assert m
    assert tuple(re.findall(r"\*\s*(\w+);", m.group(1))) == FIELDS
    L = _binding.lib()
    for name in CALLS:
        assert re.search(r"\b%s\s*\(" % name, code), name
        assert name in _binding.EXPORTED_SYMBOLS and hasattr(L, name), name
    assert re.search(r"typedef struct mgs_render_options \{[^}]*const mgs_view_ssim\* ssim;", code)
    names = [L.mgs_profile_stage_name(i).decode() for i in range(L.mgs_profile_num_stages())]
    assert names[-2:] == ["ssim_fwd", "ssim_bwd"] and names[:3] == ["project_fwd", "depth_sort", "scan"]


def test_struct_layout_matches_the_header():
    assert tuple(f for f, _ in _binding.ViewSsim._fields_) == FIELDS
    assert ctypes.sizeof(_binding.ViewSsim) == len(FIELDS) * ctypes.sizeof(ctypes.c_void_p)


def _view(**kw):
    w = _binding.View()
    # enough of a view to pass the per-view checks; no pointer is ever dereferenced on the host
    for k in ("viewmatrix", "projmatrix", "cam_pos", "background", "geometry_state", "binning_state", "image_state", "out_color",
              "radii", "dL_dpix", "blend_scratch", "target_color", "cot_color", "loss_acc"):
        setattr(w, k, 16)
    w.width, w.height, w.binning_capacity = 8, 8, 16
    for k, v in kw.items():
        setattr(w, k, v)
    return w


@pytest.mark.parametrize("case", ["no_target_color", "no_terms", "no_loss_acc", "no_cot_color", "no_out_color"])
def test_ssim_option_checks_its_arguments_without_a_gpu(case):
    L = _binding.lib()
    views = (_binding.View * 1)(_view(**{"no_target_color": dict(target_color=None),
                                         "no_out_color": dict(out_color=None)}.get(case, {})))
    ss = (_binding.ViewSsim * 1)()
    ss[0].ssim_terms, ss[0].loss_acc, ss[0].cot_color = 16, 16, 16
    if case == "no_terms":
        ss[0].ssim_terms = None
    elif case == "no_loss_acc":
        ss[0].loss_acc = None
    elif case == "no_cot_color":
        ss[0].cot_color = None
    offs = (ctypes.c_int * 2)(0, 1)
    clouds = (_binding.Cloud * 1)()
    clouds[0].P, clouds[0].means3D, clouds[0].opacities, clouds[0].shs, clouds[0].scales, clouds[0].rotations = 10, 16, 16, 16, 16, 16
    clouds[0].dL_dmean3D, clouds[0].dL_dopacity, clouds[0].dL_dsh = 16, 16, 16
    ss = _binding.RenderOptions(ssim=ss)
    if case != "no_out_color":  # out_color is required of every forward view anyway
        rc = L.mgs_forward_views(1, views, ss, 10, 1, 4, 0, 16, 16, None, None, 16, 16, 1.0, 16, None, 0, 0, None)
        assert rc == -1  # MGS_ERR_INVALID_ARG
        assert "SSIM" in _binding.last_error()
        rc = L.mgs_forward_clouds(1, clouds, offs, views, ss, 1, 4, 0, 1.0, 0, 0, None)
        assert rc == -1 and "SSIM" in _binding.last_error()
    rc = L.mgs_backward_views(1, views, ss, 10, 1, 4, 0, 16, 16, None, None, 16, 1.0, 16, None,
                              16, 16, None, None, None, 16, 16, 16, 1, 0, 3, 0, None)
    assert rc == -1 and "SSIM" in _binding.last_error()
    rc = L.mgs_backward_clouds(1, clouds, offs, views, ss, 1, 4, 0, 1.0, 0, 0, None)
    assert rc == -1 and "SSIM" in _binding.last_error()


def test_standalone_ssim_calls_check_their_arguments_without_a_gpu():
    L = _binding.lib()
    for dims in ((0, 3, 4, 4), (1, 0, 4, 4), (1, 3, 0, 4), (1, 3, 4, -1), (65536, 1, 4, 4), (1, 65536, 4, 4)):
        assert L.mgs_ssim(*dims, 16, 16, 16, 16, None) == -1, dims
        assert L.mgs_ssim_backward(*dims, 16, 16, 16, None, None, 16, None) == -1, dims
    for k in range(4):
        ptrs = [16] * 4
        ptrs[k] = None
        assert L.mgs_ssim(1, 3, 4, 4, *ptrs, None) == -1, k
    for k in (0, 1, 2, 5):  # x, g, ssim_terms, cot_out are required; scale and cot_in may be NULL
        ptrs = [16] * 6
        ptrs[k] = None
        assert L.mgs_ssim_backward(1, 3, 4, 4, *ptrs, None) == -1, k


def test_render_paths_reject_ssim_without_targets():
    """ssim=True without targets is an error before any device work (the arguments never reach a GPU)"""
    import torch
    from manigaussian_b200.gaussian_renderer import render_clouds, render_views
    from manigaussian_b200 import losses
    e = torch.zeros((1, 3))
    kw = dict(pts_xyz=e, rotations=torch.zeros((1, 4)), scales=e, opacity=torch.zeros((1, 1)), pts_rgb=e)
    with pytest.raises(ValueError, match="ssim"):
        render_views([None], ssim=True, **kw)
    with pytest.raises(ValueError, match="ssim"):
        render_clouds([dict(cameras=[None], **kw)], ssim=True)
    a = torch.rand(3, 8, 8)
    with pytest.raises(ValueError, match="window_size"):
        losses.ssim(a, a, window_size=7)
    with pytest.raises(ValueError, match="size_average"):
        losses.ssim(a, a, size_average=False)
    with pytest.raises(ValueError, match="img2"):
        losses.ssim(a, a.clone().requires_grad_())
    with pytest.raises(ValueError, match="CUDA"):
        losses.ssim(a, a)

"""The depth and mask loss heads without a GPU: the numpy oracle (tests/depth_heads_oracle.py) against torch's own
expressions of INTEGRATION.md §4 under autograd on the CPU, and the C ABI of the heads (declarations, exports, the
ctypes layout of mgs_view_depth_mask, argument checks that return before any GPU work)."""
import ctypes
import os
import re

import numpy as np
import pytest

import util
from manigaussian_b200 import _binding
import depth_heads_oracle as O

FIELDS = ("target_depth", "target_mask", "cot_depth", "cot_alpha_depth", "cot_alpha_mask", "loss_acc", "cot_scale")


def _torch_recipe(D, A, g, m):
    """INTEGRATION.md §4 per view, in torch on the CPU: the losses and dL/dD, dL/dA of loss_depth + loss_mask"""
    import torch
    Dt = torch.tensor(D, requires_grad=True)
    At = torch.tensor(A, requires_grad=True)
    gt, mt = torch.tensor(g), torch.tensor(m)
    valid = (gt > 0) & (At.detach() > 0.5)
    d = Dt / At.clamp_min(1e-4)  # the recipe's form: on valid pixels (A > 0.5) the clamp is the identity
    loss_depth = (d - gt).abs()[valid].mean() if bool(valid.any()) else (Dt * 0).sum()
    loss_mask = torch.nn.functional.binary_cross_entropy(At.clamp(1e-4, 1 - 1e-4), mt)
    (loss_depth + loss_mask).backward()
    return float(loss_depth.detach()), float(loss_mask.detach()), Dt.grad.numpy(), At.grad.numpy(), int(valid.sum())


def _planes(seed, H=23, W=31, empty=False):
    rng = np.random.default_rng(seed)
    A = rng.uniform(0, 1, (H, W)).astype(np.float32)
    # the edges of both heads: A at 0.5 (not valid), at EPS and 1 - EPS (the clamp passes), 0 and 1 - 1e-4 exactly, above
    A.flat[:8] = np.array([0.5, 1e-4, 1 - 1e-4, 0.0, np.nextafter(np.float32(0.5), np.float32(1)), 5e-5, 0.99995, 1.0], np.float32)
    D = (A * rng.uniform(0.5, 3.0, (H, W))).astype(np.float32)
    d = np.where(A > 0, D / np.where(A > 0, A, 1), 0).astype(np.float32)
    # targets at least 1e-3 away from d, so that no sign depends on the last ulp; a third of them 0 (unknown depth)
    g = (d + rng.choice([-1, 1], (H, W)) * rng.uniform(1e-3, 0.5, (H, W))).astype(np.float32)
    g[rng.uniform(size=(H, W)) < 0.3] = 0
    g = np.maximum(g, 0).astype(np.float32)
    if empty:
        g[:] = 0
    m = rng.uniform(0, 1, (H, W)).astype(np.float32)
    m[rng.uniform(size=(H, W)) < 0.5] = np.round(m[rng.uniform(size=(H, W)) < 0.5].mean())
    return D, A, g, m


@pytest.mark.parametrize("seed,empty", [(0, False), (1, False), (2, True)])
def test_oracle_matches_torch_recipe(seed, empty):
    D, A, g, m = _planes(seed, empty=empty)
    ld, lm, gD, gA, n = _torch_recipe(D, A, g, m)
    o_ld, o_n, cd, ca = O.depth_head(D, A, g)
    o_lm, cm = O.mask_head(A, m)
    assert o_n == n
    if empty:
        assert n == 0 and o_ld == 0.0 and not cd.any() and not ca.any()
    assert abs(o_ld - ld) <= 1e-6 * max(1.0, abs(ld))
    assert abs(o_lm - lm) <= 1e-6 * max(1.0, abs(lm))
    dD, dA = O.gradients(D, A, g, m)
    assert np.allclose(dD, gD, rtol=1e-5, atol=1e-9)
    assert np.allclose(dA, gA, rtol=1e-5, atol=1e-9)
    # the clamp's edges pass the gradient, outside them nothing does
    assert cm.flat[1] != 0 and cm.flat[2] != 0 and cm.flat[3] == 0 and cm.flat[5] == 0 and cm.flat[7] == 0
    # A = 0.5 is not valid for the depth head
    assert cd.flat[0] == 0 and ca.flat[0] == 0


def test_header_declares_the_depth_mask_struct_and_option():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    code = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    m = re.search(r"typedef struct mgs_view_depth_mask \{(.*?)\} mgs_view_depth_mask;", code, flags=re.S)
    assert m
    fields = re.findall(r"\*\s*(\w+);", m.group(1))
    assert tuple(fields) == FIELDS
    assert re.search(r"typedef struct mgs_render_options \{[^}]*const mgs_view_depth_mask\* depth_mask;", code)


def test_struct_layout_matches_the_header():
    assert tuple(f for f, _ in _binding.ViewDepthMask._fields_) == FIELDS
    assert ctypes.sizeof(_binding.ViewDepthMask) == len(FIELDS) * ctypes.sizeof(ctypes.c_void_p)


def _view(**kw):
    w = _binding.View()
    # enough of a view to pass the per-view checks; no pointer is ever dereferenced on the host
    for k in ("viewmatrix", "projmatrix", "cam_pos", "background", "geometry_state", "binning_state", "image_state", "out_color",
              "radii", "dL_dpix", "blend_scratch"):
        setattr(w, k, 16)
    w.width, w.height, w.binning_capacity = 8, 8, 16
    for k, v in kw.items():
        setattr(w, k, v)
    return w


@pytest.mark.parametrize("case", ["depth_without_planes", "mask_without_plane", "no_accumulator", "no_colour_head"])
def test_depth_mask_option_checks_its_arguments_without_a_gpu(case):
    L = _binding.lib()
    colour = dict(target_color=16, cot_color=16, loss_acc=16)
    views = (_binding.View * 1)(_view(**({} if case == "no_colour_head" else colour)))
    dm = (_binding.ViewDepthMask * 1)()
    dm[0].loss_acc = 16
    if case == "depth_without_planes":
        dm[0].target_depth, dm[0].cot_depth = 16, 16
    elif case == "mask_without_plane":
        dm[0].target_mask = 16
    elif case == "no_accumulator":
        dm[0].target_depth, dm[0].cot_depth, dm[0].cot_alpha_depth, dm[0].loss_acc = 16, 16, 16, None
    else:
        dm[0].target_mask, dm[0].cot_alpha_mask = 16, 16
    dm = _binding.RenderOptions(depth_mask=dm)
    rc = L.mgs_forward_views(1, views, dm, 10, 1, 4, 0, 16, 16, None, None, 16, 16, 1.0, 16, None, 0, 0, None)
    assert rc == -1  # MGS_ERR_INVALID_ARG
    assert ("colour head" if case == "no_colour_head" else "target" if case != "no_accumulator" else "loss_acc") in _binding.last_error()
    offs = (ctypes.c_int * 2)(0, 1)
    clouds = (_binding.Cloud * 1)()
    clouds[0].P, clouds[0].means3D, clouds[0].opacities, clouds[0].shs, clouds[0].scales, clouds[0].rotations = 10, 16, 16, 16, 16, 16
    rc = L.mgs_forward_clouds(1, clouds, offs, views, dm, 1, 4, 0, 1.0, 0, 0, None)
    assert rc == -1
    if case != "no_colour_head":  # the backward does not need the colour head's targets
        rc = L.mgs_backward_views(1, views, dm, 10, 1, 4, 0, 16, 16, None, None, 16, 1.0, 16, None,
                                  16, 16, None, None, None, 16, 16, 16, 1, 0, 3, 0, None)
        assert rc == -1
        clouds[0].dL_dmean3D, clouds[0].dL_dopacity, clouds[0].dL_dsh = 16, 16, 16
        rc = L.mgs_backward_clouds(1, clouds, offs, views, dm, 1, 4, 0, 1.0, 0, 0, None)
        assert rc == -1

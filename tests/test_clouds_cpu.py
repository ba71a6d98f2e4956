"""CPU-side checks of the multi-cloud entry points: mgs_forward_clouds / mgs_backward_clouds refuse malformed arguments with
MGS_ERR_INVALID_ARG and a message before they enqueue any device work (the pointers below are never dereferenced), and
render_clouds refuses clouds it cannot render in one call before it touches a device."""
import ctypes

import pytest
import torch

import util  # noqa: F401  (sys.path)
from manigaussian_b200 import _binding

MGS_ERR_INVALID_ARG = -1
FAKE = 4096  # a non-NULL device address that no check dereferences


def _views(n):
    arr = (_binding.View * n)()
    for w in arr:
        w.viewmatrix = w.projmatrix = w.cam_pos = w.background = FAKE
        w.geometry_state = w.binning_state = w.image_state = FAKE
        w.out_color = w.radii = w.dL_dpix = w.dL_dpix_F = w.blend_scratch = FAKE
        w.width, w.height, w.binning_capacity = 64, 64, 1000
    return arr


def _clouds(n, P=10):
    arr = (_binding.Cloud * n)()
    for k in arr:
        k.P = P
        for name, _ in _binding.Cloud._fields_[1:]:
            setattr(k, name, FAKE)
        k.colors_precomp = k.cov3D_precomp = None
    return arr


def _offsets(*o):
    return (ctypes.c_int * len(o))(*o)


def _both(B, clouds, offsets, views):
    L = _binding.lib()
    rf = L.mgs_forward_clouds(B, clouds, offsets, views, None, 1, 4, 3, 1.0, 0, 0, None)
    ef = _binding.last_error()
    rb = L.mgs_backward_clouds(B, clouds, offsets, views, None, 1, 4, 3, 1.0, 0, 0, None)
    eb = _binding.last_error()
    return (rf, ef), (rb, eb)


@pytest.mark.parametrize("case", ["B=0", "offsets_not_from_0", "offsets_not_increasing", "P=0", "P<0"])
def test_malformed_clouds_are_refused_by_both_clouds_calls(case):
    B, clouds, offsets, views = 2, _clouds(2), _offsets(0, 1, 3), _views(3)
    if case == "B=0":
        B = 0
    elif case == "offsets_not_from_0":
        offsets = _offsets(1, 2, 3)
    elif case == "offsets_not_increasing":
        offsets = _offsets(0, 2, 2)
    elif case == "P=0":
        clouds[1].P = 0
    else:
        clouds[0].P = -5
    for rc, msg in _both(B, clouds, offsets, views):
        assert rc == MGS_ERR_INVALID_ARG and msg, msg


def test_missing_cloud_pointers_are_refused():
    L = _binding.lib()
    views, offs = _views(3), _offsets(0, 1, 3)
    c = _clouds(2)
    c[1].means3D = None
    for rc, msg in _both(2, c, offs, views):
        assert rc == MGS_ERR_INVALID_ARG and "means3D" in msg
    c = _clouds(2)
    c[0].opacities = None
    assert L.mgs_forward_clouds(2, c, offs, views, None, 1, 4, 3, 1.0, 0, 0, None) == MGS_ERR_INVALID_ARG
    c = _clouds(2)
    c[1].shs = None  # neither SHs nor precomputed colours
    assert L.mgs_forward_clouds(2, c, offs, views, None, 1, 4, 3, 1.0, 0, 0, None) == MGS_ERR_INVALID_ARG
    c = _clouds(2)
    c[0].scales = None  # neither scales+rotations nor a covariance
    assert L.mgs_forward_clouds(2, c, offs, views, None, 1, 4, 3, 1.0, 0, 0, None) == MGS_ERR_INVALID_ARG
    c = _clouds(2)
    c[1].dL_dopacity = None
    assert L.mgs_backward_clouds(2, c, offs, views, None, 1, 4, 3, 1.0, 0, 0, None) == MGS_ERR_INVALID_ARG
    # a view of the second cloud without its state buffers / without its feature cotangents
    for field, direction in (("image_state", "mgs_forward_clouds"), ("image_state", "mgs_backward_clouds"),
                             ("dL_dpix_F", "mgs_backward_clouds")):
        v = _views(3)
        setattr(v[2], field, None)
        assert getattr(L, direction)(2, _clouds(2), offs, v, None, 1, 4, 3, 1.0, 0, 0, None) == MGS_ERR_INVALID_ARG, (field, direction)
        assert "view" in _binding.last_error()


def test_cloud_shs_without_their_gradient_are_refused():
    """dL_dsh carries the view-direction term of dL_dmean3D: without it that term would be dropped silently."""
    c = _clouds(2)
    c[1].dL_dsh = None
    rc = _binding.lib().mgs_backward_clouds(2, c, _offsets(0, 1, 3), _views(3), None, 1, 4, 3, 1.0, 0, 0, None)
    assert rc == MGS_ERR_INVALID_ARG and "dL_dsh" in _binding.last_error()


def _settings(sh_degree=1, W=16, H=16):
    from manigaussian_b200 import GaussianRasterizationSettings
    return GaussianRasterizationSettings(H, W, 0.3, 0.3, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), sh_degree, torch.zeros(3),
                                         False, False, True)


def _cloud(P=8, M=4, F=3, sh_degree=1):
    return dict(cameras=[_settings(sh_degree)], pts_xyz=torch.rand(P, 3), rotations=torch.rand(P, 4), scales=torch.rand(P, 3),
                opacity=torch.rand(P, 1), features_color=torch.rand(P, M, 3),
                features_language=torch.rand(P, F) if F else None)


def test_render_clouds_refuses_clouds_it_cannot_render_together():
    from manigaussian_b200.gaussian_renderer import render_clouds
    with pytest.raises(ValueError, match="SH degree"):
        render_clouds([_cloud(), _cloud(sh_degree=3)])
    with pytest.raises(ValueError, match="SH degree"):
        render_clouds([_cloud(M=4), _cloud(M=16)])
    with pytest.raises(ValueError, match="feature width F"):
        render_clouds([_cloud(F=3), _cloud(F=32)])
    with pytest.raises(ValueError, match="feature width F"):
        render_clouds([_cloud(F=3), _cloud(F=0)])
    with pytest.raises(ValueError, match="colour mode"):
        rgb = _cloud()
        rgb.pop("features_color")
        rgb["pts_rgb"] = torch.rand(8, 3)
        render_clouds([_cloud(), rgb])
    with pytest.raises(ValueError, match="P = 0"):
        render_clouds([_cloud(), _cloud(P=0)])
    with pytest.raises(ValueError, match="targets"):
        render_clouds([dict(_cloud(), targets={"rgb": torch.zeros(1, 3, 16, 16)}), _cloud()])

"""`render()` and its multi-view form `render_views()` -- the immediate caller of the rasterizer (SURVEY.md 8(f) row f1).

`render` keeps the signature, semantics and return dictionary of ManiGaussian's
agents/manigaussian_bc/gaussian_renderer/__init__.py:17-94, so NeuralRenderer.pts2render
(agents/manigaussian_bc/neural_rendering.py:383-402) runs on it unchanged.  Differences are only in what it avoids:
the background colour is uploaded once per (device, colour) instead of every call (:25), tan(fov/2) and the image size
come from host scalars when the camera dictionary was built by `manigaussian_b200.cameras` (no `.item()` syncs, :35-40),
the feature normalisation (:66-68) is the fused sm_90a kernel behind `mgs_activate`, and no dummy [P,3] zero feature
tensor is made when features are absent (:70-71).

`render_views` renders V cameras of ONE Gaussian cloud in a single autograd node: the projection/binning chains of all
views are enqueued on per-view streams by one C call that never synchronises with the host, every view's backward SUMS its
per-Gaussian gradients in registers into one packed buffer (`parallel.PackedGradients`), and -- for the view-parallel
multi-GPU mode -- that buffer is all-reduced with ONE collective before the gradients are handed back to autograd.
The reference has no counterpart (bs == 1 is asserted, neural_rendering.py:386; one view per call).

`render_clouds` renders several clouds -- the current and the deformed next frame of the dynamic-field step, for every
sample of the batch -- in one autograd node and one C call per direction, every view on its own stream.
"""
import math

import torch

from . import gaussian_params as _gp
from .cameras import CameraBatch
from .parallel import PackedGradients
from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, _prep, _prep_clouds, camera_rays_backward_raw,
                         camera_rays_raw, deform_backward_raw, deform_raw, field_query_backward_raw,
                         field_query_raw, fps_raw, knn_raw, lift_views_raw, neighbour_reg_backward_raw, neighbour_reg_raw, visibility_views_raw,
                         visibility_views_backward_raw, rasterize_clouds_backward_raw, rasterize_clouds_raw, rasterize_views_backward_raw, rasterize_views_raw)

_BG_CACHE = {}
MIN_DENOMINATOR = 1e-12  # gaussian_renderer/__init__.py:67; compiled into the kernel (activate.cu FEAT_EPS)


def _background(bg_color, device):
    if torch.is_tensor(bg_color):
        return bg_color.to(device=device, dtype=torch.float32)
    key = (str(device), tuple(float(c) for c in bg_color))
    t = _BG_CACHE.get(key)
    if t is None:
        t = torch.tensor(key[1], dtype=torch.float32, device=device)
        _BG_CACHE[key] = t
    return t


class _NormalizeFeatures(torch.autograd.Function):
    """feature / (||feature|| + 1e-12) along the last dimension, fused forward and backward kernels."""

    @staticmethod
    def forward(ctx, feature):
        dev = feature.device
        f = _prep(feature, dev)
        ctx.save_for_backward(f)
        return _gp.normalize_features_raw(f)

    @staticmethod
    def backward(ctx, g):
        (f,) = ctx.saved_tensors
        return _gp.normalize_features_backward_raw(f, g)


def normalize_features(features_language):
    return _NormalizeFeatures.apply(features_language)


def _camera_scalars(nv, idx):
    host = nv.get("_host")
    if host is not None:
        return host["tanfovx"][idx], host["tanfovy"][idx], int(host["height"]), int(host["width"])
    # reference-built dictionary: the values live on the device and reading them synchronises, as in the reference
    return (math.tan(float(nv["FovX"][idx]) * 0.5), math.tan(float(nv["FovY"][idx]) * 0.5),
            int(nv["height"][idx]), int(nv["width"][idx]))


def _with_planar_depth(s):
    """The settings `s` with planar_depth=True (include/mgs_rasterizer.h, mgs_render_options.planar_depth), its other attributes kept."""
    return GaussianRasterizationSettings(*tuple(s)[:13], antialiasing=getattr(s, "antialiasing", False),
                                         orthographic=getattr(s, "orthographic", False), fisheye=getattr(s, "fisheye", None),
                                         distortion=getattr(s, "distortion", None), planar_depth=True)


def render(data, idx, pts_xyz, rotations, scales, opacity, bg_color, pts_rgb=None, features_color=None,
           features_language=None, return_depth=False, return_alpha=False, antialiasing=False, return_median_depth=False,
           return_normal=False, planar_depth=False, flow_xyz=None, flow_camera=None):
    """Render view `idx` of data['novel_view'].  Same arguments and result as the reference's render(); with
    return_depth=True the dictionary also holds "depth" [H,W] (view-space z, alpha-blended, no background term), with
    return_alpha=True "alpha" [H,W] (accumulated opacity 1 - final_T; depth / alpha is the expected depth), with
    return_median_depth=True "median_depth" [H,W] (the depth of the contributor at which the pixel's opacity crosses one
    half, differentiable) and "median_id" [H,W] int32 (that Gaussian's index, -1 where nothing covers the pixel;
    INTEGRATION.md §7), with return_normal=True "normal" [3,H,W] (each Gaussian's shortest axis in world space, turned to
    face the camera, alpha-blended and not normalised: normal / alpha is the expected normal; differentiable, INTEGRATION.md
    §8).  antialiasing=True renders with the anti-aliased projection (opacity compensation for the 0.3 px^2
    dilation, INTEGRATION.md §5).  flow_xyz [P,3] (next-frame means paired with pts_xyz) adds "flow" [2,H,W], as
    render_views' flow_xyz; flow_camera: the next frame's (viewmatrix, projmatrix), or None for the view's own camera."""
    device = pts_xyz.device
    nv = data["novel_view"]
    bg = _background(bg_color, device)
    # zero tensor whose gradient receives the screen-space mean gradients (reference :28-32)
    screenspace_points = torch.zeros_like(pts_xyz, dtype=torch.float32, requires_grad=True, device=device) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    tanfovx, tanfovy, H, W = _camera_scalars(nv, idx)
    raster_settings = GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=tanfovx, tanfovy=tanfovy, bg=bg, scale_modifier=1.0,
        viewmatrix=nv["world_view_transform"][idx], projmatrix=nv["full_proj_transform"][idx],
        sh_degree=3 if features_color is None else 1, campos=nv["camera_center"][idx], prefiltered=False, debug=False,
        include_feature=(features_language is not None), antialiasing=bool(antialiasing), planar_depth=bool(planar_depth))
    rasterizer = GaussianRasterizer(raster_settings=raster_settings, return_depth=return_depth, return_alpha=return_alpha,
                                    return_median_depth=return_median_depth, return_normal=return_normal)
    shs, colors_precomp = None, None
    if features_color is not None:
        shs = features_color
    else:
        assert pts_rgb is not None
        colors_precomp = pts_rgb
    feat = normalize_features(features_language) if features_language is not None else None
    pose = None
    if flow_xyz is not None:
        for bad, what in ((return_normal, "return_normal"), (planar_depth, "planar_depth")):
            if bad:
                raise ValueError(f"flow_xyz cannot be combined with {what}")
        nxt = None
        if flow_camera is not None:
            nxt = [raster_settings._replace(viewmatrix=flow_camera[0], projmatrix=flow_camera[1])]
        pose = (_flow_inputs([raster_settings], pts_xyz, flow_xyz, nxt, None, bg, 0, False) or [None])[0]
    out = rasterizer(means3D=pts_xyz, means2D=screenspace_points, shs=shs, colors_precomp=colors_precomp,
                     language_feature_precomp=feat, opacities=opacity, scales=scales, rotations=rotations, cov3D_precomp=None,
                     flow_means3D=flow_xyz, flow_pose=pose)
    ret = {"render": out[0], "render_embed": out[1], "viewspace_points": screenspace_points, "radii": out[2]}
    nf = int(flow_xyz is not None)
    if flow_xyz is not None:
        ret["flow"] = out[-1]
    if return_depth:
        ret["depth"] = out[3]
    if return_alpha:
        ret["alpha"] = out[3 + bool(return_depth)]
    if return_median_depth:
        ret["median_depth"], ret["median_id"] = out[-2 - bool(return_normal) - nf], out[-1 - bool(return_normal) - nf]
    if return_normal:
        ret["normal"] = out[-1]
    return ret


def _same_value(a, b):
    """Whether two settings values agree.  A CUDA tensor (a learnable field of view) is not read back: the flow kernels take
    every intrinsic from the view itself, so only host values can disagree in a way that matters, and a device comparison
    would synchronise the host and break CUDA-graph capture."""
    if (torch.is_tensor(a) and a.is_cuda) or (torch.is_tensor(b) and b.is_cuda):
        return True
    return float(a) == float(b)


def _flow_inputs(views, pts_xyz, flow_xyz, flow_cameras, view_ids, bg, sh_degree, include):
    """Checks flow_xyz against the cloud and returns the per-view next-frame poses (None: every view's own camera)."""
    if not torch.is_tensor(flow_xyz) or tuple(flow_xyz.shape) != (pts_xyz.shape[0], 3) or flow_xyz.dtype != torch.float32 \
            or flow_xyz.device != pts_xyz.device:
        raise ValueError(f"flow_xyz: expected [{pts_xyz.shape[0]},3] fp32 on {pts_xyz.device}")
    if flow_cameras is None:
        return None
    if isinstance(flow_cameras, CameraBatch):
        ids = list(range(len(flow_cameras))) if view_ids is None else list(view_ids)
        nxt = [flow_cameras.settings(i, bg, sh_degree, include) for i in ids]
    else:
        nxt = list(flow_cameras if view_ids is None else [flow_cameras[i] for i in view_ids])
    if len(nxt) != len(views):
        raise ValueError(f"flow_cameras: expected {len(views)} views, got {len(nxt)}")
    poses = []
    for s, n in zip(views, nxt):
        for name in ("image_height", "image_width", "tanfovx", "tanfovy"):
            if not _same_value(getattr(s, name), getattr(n, name)):
                raise ValueError(f"flow_cameras: {name} differs from the view's (only the pose may change)")
        if bool(getattr(s, "orthographic", False)) != bool(getattr(n, "orthographic", False)):
            raise ValueError("flow_cameras: the camera model (orthographic) differs from the view's (only the pose may change)")
        for name in ("fisheye", "distortion"):
            a, b = getattr(s, name, None), getattr(n, name, None)
            if (a is None) != (b is None) or (a is not None and not all(_same_value(x, y) for x, y in zip(tuple(a), tuple(b)))):
                raise ValueError(f"flow_cameras: the camera model ({name}) differs from the view's (only the pose may change)")
        if any(torch.is_tensor(t) and t.requires_grad for t in (n.viewmatrix, n.projmatrix)):
            raise ValueError("flow_cameras: next-frame poses are constants of the loss and must not require grad")
        poses.append((n.viewmatrix, n.projmatrix))
    return poses


def _device_tan_fov(views):
    """The views' field of view {tan_fovx, tan_fovy} [V,2] when any view carries it as CUDA tensors (e.g. cameras from
    `cameras.camera_batch` of a learnable intr), stacked with its autograd history; None when every view has host floats."""
    dev = next((t.device for s in views for t in (s.tanfovx, s.tanfovy) if torch.is_tensor(t) and t.is_cuda), None)
    if dev is None:
        return None
    # host floats of other views are written by fill kernels: no host->device copy, so a CUDA graph can capture it
    el = lambda t: t.reshape(()).to(torch.float32) if (torch.is_tensor(t) and t.is_cuda) else torch.full((), float(t), device=dev)  # noqa: E731
    return torch.stack([torch.stack([el(s.tanfovx), el(s.tanfovy)]) for s in views])


def _batch_cameras(cameras, ids):
    """The stacked camera tensors of CameraBatch views `ids`, taken from the batch's own [B,...] tensors (no per-view
    slicing and restacking): (viewmatrix [V,4,4], projmatrix [V,4,4], campos [V,3], tan_fov [V,2] or None)"""
    every = list(ids) == list(range(len(cameras)))
    pick = lambda t: (t if every else t[list(ids)]).to(torch.float32)  # noqa: E731
    tf = pick(cameras.tan_fov) if cameras.tan_fov is not None else None
    return pick(cameras.world_view_transform), pick(cameras.full_proj_transform), pick(cameras.camera_center), tf


def _camera_inputs(views, force=False, batch=None):
    """The views' stacked camera tensors (viewmatrix [V,4,4], projmatrix [V,4,4], campos [V,3], tan_fov [V,2] or None) as
    explicit inputs of a node when any of them requires grad (or `force`): the node then returns their gradients.  Else
    (None, None, None, tan_fov).  tan_fov is the device field of view of _device_tan_fov (None without one).  `batch`: the
    same tensors from _batch_cameras, used as they are."""
    if batch is not None:
        if force or any(t is not None and t.requires_grad for t in batch):
            return batch
        return None, None, None, batch[3]
    fields = [[getattr(s, n) for s in views] for n in ("viewmatrix", "projmatrix", "campos")]
    tf = _device_tan_fov(views)
    if not force and not any(torch.is_tensor(t) and t.requires_grad for f in fields for t in f) and not (tf is not None and tf.requires_grad):
        return None, None, None, tf
    return tuple(torch.stack([torch.as_tensor(t, dtype=torch.float32).reshape(shape) for t in f])
                 for f, shape in zip(fields, ((4, 4), (4, 4), (3,)))) + (tf,)


def _camera_outputs(ctx, cam, first):
    """Gradients for the camera inputs at positions first .. first + 3 of the node (None where not needed; the 4th, tan_fov,
    only with a device field of view)"""
    if cam is None:
        return None, None, None, None
    V = cam[0].shape[0]
    shapes = ((V, 4, 4), (V, 4, 4), (V, 3), (V, 2))
    cam = tuple(cam) + (None,) * (4 - len(cam))
    return tuple(g.view(shape) if (g is not None and ctx.needs_input_grad[first + i]) else None
                 for i, (g, shape) in enumerate(zip(cam, shapes)))


def _depth_mask_heads(t_depth, t_mask, V, H, W, dev, where="targets"):
    """The depth / mask heads' `depth_mask` tuple for the raw calls (targets [V,H,W], their cotangent planes, the [V,3]
    accumulator), or None when neither target is given."""
    if t_depth is None and t_mask is None:
        return None
    t_depth, t_mask = _prep(t_depth, dev), _prep(t_mask, dev)
    for name, t in (("depth", t_depth), ("mask", t_mask)):
        if t is not None and tuple(t.shape) != (V, H, W):
            raise ValueError(f"{where}: the {name} target must be [V,H,W] = [{V},{H},{W}]")
    opts = dict(dtype=torch.float32, device=dev)
    plane = lambda on: torch.empty((V, H, W), **opts) if on else None
    return (t_depth, t_mask, plane(t_depth is not None), plane(t_depth is not None), plane(t_mask is not None),
            torch.empty((V, 3), **opts))


def _depth_mask_losses(dm, N, dev):
    """(loss_depth, loss_mask, depth_pixels) [V] from the accumulator of a `depth_mask` tuple; empty for an absent head"""
    empty = lambda: torch.empty(0, device=dev)
    if dm is None:
        return empty(), empty(), empty()
    acc = dm[5]
    if dm[0] is not None:
        loss_depth, n = acc[:, 0] / acc[:, 1].clamp(min=1.0), acc[:, 1].clone()
    else:
        loss_depth, n = empty(), empty()
    loss_mask = acc[:, 2] / N if dm[1] is not None else empty()
    return loss_depth, loss_mask, n


def _ssim_head(V, H, W, dev):
    """The L1 + SSIM head's `ssim` tuple for the raw calls: the partials of S [V,9,H,W], the [V,4] accumulator and the
    combined colour cotangent [V,3,H,W]"""
    opts = dict(dtype=torch.float32, device=dev)
    return torch.empty((V, 9, H, W), **opts), torch.empty((V, 4), **opts), torch.empty((V, 3, H, W), **opts)


def _ssim_losses(head, N, dev):
    """(loss_l1, ssim) [V] from the accumulator of an `ssim` tuple (N = 3 H W); empty without the head"""
    if head is None:
        return torch.empty(0, device=dev), torch.empty(0, device=dev)
    return head[1][:, 0] / N, head[1][:, 1] / N


def _pair_scale(g0, g1, V, dev):
    """[V,2] upstream gradients of two per-view losses, 0 for one that received none (no host synchronisation)"""
    z = torch.zeros((V,), dtype=torch.float32, device=dev)
    return torch.stack([g0 if g0 is not None else z, g1 if g1 is not None else z], 1).contiguous()


def _depth_mask_scale(dm, g_depth, g_mask, V, dev):
    """[V,2] upstream gradients {g_depth, g_mask} of the depth / mask losses for the backward"""
    z = torch.zeros((V,), dtype=torch.float32, device=dev)
    return torch.stack([g_depth if (dm[0] is not None and g_depth is not None) else z,
                        g_mask if (dm[1] is not None and g_mask is not None) else z], 1).contiguous()


def render_views(cameras, pts_xyz, rotations, scales, opacity, bg_color=(0.0, 0.0, 0.0), pts_rgb=None, features_color=None,
                 features_language=None, view_ids=None, return_depth=False, sync_gradients=None, normalize_feature=True,
                 targets=None, return_alpha=False, antialiasing=False, ssim=False, return_median_depth=False, return_normal=False,
                 planar_depth=False, flow_xyz=None, flow_cameras=None):
    """Render several cameras of one Gaussian cloud in one autograd node.

    cameras: `cameras.CameraBatch` (or a sequence of GaussianRasterizationSettings); view_ids selects a subset (e.g. this
    rank's shard, `parallel.shard_views`).  Gaussian arguments as `render()`.  sync_gradients: None (single GPU), True
    (all-reduce over the default process group) or a process group -- the per-Gaussian gradients of this rank's views are
    then summed over ranks inside the backward with one collective.  normalize_feature=False skips the reference's
    per-render feature normalisation (for callers that already hold unit features, e.g. `activate_gaussians` output).
    targets: {"rgb": [V,3,H,W], "embed": [V,F,H,W] (optional)} fuses ManiGaussian's loss heads into the forward blend's
    epilogue: the result then also holds "loss_rgb" and "loss_embed" ([V] each: l2_loss and cosine_loss of
    agents/manigaussian_bc/loss.py per view; combine them as neural_rendering.py:300-318 does) through which -- and only
    through which -- gradients flow; "render"/"render_embed" are returned detached.  targets may also hold "depth" [V,H,W]
    (ground-truth depth, 0 = unknown) and "mask" [V,H,W] (in [0,1]): the same epilogue then evaluates the expected-depth L1
    head and the alpha mask head of INTEGRATION.md §4 per view and the result adds "loss_depth" [V] (mean |depth / alpha - gt|
    over the pixels with gt > 0 and alpha > 0.5; 0 where there is none), "depth_pixels" [V] (their count, float, not
    differentiable) and "loss_mask" [V] (binary cross-entropy of clamp(alpha, 1e-4, 1 - 1e-4) against the mask, mean over
    the pixels).
    ssim: with targets, also evaluate the photometric objective 3DGS trains with on the colour image (INTEGRATION.md §4,
    fused tiled kernels behind each view's blend): the result adds "loss_l1" [V] (mean |render - rgb|) and "ssim" [V] (SSIM
    with the 11x11 Gaussian window, sigma 1.5, as the reference's `ssim`; SSIM itself, not 1 - SSIM), both differentiable;
    e.g. loss = 0.8 * out["loss_l1"] + 0.2 * (1 - out["ssim"]).
    return_alpha: also return "alpha" [V,H,W], the accumulated opacity 1 - final_T (differentiable; depth / alpha is the
    expected depth).
    antialiasing: render with the anti-aliased projection (opacity compensation for the 0.3 px^2 dilation, INTEGRATION.md
    §5); also on when the given settings carry antialiasing=True.  Combines with every option above.
    Camera gradients: when a view's viewmatrix, projmatrix or campos requires grad (e.g. cameras from
    `cameras.camera_batch` of a learnable w2c), the backward also returns their gradients (INTEGRATION.md §6); this combines
    with every option above.  Learnable intrinsics: views whose tanfovx / tanfovy are CUDA tensors (cameras from
    `cameras.camera_batch` of a learnable intr) are projected with that device value, with no device->host read and read
    afresh at every CUDA-graph replay; when it requires grad, the backward returns its gradient through the Jacobian and the
    frustum clamp, beside the projection-matrix path.
    Orthographic views: cameras from `cameras.build_ortho_cameras`, `cameras.ortho_camera_batch` or `cameras.top_down_camera`
    (or settings with orthographic=True) are rendered with the orthographic projection (INTEGRATION.md §10); one call may mix
    them with pinhole views, and they combine with every option here.  Fisheye views: cameras from
    `cameras.build_fisheye_cameras` or `cameras.fisheye_camera_batch` (or settings with a `fisheye` attribute) are rendered
    with the Kannala-Brandt projection (INTEGRATION.md §11), mixed with pinhole and orthographic views as above.
    Distorted-pinhole views: cameras from `cameras.build_distorted_cameras` or `cameras.distorted_camera_batch` (or settings
    with a `distortion` attribute) are rendered with OpenCV's radial, tangential and rational lens distortion
    (INTEGRATION.md §12), mixed with the other three models as above.
    return_median_depth: also return "median_depth" [V,H,W], the view-space depth of the contributor at which each pixel's
    accumulated opacity crosses one half (differentiable; its gradient reaches only that Gaussian's depth), and "median_id"
    [V,H,W] int32, that Gaussian's index (-1 where nothing covers the pixel; INTEGRATION.md §7).  Not with targets.
    return_normal: also return "normal" [V,3,H,W], each Gaussian's shortest axis in world space, turned to face the view's
    camera, blended with the colour's weights (differentiable: its gradient reaches the rotations, and opacities and means
    through the blend weights; not normalised, normal / alpha is the expected normal; INTEGRATION.md §8).  Not with targets:
    the depth / mask heads have no kernel beside it.
    planar_depth: the depth plane, the depth head (targets["depth"]) and the median depth take each Gaussian's depth along
    the pixel's ray, affine in the pixel offset, instead of its centre depth (include/mgs_rasterizer.h,
    mgs_render_options.planar_depth); also on when the given settings carry planar_depth=True.  Not with return_normal.
    flow_xyz: [P,3] next-frame means paired by index with pts_xyz (e.g. the deformed cloud of the dyna step); the result then
    gains "flow" [V,2,H,W], each Gaussian's screen displacement m' - m in pixels (x right, y down) blended with the colour's
    weights (flow / alpha is the expected flow; include/mgs_rasterizer.h, flow plane), differentiable in the cloud, the
    cameras and flow_xyz.  flow_cameras: a CameraBatch or settings aligned with the views (view_ids applies) whose poses
    project flow_xyz, e.g. a wrist camera that moved; by default each view's own.  Only its view and projection matrices are
    read; the model, intrinsics and image size must be the view's.  Not with targets, return_normal, planar_depth or
    sync_gradients.
    Returns {"render" [V,3,H,W], "render_embed" [V,F,H,W] | None, "depth" [V,H,W] (if asked), "alpha" [V,H,W] (if asked),
    "viewspace_points" [V,P,3] (its .grad holds each view's screen-space mean gradients), "radii" [V,P] int32}."""
    device = pts_xyz.device
    include = features_language is not None
    sh_degree = 3 if features_color is None else 1
    if isinstance(cameras, CameraBatch):
        ids = list(range(len(cameras))) if view_ids is None else list(view_ids)
        bg = _background(bg_color, device)
        views = tuple(cameras.settings(i, bg, sh_degree, include) for i in ids)
        batch = _batch_cameras(cameras, ids) if ids else None
    else:
        views = tuple(cameras if view_ids is None else [cameras[i] for i in view_ids])
        batch = None
    if not views:
        raise ValueError("render_views needs at least one view")
    if planar_depth:
        views = tuple(_with_planar_depth(s) for s in views)
    aa = bool(antialiasing) or any(bool(getattr(s, "antialiasing", False)) for s in views)
    if features_color is None and pts_rgb is None:
        raise ValueError("Please provide excatly one of either SHs or precomputed colors!")
    feat = None
    if include:
        feat = normalize_features(features_language) if normalize_feature else features_language
    V, P = len(views), pts_xyz.shape[0]
    screenspace_points = torch.zeros((V, P, 3), dtype=torch.float32, device=device, requires_grad=True)
    if ssim and targets is None:
        raise ValueError("ssim=True needs targets (the colour target \"rgb\")")
    cams = _camera_inputs(views, batch=batch)
    flow_poses = None
    if flow_xyz is not None:
        for bad, what in ((targets is not None, "targets"), (return_normal, "return_normal"),
                          (any(bool(getattr(s, "planar_depth", False)) for s in views), "planar_depth"),
                          (sync_gradients is not None, "sync_gradients")):
            if bad:
                raise ValueError(f"flow_xyz cannot be combined with {what}")
        flow_poses = _flow_inputs(views, pts_xyz, flow_xyz, flow_cameras, view_ids, _background(bg_color, device), sh_degree,
                                  include)
    H, W = int(views[0].image_height), int(views[0].image_width)
    if any((int(s.image_height), int(s.image_width)) != (H, W) for s in views):
        raise ValueError("render_views needs one image size for all views")
    camera = cams[0] is not None
    flat = [pts_xyz, screenspace_points, features_color, pts_rgb if features_color is None else None, feat, opacity, scales,
            rotations] + (list(cams) if camera else []) + ([flow_xyz] if flow_xyz is not None else [])

    def node(tgt):  # render_clouds' node, one cloud rendered by the views calls
        if P == 0:
            raise RuntimeError("render_views needs at least one Gaussian")
        meta = ((views,), bool(return_depth), tgt, bool(return_alpha), aa, bool(ssim), camera, bool(return_median_depth),
                bool(return_normal), (flow_poses,) if flow_xyz is not None else None, True, sync_gradients)
        return _RasterizeClouds.apply(meta, *flat)
    if targets is not None:
        if return_depth:
            raise ValueError("targets and return_depth cannot be combined")
        if return_alpha:
            raise ValueError("targets and return_alpha cannot be combined")
        if return_median_depth:
            raise ValueError("targets and return_median_depth cannot be combined")
        if return_normal:
            raise ValueError("targets and return_normal cannot be combined")
        loss_rgb, loss_embed, color, feat_img, radii, loss_depth, loss_mask, depth_pixels, loss_l1, ssim_v = node([targets])
        ret = {"render": color, "render_embed": feat_img if include else None, "viewspace_points": screenspace_points,
               "radii": radii, "loss_rgb": loss_rgb, "loss_embed": loss_embed}
        if targets.get("depth") is not None:
            ret["loss_depth"], ret["depth_pixels"] = loss_depth, depth_pixels
        if targets.get("mask") is not None:
            ret["loss_mask"] = loss_mask
        if ssim:
            ret["loss_l1"], ret["ssim"] = loss_l1, ssim_v
        return ret
    flow = None
    if V == 1 and sync_gradients is None and cams[0] is None and cams[3] is None:
        # a single view needs neither side streams nor the packed accumulation buffer: the single-view operator is leaner
        st = GaussianRasterizationSettings(*tuple(views[0])[:13], antialiasing=True,
                                           orthographic=getattr(views[0], "orthographic", False),
                                           fisheye=getattr(views[0], "fisheye", None),
                                           distortion=getattr(views[0], "distortion", None),
                                           planar_depth=getattr(views[0], "planar_depth", False)) if aa else views[0]
        out = GaussianRasterizer(st, return_depth=return_depth, return_alpha=return_alpha, return_median_depth=return_median_depth,
                                 return_normal=return_normal)(
            means3D=pts_xyz, means2D=screenspace_points[0], shs=features_color,
            colors_precomp=pts_rgb if features_color is None else None, language_feature_precomp=feat, opacities=opacity,
            scales=scales, rotations=rotations, cov3D_precomp=None, flow_means3D=flow_xyz,
            flow_pose=flow_poses[0] if flow_poses is not None else None)
        color, feat_img, radii = out[0].unsqueeze(0), out[1].unsqueeze(0), out[2].unsqueeze(0)
        depth = out[3].unsqueeze(0) if return_depth else None
        alpha = out[3 + bool(return_depth)].unsqueeze(0) if return_alpha else None
        nf = int(flow_xyz is not None)
        nn = bool(return_normal) + nf
        med_depth, med_id = (out[-2 - nn].unsqueeze(0), out[-1 - nn].unsqueeze(0)) if return_median_depth else (None, None)
        normal = out[-1 - nf].unsqueeze(0) if return_normal else None
        flow = out[-1].unsqueeze(0) if flow_xyz is not None else None
    else:
        color, feat_img, radii, depth, alpha, med_depth, med_id, normal, flow = node(None)
    ret = {"render": color, "render_embed": feat_img if include else None, "viewspace_points": screenspace_points,
           "radii": radii}
    if return_depth:
        ret["depth"] = depth
    if return_alpha:
        ret["alpha"] = alpha
    if return_median_depth:
        ret["median_depth"], ret["median_id"] = med_depth, med_id
    if return_normal:
        ret["normal"] = normal
    if flow_xyz is not None:
        ret["flow"] = flow
    return ret


def lift_views(cameras, pts_xyz, rotations, scales, opacity, maps, view_ids=None, antialiasing=False):
    """Lift one 2D map per camera onto the Gaussians with the blend's own weights (INTEGRATION.md §9).

    cameras / view_ids as `render_views` (a `cameras.CameraBatch`, including device field-of-view cameras of a learnable
    intr, or a sequence of GaussianRasterizationSettings).  maps: [V,C,H,W], a list of V [C,H,W] (fp32, on the cloud's
    device), or None for the weights only; C may be 0 .. 512.  For every Gaussian g, with w_vpg = alpha T the weight with
    which view v's render blends g into pixel p (no background term):
        lifted[g][c] = sum_v sum_p w_vpg maps[v][c][p]        weight[g] = sum_v sum_p w_vpg
    lifted / weight is the Gaussian's weighted average of the maps (where weight > 0), weight alone a visibility score over
    the views.  The same cloud rendered with these cameras (orthographic, fisheye and distorted ones included) and `antialiasing` gives the weights
    used here.  Inputs that
    require grad are detached; the outputs are not differentiable.  Returns {"lifted": [P,C], "weight": [P]}; raises
    ValueError on a shape, dtype or device mismatch."""
    device = pts_xyz.device
    if isinstance(cameras, CameraBatch):
        ids = list(range(len(cameras))) if view_ids is None else list(view_ids)
        bg = _background((0.0, 0.0, 0.0), device)
        views = tuple(cameras.settings(i, bg, 0, False) for i in ids)
    else:
        views = tuple(cameras if view_ids is None else [cameras[i] for i in view_ids])
    if not views:
        raise ValueError("lift_views needs at least one view")
    aa = bool(antialiasing) or any(bool(getattr(s, "antialiasing", False)) for s in views)
    P = pts_xyz.shape[0] if (torch.is_tensor(pts_xyz) and pts_xyz.dim() == 2) else -1
    inputs = (("pts_xyz", pts_xyz, (3,)), ("rotations", rotations, (4,)), ("scales", scales, (3,)), ("opacity", opacity, None))
    for name, t, tail in inputs:
        if not torch.is_tensor(t):
            raise ValueError(f"{name}: expected a tensor")
        shape_ok = tuple(t.shape) in ((P, 1), (P,)) if tail is None else tuple(t.shape) == (P,) + tail
        if P <= 0 or not shape_ok:
            raise ValueError(f"{name}: expected [{P},{'1' if tail is None else tail[0]}], got {tuple(t.shape)}")
        if t.dtype != torch.float32:
            raise ValueError(f"{name}: expected float32, got {t.dtype}")
    V = len(views)
    if maps is not None:
        if torch.is_tensor(maps):
            if maps.dim() != 4:
                raise ValueError(f"maps: expected [V,C,H,W] or a list of [C,H,W], got {tuple(maps.shape)}")
            maps = list(maps.unbind(0))
        maps = list(maps)
        if len(maps) != V:
            raise ValueError(f"maps: expected {V} maps (one per view), got {len(maps)}")
        C = maps[0].shape[0] if torch.is_tensor(maps[0]) and maps[0].dim() == 3 else -1
        for v, (m, s) in enumerate(zip(maps, views)):
            want = (C, int(s.image_height), int(s.image_width))
            if not torch.is_tensor(m) or tuple(m.shape) != want:
                raise ValueError(f"maps[{v}]: expected {list(want)} [C,H,W], got {tuple(m.shape) if torch.is_tensor(m) else type(m)}")
            if m.dtype != torch.float32:
                raise ValueError(f"maps[{v}]: expected float32, got {m.dtype}")
        if C > 512:
            raise ValueError(f"maps: at most 512 channels, got {C}")
    for name, t in [(n, x) for n, x, _ in inputs] + [(f"maps[{v}]", m) for v, m in enumerate(maps or ())]:
        if t.device != device or not t.is_cuda:
            raise ValueError(f"{name}: expected a CUDA tensor on {device}, got {t.device}")
    if maps is not None:
        maps = [m.detach() for m in maps]
    lifted, weight = lift_views_raw(views, pts_xyz.detach(), opacity.detach(), scales.detach(), rotations.detach(), 1.0, None, maps,
                                    antialiasing=aa)
    return {"lifted": lifted, "weight": weight}


class _PointVisibility(torch.autograd.Function):
    """point_visibility(differentiable=True): uv, depth and transmittance as outputs of one node, differentiable in the points,
    the cloud and the cameras' explicit inputs (_camera_inputs); in_view is not differentiable"""

    @staticmethod
    def forward(ctx, points, pts_xyz, rotations, scales, opacity, views, aa, cam_vm=None, cam_pm=None, cam_cp=None, cam_tf=None):
        uv, depth, in_view, T, state = visibility_views_raw(views, pts_xyz.detach(), opacity.detach(), scales.detach(),
                                                            rotations.detach(), 1.0, None, points.detach(), antialiasing=aa,
                                                            tan_fov=cam_tf, keep_state=True)
        in_view = in_view.bool()
        ctx.state, ctx.opac_shape, ctx.camera = state, opacity.shape, cam_vm is not None
        # T is an output: it reaches the backward through save_for_backward (an output kept on ctx is a reference cycle)
        ctx.save_for_backward(points, pts_xyz, rotations, scales, opacity, T)
        ctx.mark_non_differentiable(in_view)
        return uv, depth, in_view, T

    @staticmethod
    def backward(ctx, g_uv, g_depth, _g_in_view, g_T):
        points, pts_xyz, rotations, scales, opacity, T = ctx.saved_tensors
        need = ctx.needs_input_grad
        want_points, want_cloud, want_cam = need[0], any(need[1:5]), ctx.camera and any(need[7:11])
        if ctx.state is None or not (want_points or want_cloud or want_cam):  # Q = 0: nothing depends on the cloud
            zero = lambda t, n: torch.zeros_like(t) if n else None  # noqa: E731
            cam = None
            if ctx.camera:
                V = T.shape[0]
                cam = tuple(torch.zeros(s, dtype=torch.float32, device=T.device) for s in ((V, 16), (V, 16), (V, 3), (V, 2)))
            return (zero(points, need[0]), zero(pts_xyz, need[1]), zero(rotations, need[2]), zero(scales, need[3]),
                    zero(opacity, need[4]), None, None, *_camera_outputs(ctx, cam, 7))
        dpts, dmeans, dop, dscales, drot, cam = visibility_views_backward_raw(
            ctx.state, points, pts_xyz, opacity, scales, rotations, 1.0, None, T, g_T, g_uv, g_depth, want_points=want_points,
            want_cloud=(need[1], need[4], need[3], need[2]), camera_grads=want_cam)
        return (dpts, dmeans, drot, dscales, dop.view(ctx.opac_shape) if dop is not None else None, None, None,
                *_camera_outputs(ctx, cam if want_cam else None, 7))


def point_visibility(cameras, points, pts_xyz, rotations, scales, opacity, view_ids=None, antialiasing=False, differentiable=False):
    """Project 3D points into every camera with occlusion (INTEGRATION.md §16).

    cameras / view_ids as `lift_views` (a `cameras.CameraBatch`, including device field-of-view cameras, or a sequence of
    GaussianRasterizationSettings of any of the four camera models, mixed).  points: [Q,3] fp32 on the cloud's device.  For
    view v and point x:
        uv[v, q]            the screen position of x in pixels (pixel centres at integers), through the camera model's own map;
        depth[v, q]         its view-space depth t.z (uv and depth are NaN where x fails the model's cull, e.g. behind the camera);
        in_view[v, q]       x passes the cull and lands in [-0.5, W - 0.5) x [-0.5, H - 0.5);
        transmittance[v, q] prod (1 - alpha_i) over the Gaussians of x's 16x16 tile that lie in front of it (depth < d), in the
                            blend's order, with the blend's alpha at the continuous uv, its 1/255 cut and its 1e-4 stop; 1 where
                            x is not in view.
    At a pixel centre behind the scene the transmittance is the render's final_T (1 - alpha) bit for bit.  By default inputs
    that require grad are detached and the outputs are not differentiable.  differentiable=True makes uv, depth and
    transmittance outputs of one autograd node (include/mgs_rasterizer.h, mgs_visibility_views_backward), with the same
    forward values: differentiable in points, pts_xyz, rotations, scales, opacity and, for a `cameras.CameraBatch` with a
    learnable w2c or intr, its tensors.  The transmittance reaches the Gaussians of its product and uv (the tile, the depth cut,
    the 1/255 cut and the stop are constants; dT/dalpha_i = -T / (1 - alpha_i) with the blend's convention at the 0.99 clamp),
    uv and depth reach the point and the camera where the camera model's cull passes; in_view has no gradient.  Only the
    gradients autograd asks for are computed.  Returns {"uv": [V,Q,2], "depth": [V,Q], "in_view": [V,Q] bool,
    "transmittance": [V,Q]}; raises ValueError on a shape, dtype or device mismatch, and on a `differentiable` that is not a
    bool (a tensor or a string would silently pick a path)."""
    if not isinstance(differentiable, bool):
        raise ValueError(f"differentiable: expected True or False, got {type(differentiable).__name__}")
    device = pts_xyz.device
    batch = None
    if isinstance(cameras, CameraBatch):
        ids = list(range(len(cameras))) if view_ids is None else list(view_ids)
        bg = _background((0.0, 0.0, 0.0), device)
        views = tuple(cameras.settings(i, bg, 0, False) for i in ids)
        batch = _batch_cameras(cameras, ids) if (ids and differentiable) else None
    else:
        views = tuple(cameras if view_ids is None else [cameras[i] for i in view_ids])
    if not views:
        raise ValueError("point_visibility needs at least one view")
    aa = bool(antialiasing) or any(bool(getattr(s, "antialiasing", False)) for s in views)
    P = pts_xyz.shape[0] if (torch.is_tensor(pts_xyz) and pts_xyz.dim() == 2) else -1
    inputs = (("pts_xyz", pts_xyz, (3,)), ("rotations", rotations, (4,)), ("scales", scales, (3,)), ("opacity", opacity, None))
    for name, t, tail in inputs:
        if not torch.is_tensor(t):
            raise ValueError(f"{name}: expected a tensor")
        shape_ok = tuple(t.shape) in ((P, 1), (P,)) if tail is None else tuple(t.shape) == (P,) + tail
        if P <= 0 or not shape_ok:
            raise ValueError(f"{name}: expected [{P},{'1' if tail is None else tail[0]}], got {tuple(t.shape)}")
        if t.dtype != torch.float32:
            raise ValueError(f"{name}: expected float32, got {t.dtype}")
    if not torch.is_tensor(points) or points.dim() != 2 or points.shape[1] != 3:
        raise ValueError(f"points: expected [Q,3], got {tuple(points.shape) if torch.is_tensor(points) else type(points)}")
    if points.dtype != torch.float32:
        raise ValueError(f"points: expected float32, got {points.dtype}")
    for name, t in [(n, x) for n, x, _ in inputs] + [("points", points)]:
        if t.device != device or not t.is_cuda:
            raise ValueError(f"{name}: expected a CUDA tensor on {device}, got {t.device}")
    if differentiable:
        uv, depth, in_view, T = _PointVisibility.apply(points, pts_xyz, rotations, scales, opacity, views, aa,
                                                       *_camera_inputs(views, batch=batch))
        return {"uv": uv, "depth": depth, "in_view": in_view, "transmittance": T}
    uv, depth, in_view, T = visibility_views_raw(views, pts_xyz.detach(), opacity.detach(), scales.detach(), rotations.detach(), 1.0,
                                                 None, points.detach(), antialiasing=aa)
    return {"uv": uv, "depth": depth, "in_view": in_view.bool(), "transmittance": T}


class _CameraRays(torch.autograd.Function):
    """camera_rays with a pixel or camera tensor that requires grad: origin and direction as outputs of one node,
    differentiable in the pixels and the cameras' explicit inputs (_camera_inputs); valid is not differentiable"""

    @staticmethod
    def forward(ctx, pixels, views, shape, cam_vm=None, cam_pm=None, cam_cp=None, cam_tf=None):
        origin, direction, valid = camera_rays_raw(views, pixels.detach() if pixels is not None else None,
                                                   tan_fov=cam_tf.detach() if cam_tf is not None else None)
        valid = valid.bool().view(shape)
        ctx.views, ctx.camera = views, cam_vm is not None
        ctx.save_for_backward(pixels, cam_tf)
        ctx.mark_non_differentiable(valid)
        return origin.view(shape + (3,)), direction.view(shape + (3,)), valid

    @staticmethod
    def backward(ctx, g_origin, g_direction, _g_valid):
        pixels, tf = ctx.saved_tensors
        need = ctx.needs_input_grad
        want_cam = ctx.camera and any(need[3:7])
        V = len(ctx.views)
        flat = lambda g: g.reshape(V, -1, 3) if g is not None else None  # noqa: E731
        dpix, cam = camera_rays_backward_raw(ctx.views, pixels.detach() if pixels is not None else None, flat(g_origin),
                                             flat(g_direction), tan_fov=tf.detach() if tf is not None else None,
                                             want_pixels=need[0], camera_grads=want_cam)
        return (dpix if need[0] else None, None, None, *_camera_outputs(ctx, cam if want_cam else None, 3))


def camera_rays(cameras, pixels=None, view_ids=None):
    """The ray of each pixel through every camera's own lens model (INTEGRATION.md §19): the inverse of the map the renderer
    projects with, for all four camera models (include/mgs_rasterizer.h, mgs_camera_rays).

    cameras / view_ids as `point_visibility` (a `cameras.CameraBatch`, including a learnable w2c or intr, or a sequence of
    GaussianRasterizationSettings of any of the four camera models, mixed).  pixels: None for every pixel centre of the
    views' shared H x W image, or [V,Q,2] fp32 pixel positions (u, v) on the cameras' device, pixel centres at integers.  For
    view v and a pixel, the world points p(z) = origin + z * direction are those whose screen position is the pixel, z their
    view-space depth: direction's view-space z component is 1 (it is not unit length), so `origin + depth[..., None] *
    direction` unprojects a z-depth image, or the renderer's own depth / alpha.  valid is False where the pixel is not the image
    of points the projection keeps (past a fisheye's theta_max, a distorted lens's r_max or fold, or a non-finite pixel); origin
    and direction are NaN there.  Returns {"origin", "direction": [V,H,W,3] or [V,Q,3], "valid": [V,H,W] or [V,Q] bool}.
    One autograd node exactly when pixels or a camera tensor requires grad: origin and direction are then differentiable in
    the pixels, the view and projection matrices and the field of view (fisheye and distorted views), by implicit
    differentiation of the lens maps; the principal point and distortion coefficients are constants.  Raises ValueError on a
    shape, dtype or device mismatch, and on the grid with views of different sizes."""
    batch = None
    if isinstance(cameras, CameraBatch):
        ids = list(range(len(cameras))) if view_ids is None else list(view_ids)
        dev = cameras.world_view_transform.device
        bg = _background((0.0, 0.0, 0.0), dev)
        views = tuple(cameras.settings(i, bg, 0, False) for i in ids)
        batch = _batch_cameras(cameras, ids) if ids else None
    else:
        views = tuple(cameras if view_ids is None else [cameras[i] for i in view_ids])
    if not views:
        raise ValueError("camera_rays needs at least one view")
    device = torch.as_tensor(views[0].viewmatrix).device
    for v, s in enumerate(views):
        if not (torch.is_tensor(s.viewmatrix) and s.viewmatrix.is_cuda and s.viewmatrix.device == device):
            raise ValueError(f"cameras[{v}]: expected a CUDA viewmatrix on {device}")
    V = len(views)
    if pixels is None:
        sizes = {(int(s.image_height), int(s.image_width)) for s in views}
        if len(sizes) != 1:
            raise ValueError(f"pixels=None (every pixel centre) needs views of one size, got {sorted(sizes)}")
        shape = (V,) + sizes.pop()
    else:
        if not torch.is_tensor(pixels) or pixels.dim() != 3 or tuple(pixels.shape[::2]) != (V, 2):
            raise ValueError(f"pixels: expected [{V},Q,2], got {tuple(pixels.shape) if torch.is_tensor(pixels) else type(pixels)}")
        if pixels.dtype != torch.float32:
            raise ValueError(f"pixels: expected float32, got {pixels.dtype}")
        if pixels.device != device:
            raise ValueError(f"pixels: expected a CUDA tensor on {device}, got {pixels.device}")
        shape = (V, int(pixels.shape[1]))
    cam = _camera_inputs(views, batch=batch)
    if (pixels is not None and pixels.requires_grad) or cam[0] is not None:
        origin, direction, valid = _CameraRays.apply(pixels, views, shape, *cam)
        return {"origin": origin, "direction": direction, "valid": valid}
    tf = cam[3].detach() if cam[3] is not None else None
    origin, direction, valid = camera_rays_raw(views, pixels, tan_fov=tf)
    return {"origin": origin.view(shape + (3,)), "direction": direction.view(shape + (3,)), "valid": valid.bool().view(shape)}


def knn(points, k, queries=None):
    """The k nearest neighbours of each query among `points` (INTEGRATION.md §17), by the fp32 squared distance
    d2 = (qx - px)^2 + (qy - py)^2 + (qz - pz)^2; the exact k-nearest set, with no approximate mode.
    points [N,3] float32 on a CUDA device; queries [Q,3] float32 on the same device, or None for the points themselves (each
    point's own index is then never returned; a duplicate of it at distance 0 is).  k is 1 .. 32.
    Returns {"index": [Q,k] int64, "dist2": [Q,k] float32} on the points' device, each row ascending by (d2, index), so ties
    go to the lower index.  A point with a non-finite coordinate is never a neighbour and a non-finite query gets only
    padding; where fewer than k neighbours exist the remaining slots hold index -1 and d2 = +inf.
    Neither output is differentiable (inputs that require grad are detached).  A loss that needs the gradient of a
    distance recomputes it from the index with autograd, e.g. ((points[index] - points[:, None]) ** 2).sum(-1).
    Nothing is read back to the host, so a call can be captured in a CUDA graph.  Raises ValueError for a non-float32 or
    non-[.,3] input, inputs on different devices and k outside 1 .. 32."""
    for name, t in (("points", points), ("queries", queries)):
        if t is None and name == "queries":
            continue
        if not torch.is_tensor(t) or t.dim() != 2 or t.shape[1] != 3:
            raise ValueError(f"knn: {name}: expected [.,3], got {tuple(t.shape) if torch.is_tensor(t) else type(t)}")
        if t.dtype != torch.float32:
            raise ValueError(f"knn: {name}: expected float32, got {t.dtype}")
    if queries is not None and queries.device != points.device:
        raise ValueError(f"knn: queries: expected a tensor on {points.device}, got {queries.device}")
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= 32:
        raise ValueError(f"knn: k must be an int in 1 .. 32, got {k!r}")
    index, dist2 = knn_raw(points.detach(), k, None if queries is None else queries.detach())
    return {"index": index, "dist2": dist2}


def farthest_point_sample(points, n, lengths=None, start=None):
    """Farthest-point sampling (INTEGRATION.md §21): n picks from a cloud, each the unpicked finite point farthest from the
    picks before it by the fp32 squared distance D = ((dx*dx) + (dy*dy)) + (dz*dz), every operation rounded to float32
    (no FMA), ties to the lower index.  Pick 0 is `start` when it names a finite point of the cloud, else the lowest-index
    finite point.  Only points with three finite coordinates are picked.
    points [P,3] or [B,P,3] float32 on a CUDA device; lengths int64 [B] on the same device (cloud b is points[b, :lengths[b]],
    clamped to 0 .. P), or None; start int64 [B] on the same device ([] or [1] for a [P,3] cloud), or None.  n >= 0.
    Returns {"index": int64, "dist2": float32}, each [n] or [B,n]: the picks as indices into their cloud, and each pick's
    squared distance to the nearest earlier pick (+inf for pick 0).  Where fewer than n finite points exist the rest of the
    row holds index -1 and d2 = +inf.  The outputs are bitwise identical from call to call.
    Neither output is differentiable (inputs that require grad are detached): gather points[index] for gradients.
    Nothing is read back to the host, so a call can be captured in a CUDA graph.  Raises ValueError for a non-float32 or
    non-[.,3] / [.,.,3] points, a non-int64 or misshapen lengths or start, tensors on different devices and an n that is not
    an int >= 0."""
    if not torch.is_tensor(points) or points.dim() not in (2, 3) or points.shape[-1] != 3:
        got = tuple(points.shape) if torch.is_tensor(points) else type(points)
        raise ValueError(f"farthest_point_sample: points: expected [P,3] or [B,P,3], got {got}")
    if points.dtype != torch.float32:
        raise ValueError(f"farthest_point_sample: points: expected float32, got {points.dtype}")
    batched = points.dim() == 3
    B = points.shape[0] if batched else 1
    for name, t in (("lengths", lengths), ("start", start)):
        if t is None:
            continue
        if not torch.is_tensor(t) or t.dtype != torch.int64:
            raise ValueError(f"farthest_point_sample: {name}: expected int64, got {t.dtype if torch.is_tensor(t) else type(t)}")
        if tuple(t.shape) not in (((B,),) if batched else ((), (1,))):
            raise ValueError(f"farthest_point_sample: {name}: expected [{B if batched else '] or [1'}], got {tuple(t.shape)}")
        if t.device != points.device:
            raise ValueError(f"farthest_point_sample: {name}: expected a tensor on {points.device}, got {t.device}")
    if isinstance(n, bool) or not isinstance(n, int) or n < 0:
        raise ValueError(f"farthest_point_sample: n must be an int >= 0, got {n!r}")
    p = points.detach() if batched else points.detach()[None]
    lengths, start = (None if t is None else t.reshape(B) for t in (lengths, start))
    index, dist2 = fps_raw(p, n, lengths, start)
    if not batched:
        index, dist2 = index[0], dist2[0]
    return {"index": index, "dist2": dist2}


class _NeighbourReg(torch.autograd.Function):
    """the three neighbour regularisers: one node, differentiable in xyz, rot, xyz_next and rot_next"""

    @staticmethod
    def forward(ctx, xyz, rot, xyz_next, rot_next, index, weight):
        loss, state = neighbour_reg_raw(xyz.detach(), rot.detach(), xyz_next.detach(), rot_next.detach(), index, weight)
        ctx.save_for_backward(xyz, rot, xyz_next, rot_next, index, weight, state)
        return tuple(loss.unbind(0))

    @staticmethod
    def backward(ctx, g_rigid, g_rotation, g_isometry):
        xyz, rot, xyz_next, rot_next, index, weight, state = ctx.saved_tensors
        needs = tuple(ctx.needs_input_grad[:4])
        if not any(needs):
            return (None,) * 6
        zero = torch.zeros((), dtype=torch.float32, device=xyz.device)
        grad = torch.stack([zero if g is None else g.float() for g in (g_rigid, g_rotation, g_isometry)])
        g = neighbour_reg_backward_raw(state, xyz.detach(), rot.detach(), xyz_next.detach(), rot_next.detach(), index, weight,
                                       grad, needs=needs)
        return g + (None, None)


def neighbour_regularisers(xyz, rot, xyz_next, rot_next, index, weight):
    """The neighbour regularisers of Dynamic 3D Gaussians (Luiten et al.; INTEGRATION.md §18) between a cloud and its
    deformed next frame, fused (definition in include/mgs_rasterizer.h, mgs_neighbour_reg).
    xyz, xyz_next [P,3] and rot, rot_next [P,4] (quaternions (r, x, y, z), real part first, normalised inside) float32 on one
    CUDA device; index [P,k] int64 with k = 1 .. 32, as knn returns it (slots outside 0 .. P-1, such as knn's -1 padding,
    are skipped); weight [P,k] float32, a constant, e.g. torch.exp(-lam * dist2) from the same knn call.  With
    rel_i = normalize(rot_next_i) * conj(normalize(rot_i)), R_i its rotation matrix, o = xyz_j - xyz_i and
    o' = xyz_next_j - xyz_next_i, the three terms are 1/(P k) times the sums over the valid slots of
        rigid: w |o' - R_i o|,   rotation: w |rel_j - rel_i|,   isometry: w | |o'| - |o| |.
    Returns {"rigid", "rotation", "isometry"}, three 0-dim tensors of one autograd node, differentiable in xyz, rot, xyz_next
    and rot_next (only the gradients autograd asks for are computed).  Nothing is read back to the host.  Raises ValueError
    for a shape, dtype or device mismatch, index not int64 [P,k], k outside 1 .. 32 and a weight that requires grad."""
    where = "neighbour_regularisers"
    tensors = (("xyz", xyz, 3), ("rot", rot, 4), ("xyz_next", xyz_next, 3), ("rot_next", rot_next, 4),
               ("index", index, None), ("weight", weight, None))
    for name, t, _ in tensors:
        if not torch.is_tensor(t):
            raise ValueError(f"{where}: {name}: expected a tensor, got {type(t)}")
    P = xyz.shape[0] if xyz.dim() == 2 else -1
    k = index.shape[1] if index.dim() == 2 else -1
    for name, t, c in tensors:
        want = (P, c if c is not None else k)
        if tuple(t.shape) != want or P < 0:
            raise ValueError(f"{where}: {name}: expected [{P},{c if c is not None else 'k'}], got {tuple(t.shape)}")
        if t.dtype != (torch.int64 if name == "index" else torch.float32):
            raise ValueError(f"{where}: {name}: expected {'int64' if name == 'index' else 'float32'}, got {t.dtype}")
        if t.device != xyz.device:
            raise ValueError(f"{where}: {name}: expected a tensor on {xyz.device}, got {t.device}")
    if not 1 <= k <= 32:
        raise ValueError(f"{where}: k must be in 1 .. 32, got {k}")
    if weight.requires_grad:
        raise ValueError(f"{where}: weight requires grad, but no gradient flows to it: pass weight.detach()")
    rigid, rotation, isometry = _NeighbourReg.apply(xyz, rot, xyz_next, rot_next, index, weight)
    return {"rigid": rigid, "rotation": rotation, "isometry": isometry}


class _Deform(torch.autograd.Function):
    """a cloud deformed by a control graph: one node, differentiable in xyz, rot, node_xyz, node_rot, node_t and weight"""

    @staticmethod
    def forward(ctx, xyz, rot, node_xyz, node_rot, node_t, index, weight):
        out_xyz, out_rot, state = deform_raw(xyz.detach(), rot.detach(), node_xyz.detach(), node_rot.detach(), node_t.detach(),
                                             index, weight.detach())
        ctx.save_for_backward(xyz, rot, node_xyz, node_rot, node_t, index, weight, state)
        return out_xyz, out_rot

    @staticmethod
    def backward(ctx, g_xyz, g_rot):
        xyz, rot, node_xyz, node_rot, node_t, index, weight, state = ctx.saved_tensors
        n = ctx.needs_input_grad
        needs = (n[0], n[1], n[2], n[3], n[4], n[6])
        if not any(needs):
            return (None,) * 7
        g = deform_backward_raw(state, xyz.detach(), rot.detach(), node_xyz.detach(), node_rot.detach(), node_t.detach(), index,
                                weight.detach(), g_xyz, g_rot, needs=needs)
        return g[:5] + (None, g[5])


def deform_gaussians(xyz, rot, node_xyz, node_rot, node_t, index, weight):
    """A cloud deformed by a sparse control graph (embedded deformation, SC-GS; INTEGRATION.md §20), fused (definition in
    include/mgs_rasterizer.h, mgs_deform).  xyz [P,3] and rot [P,4] are the cloud, node_xyz [N,3], node_rot [N,4] and
    node_t [N,3] the control nodes (N >= 0), all float32 on one CUDA device, quaternions (r, x, y, z), real part first;
    index [P,k] int64 with k = 1 .. 32, as knn(node_xyz, k, queries=xyz) returns it (slots outside 0 .. N-1, such as knn's
    -1 padding, are skipped); weight [P,k] float32, used exactly as given.  With q^_j = normalize(node_rot_j) (negated where
    its real part is below 0), R_j its rotation matrix and c_j = node_xyz_j + node_t_j - R_j node_xyz_j, each Gaussian moves to
        xyz'_i = xyz_i + sum_s w (R_j xyz_i + c_j - xyz_i),   rot'_i = normalize(e + sum_s w (q^_j - e)) (x) rot_i
    over its valid slots, e = (1, 0, 0, 0).  Weight missing from 1 goes to the identity motion.  Returns {"xyz": [P,3],
    "rot": [P,4]}, both outputs of one autograd node, differentiable in xyz, rot, node_xyz, node_rot, node_t and weight (only
    the gradients autograd asks for are computed).  Nothing is read back to the host.  Raises ValueError for a shape, dtype
    or device mismatch, index not int64 [P,k] and k outside 1 .. 32."""
    where = "deform_gaussians"
    tensors = (("xyz", xyz), ("rot", rot), ("node_xyz", node_xyz), ("node_rot", node_rot), ("node_t", node_t),
               ("index", index), ("weight", weight))
    for name, t in tensors:
        if not torch.is_tensor(t):
            raise ValueError(f"{where}: {name}: expected a tensor, got {type(t)}")
    P = xyz.shape[0] if xyz.dim() == 2 else -1
    N = node_xyz.shape[0] if node_xyz.dim() == 2 else -1
    k = index.shape[1] if index.dim() == 2 else -1
    want = {"xyz": (P, 3), "rot": (P, 4), "node_xyz": (N, 3), "node_rot": (N, 4), "node_t": (N, 3), "index": (P, k),
            "weight": (P, k)}
    for name, t in tensors:
        rows, cols = want[name]
        if tuple(t.shape) != want[name] or rows < 0:
            raise ValueError(f"{where}: {name}: expected [{rows},{'k' if name in ('index', 'weight') else cols}], "
                             f"got {tuple(t.shape)}")
        if t.dtype != (torch.int64 if name == "index" else torch.float32):
            raise ValueError(f"{where}: {name}: expected {'int64' if name == 'index' else 'float32'}, got {t.dtype}")
        if t.device != xyz.device:
            raise ValueError(f"{where}: {name}: expected a tensor on {xyz.device}, got {t.device}")
    if not 1 <= k <= 32:
        raise ValueError(f"{where}: k must be in 1 .. 32, got {k}")
    out_xyz, out_rot = _Deform.apply(xyz, rot, node_xyz, node_rot, node_t, index, weight)
    return {"xyz": out_xyz, "rot": out_rot}


class _QueryField(torch.autograd.Function):
    """density and features of the field at points: one node, differentiable in the points and every Gaussian tensor"""

    @staticmethod
    def forward(ctx, channel_first, points, pts_xyz, rotations, scales, opacity, features):
        density, out, state, pairs, _ = field_query_raw(points.detach(), pts_xyz.detach(), scales.detach(), rotations.detach(),
                                                        opacity.detach(), None if features is None else features.detach(),
                                                        channel_first=channel_first)
        ctx.channel_first = channel_first
        ctx.opacity_shape = opacity.shape
        ctx.has_features = features is not None
        ctx.save_for_backward(points, rotations, scales, features, state, pairs)
        if out is None:
            out = torch.empty(0, dtype=torch.float32, device=points.device)
            ctx.mark_non_differentiable(out)
        return density, out

    @staticmethod
    def backward(ctx, grad_density, grad_features):
        points, rotations, scales, features, state, pairs = ctx.saved_tensors
        need = ctx.needs_input_grad
        needs = (need[1], need[2], need[4], need[3], need[5], ctx.has_features and need[6])
        if not any(needs):
            return (None,) * 7
        g = field_query_backward_raw(state, pairs, points.detach(), scales.detach(), rotations.detach(),
                                     features.detach() if ctx.has_features else None, grad_density,
                                     grad_features if ctx.has_features else None, channel_first=ctx.channel_first, needs=needs)
        dop = g[4].view(ctx.opacity_shape) if g[4] is not None else None
        return None, g[0], g[1], g[3], g[2], dop, g[5]


def _field_inputs(where, pts_xyz, rotations, scales, opacity, features, points=None):
    """ValueError on a shape, dtype or device mismatch of query_field / voxelize's tensors"""
    P = pts_xyz.shape[0] if (torch.is_tensor(pts_xyz) and pts_xyz.dim() == 2) else -1
    inputs = [("pts_xyz", pts_xyz, (3,)), ("rotations", rotations, (4,)), ("scales", scales, (3,)), ("opacity", opacity, None)]
    for name, t, tail in inputs:
        if not torch.is_tensor(t):
            raise ValueError(f"{where}: {name}: expected a tensor")
        shape_ok = tuple(t.shape) in ((P, 1), (P,)) if tail is None else tuple(t.shape) == (P,) + tail
        if P <= 0 or not shape_ok:
            raise ValueError(f"{where}: {name}: expected [{P},{'1' if tail is None else tail[0]}], got {tuple(t.shape)}")
    if features is not None:
        if not torch.is_tensor(features) or features.dim() != 2 or features.shape[0] != P:
            raise ValueError(f"{where}: features: expected [{P},C], got {tuple(features.shape) if torch.is_tensor(features) else type(features)}")
        if features.shape[1] > 512:
            raise ValueError(f"{where}: features: at most 512 channels, got {features.shape[1]}")
        inputs.append(("features", features, None))
    if points is not None:
        if not torch.is_tensor(points) or points.dim() != 2 or points.shape[1] != 3 or points.shape[0] == 0:
            raise ValueError(f"{where}: points: expected [Q,3] with Q > 0, got {tuple(points.shape) if torch.is_tensor(points) else type(points)}")
        inputs.insert(0, ("points", points, None))
    device = pts_xyz.device
    for name, t, _ in inputs:
        if t.dtype != torch.float32:
            raise ValueError(f"{where}: {name}: expected float32, got {t.dtype}")
    for name, t, _ in inputs:
        if t.device != device or not t.is_cuda:
            raise ValueError(f"{where}: {name}: expected a CUDA tensor on {device}, got {t.device}")


def query_field(points, pts_xyz, rotations, scales, opacity, features=None):
    """The Gaussian field at 3D points (INTEGRATION.md §14): for every point x,
        density(x) = sum_i g_i(x),   features(x)[c] = sum_i g_i(x) features[i][c],
        g_i(x) = o_i exp(-|S_i^-1 R(q_i / |q_i|) (x - mu_i)|^2 / 2) where that is >= 1/255, else 0.
    points [Q,3]; pts_xyz [P,3], rotations [P,4] (normalised here), scales [P,3] (activated), opacity [P] or [P,1]
    (activated), features [P,C] (C <= 512, used as given) or None; float32 on one CUDA device.  One autograd node,
    differentiable in every tensor argument (the 1/255 cutoff held fixed); one host synchronisation per call.  Returns
    {"density": [Q], "features": [Q,C] or None}; raises ValueError on a shape, dtype or device mismatch."""
    _field_inputs("query_field", pts_xyz, rotations, scales, opacity, features, points)
    density, out = _QueryField.apply(False, points, pts_xyz, rotations, scales, opacity, features)
    return {"density": density, "features": out if features is not None else None}


def _grid(bounds, resolution, where="voxelize"):
    b = [float(v) for v in bounds]
    if len(b) != 6 or not all(b[k + 3] > b[k] for k in range(3)):
        raise ValueError(f"{where}: bounds must be (x0, y0, z0, x1, y1, z1) with x1 > x0, y1 > y0, z1 > z0, got {bounds}")
    n = [int(resolution)] * 3 if isinstance(resolution, int) else [int(r) for r in resolution]
    if len(n) != 3 or min(n) <= 0:
        raise ValueError(f"{where}: resolution must be a positive int or three of them, got {resolution}")
    return b, n


def voxel_centres(bounds, resolution, device):
    """Centres lo + (i + 1/2) (hi - lo) / n of an [X,Y,Z] grid over bounds (x0, y0, z0, x1, y1, z1), as [X*Y*Z,3] points in
    x-major order (point (i, j, k) at (i Y + j) Z + k)."""
    b, n = _grid(bounds, resolution)
    axes = [torch.tensor(b[k], dtype=torch.float64) + (torch.arange(n[k], dtype=torch.float64) + 0.5) * ((b[k + 3] - b[k]) / n[k])
            for k in range(3)]
    grid = torch.stack(torch.meshgrid(*axes, indexing="ij"), dim=-1).reshape(-1, 3)
    return grid.to(device=device, dtype=torch.float32), n


def voxelize(bounds, resolution, pts_xyz, rotations, scales, opacity, features=None):
    """query_field at the centres of an [X,Y,Z] voxel grid over bounds (x0, y0, z0, x1, y1, z1), e.g. SCENE_BOUNDS, with
    resolution n or (X, Y, Z): voxel (i, j, k) is sampled at lo + (i + 1/2, j + 1/2, k + 1/2) (hi - lo) / n.  The same node,
    differentiable in the Gaussian tensors; the features come out channel first as PerAct's voxel input takes them, written
    in that layout by the kernel.  Returns {"density": [X,Y,Z], "features": [C,X,Y,Z] or None}."""
    _grid(bounds, resolution)
    _field_inputs("voxelize", pts_xyz, rotations, scales, opacity, features)
    points, n = voxel_centres(bounds, resolution, pts_xyz.device)
    density, out = _QueryField.apply(True, points, pts_xyz, rotations, scales, opacity, features)
    return {"density": density.view(*n), "features": out.view(-1, *n) if features is not None else None}


def _views_of(where, cameras, view_ids):
    """the GaussianRasterizationSettings of `cameras` (a CameraBatch or a sequence of settings) picked by view_ids, and
    their device; ValueError without a view or with a viewmatrix that is not a tensor on the first view's device (the caller
    checks that it is a CUDA device after its other checks)"""
    if isinstance(cameras, CameraBatch):
        ids = list(range(len(cameras))) if view_ids is None else list(view_ids)
        bg = _background((0.0, 0.0, 0.0), cameras.world_view_transform.device)
        views = tuple(cameras.settings(i, bg, 0, False) for i in ids)
    else:
        views = tuple(cameras if view_ids is None else [cameras[i] for i in view_ids])
    if not views:
        raise ValueError(f"{where} needs at least one view")
    device = torch.as_tensor(views[0].viewmatrix).device
    for v, s in enumerate(views):
        if not (torch.is_tensor(s.viewmatrix) and s.viewmatrix.device == device):
            raise ValueError(f"{where}: cameras[{v}]: expected a viewmatrix on {device}")
    return views, device


def _check_tensor(where, name, t, shape, device):
    """ValueError unless t is a float32 tensor of `shape` (None entries free) on `device`"""
    if not torch.is_tensor(t) or t.dim() != len(shape) or any(n is not None and int(m) != n for m, n in zip(t.shape, shape)):
        want = "[" + ",".join("." if n is None else str(n) for n in shape) + "]"
        raise ValueError(f"{where}: {name}: expected {want}, got {tuple(t.shape) if torch.is_tensor(t) else type(t)}")
    if t.dtype != torch.float32:
        raise ValueError(f"{where}: {name}: expected float32, got {t.dtype}")
    if t.device != device:
        raise ValueError(f"{where}: {name}: expected a tensor on {device}, got {t.device}")


def tsdf_fuse(cameras, depth, bounds, resolution, trunc, color=None, view_ids=None, volume=None):
    """Fuse depth images into a truncated signed-distance volume (INTEGRATION.md §22), through every camera's own lens model
    (include/mgs_rasterizer.h, mgs_tsdf_fuse): each voxel centre is projected with the renderer's map of a mean and its
    cull, takes the depth d of the pixel it lands on (floor(px + 0.5), floor(py + 0.5)), and with s = d - z (z its view-space
    depth) and views in order: skipped where d is not finite, d <= 0 or s < -trunc, else f = min(1, s / trunc) and
    tsdf <- (tsdf w + f) / (w + 1), colour likewise, w <- w + 1, in float32 with no FMA.
    cameras / view_ids as `camera_rays` (a CameraBatch or a sequence of settings of any of the four camera models, mixed;
    learnable camera tensors are detached).  depth [V,H,W] float32 view-space z (the renderer's depth / alpha, or a sensor's
    z-depth image; 0 where there is no return), every view H x W.  color [V,C,H,W] float32 (1 <= C <= 32) or None.  bounds
    and resolution as `voxelize` (voxel (i, j, k) at voxel_centres' point); trunc > 0 the truncation distance in world units.
    volume: an earlier result, fused into in place (a long stream can be fused in batches of views: one call over V views is
    bitwise equal to successive calls over any split of them in order), or None for a fresh volume (tsdf 1, weight 0,
    colour 0).  Returns {"tsdf": [X,Y,Z], "weight": [X,Y,Z], "color": [C,X,Y,Z] or None}; a voxel no view updates keeps its
    bits, and the result is bitwise repeatable.  Not differentiable (inputs that require grad are detached).  Nothing is read
    back to the host, so a call can be captured in a CUDA graph.  Raises ValueError on a bad shape, dtype, device, size
    mismatch, trunc, channel count, bounds or resolution."""
    where = "tsdf_fuse"
    views, device = _views_of(where, cameras, view_ids)
    V = len(views)
    sizes = {(int(s.image_height), int(s.image_width)) for s in views}
    if len(sizes) != 1:
        raise ValueError(f"{where}: every view must have the same size, got {sorted(sizes)}")
    H, W = sizes.pop()
    b, n = _grid(bounds, resolution, where)
    if isinstance(trunc, bool) or not isinstance(trunc, (int, float)) or not math.isfinite(trunc) or not trunc > 0:
        raise ValueError(f"{where}: trunc must be a finite number > 0, got {trunc!r}")
    _check_tensor(where, "depth", depth, (V, H, W), device)
    C = 0
    if color is not None:
        _check_tensor(where, "color", color, (V, None, H, W), device)
        C = int(color.shape[1])
        if not 1 <= C <= 32:
            raise ValueError(f"{where}: color: expected 1 to 32 channels, got {C}")
    vol = None
    if volume is not None:
        if not isinstance(volume, dict) or not {"tsdf", "weight"} <= set(volume):
            raise ValueError(f"{where}: volume: expected an earlier result (a dict with tsdf, weight and color)")
        _check_tensor(where, "volume['tsdf']", volume["tsdf"], tuple(n), device)
        _check_tensor(where, "volume['weight']", volume["weight"], tuple(n), device)
        vc = volume.get("color")
        if (vc is None) != (color is None):
            raise ValueError(f"{where}: volume: its colour and color must both be given or both be None")
        if vc is not None:
            _check_tensor(where, "volume['color']", vc, (C,) + tuple(n), device)
        for key in ("tsdf", "weight", "color"):
            if volume.get(key) is not None and not volume[key].is_contiguous():
                raise ValueError(f"{where}: volume['{key}']: expected a contiguous tensor (it is updated in place)")
        vol = (volume["tsdf"].detach(), volume["weight"].detach(), vc.detach() if vc is not None else None)
    if device.type != "cuda":
        raise ValueError(f"{where}: cameras: expected a CUDA viewmatrix, got one on {device}")
    from .rasterizer import tsdf_fuse_raw
    tsdf, weight, cvol = tsdf_fuse_raw(views, depth.detach(), b, n, float(trunc), None if color is None else color.detach(),
                                       volume=vol)
    if volume is not None:
        return volume
    return {"tsdf": tsdf, "weight": weight, "color": cvol}


def marching_cubes(values, level, bounds, weight=None, color=None):
    """The level surface of a scalar grid as an indexed triangle mesh (INTEGRATION.md §22; include/mgs_rasterizer.h,
    mgs_marching_cubes_count): values [X,Y,Z] float32 (a TSDF at level 0, or voxelize's density at a density level), grid
    point (i, j, k) at its voxel centre over bounds (as `voxelize`).  weight [X,Y,Z] or None: a grid point is valid where its
    value is finite and its weight is > 0 (unobserved TSDF voxels produce nothing); a cell with an invalid corner emits no
    triangle.  color [C,X,Y,Z] (1 <= C <= 32) or None gives per-vertex attributes.
    Returns {"vertices": [Nv,3] float32, "faces": [Nf,3] int64, "colors": [Nv,C] or None}.  Each crossed edge a triangle uses
    has one vertex, shared by the cells around it, interpolated linearly at the level (t = (level - v_a) / (v_b - v_a), float32,
    no FMA); each face's normal (v1 - v0) x (v2 - v0) points toward increasing value: out of a TSDF surface, into a density
    blob (use faces[:, [0, 2, 1]] for outward faces there).  Ambiguous faces are split the same way from both sides, so a
    level set inside the valid region gives a closed mesh; zero-area triangles are kept; a side below 2 gives an empty mesh.
    The mesh is bitwise repeatable.  One device->host synchronisation per call reads the two totals that size the outputs,
    so the call cannot be captured in a CUDA graph.  Not differentiable.  Raises ValueError on a bad shape, dtype, device,
    channel count or bounds."""
    where = "marching_cubes"
    if not torch.is_tensor(values) or values.dim() != 3:
        raise ValueError(f"{where}: values: expected [X,Y,Z], got {tuple(values.shape) if torch.is_tensor(values) else type(values)}")
    device = values.device
    _check_tensor(where, "values", values, (None, None, None), device)
    n = tuple(int(x) for x in values.shape)
    if isinstance(level, bool) or not isinstance(level, (int, float)) or not math.isfinite(level):
        raise ValueError(f"{where}: level must be a finite number, got {level!r}")
    b, _ = _grid(bounds, 1, where)
    if weight is not None:
        _check_tensor(where, "weight", weight, n, device)
    if color is not None:
        _check_tensor(where, "color", color, (None,) + n, device)
        if not 1 <= color.shape[0] <= 32:
            raise ValueError(f"{where}: color: expected 1 to 32 channels, got {color.shape[0]}")
    from .rasterizer import marching_cubes_raw
    vertices, faces, colors = marching_cubes_raw(values.detach(), float(level), b, None if weight is None else weight.detach(),
                                                 None if color is None else color.detach())
    return {"vertices": vertices, "faces": faces, "colors": colors}


_MCMC_BASE = (("pts_xyz", 3), ("rotations", 4), ("scales", 3), ("opacity", 1))
_MCMC_MAX_ROWS, _MCMC_MAX_MOMENTS = 16, 64  # MGS_MCMC_MAX_ROWS / MGS_MCMC_MAX_MOMENTS (include/mgs_rasterizer.h)


def _mcmc_tensor(where, name, t, P, device, width=None):
    """ValueError unless t is a contiguous float32 [P, ...] tensor on `device`; with a width, [P,width] (or [P] for width 1)"""
    got = tuple(t.shape) if torch.is_tensor(t) else type(t)
    if width is None:
        ok = torch.is_tensor(t) and t.dim() >= 1 and (P is None or t.shape[0] == P)
        want = f"[{'P' if P is None else P}, ...]"
    else:
        shapes = ((P, width),) + (((P,),) if width == 1 else ())
        ok = torch.is_tensor(t) and (tuple(t.shape) in shapes if P is not None else (t.dim() == 2 and t.shape[1] == width))
        want = " or ".join("[" + ",".join(str(x) for x in s) + "]" for s in shapes) if P is not None else f"[P,{width}]"
    if not ok:
        raise ValueError(f"{where}: {name}: expected {want}, got {got}")
    if t.dtype != torch.float32:
        raise ValueError(f"{where}: {name}: expected float32, got {t.dtype}")
    if device is not None and t.device != device:
        raise ValueError(f"{where}: {name}: expected a tensor on {device}, got {t.device}")
    if not t.is_contiguous():
        raise ValueError(f"{where}: {name}: expected a contiguous tensor (it is read and written in place)")


def _mcmc_rng(where, rng, device):
    if not torch.is_tensor(rng) or rng.dtype != torch.int64 or tuple(rng.shape) != (2,) or not rng.is_contiguous():
        got = (rng.dtype, tuple(rng.shape)) if torch.is_tensor(rng) else type(rng)
        raise ValueError(f"{where}: rng: expected a contiguous int64 [2] tensor {{seed, offset}}, got {got}")
    if rng.device != device:
        raise ValueError(f"{where}: rng: expected a tensor on {device}, got {rng.device}")


def _mcmc_logit(min_opacity):
    """t = fp32(logit(min_opacity)): a Gaussian whose opacity logit is <= t is dead"""
    return float(torch.tensor(math.log(min_opacity / (1.0 - min_opacity)), dtype=torch.float32))


def _check_leaves(where, params):
    for name, t in params.items():
        if not t.is_leaf:
            raise ValueError(f"{where}: params[{name!r}] is not a leaf tensor: an optimizer can only hold leaves")


def _swap_params(params, optimizer, new, new_moment):
    """Put the tensors of `new` ({name: tensor}, a new row count) into `params` in place of the tensors of the same names,
    as Parameters where those were and with their requires_grad, and into the optimizer's param groups and state: each
    state tensor shaped like its parameter becomes new_moment(name, key, old tensor), every other entry (Adam's step) is
    kept.  This is what gsplat's _update_param_with_optimizer does."""
    wrapped = {}
    for name, q in new.items():
        p = params[name]
        wrapped[name] = torch.nn.Parameter(q, p.requires_grad) if isinstance(p, torch.nn.Parameter) else q.requires_grad_(p.requires_grad)
    if optimizer is not None:
        names = {id(p): name for name, p in params.items()}
        for group in optimizer.param_groups:
            for k, p in enumerate(group["params"]):
                name = names.get(id(p))
                if name not in wrapped:
                    continue
                q = wrapped[name]
                state = optimizer.state.pop(p, None)
                if state is not None:
                    for key, v in state.items():
                        if torch.is_tensor(v) and v.shape == p.shape:
                            state[key] = new_moment(name, key, v)
                    optimizer.state[q] = state
                group["params"][k] = q
    params.update(wrapped)


def mcmc_relocate(params, optimizer=None, n=None, min_opacity=0.005, *, rng):
    """MCMC relocation and growth (3DGS as Markov chain Monte Carlo, Kheradmand et al. 2024, as gsplat's MCMCStrategy runs it;
    INTEGRATION.md §23; definition in include/mgs_rasterizer.h, mgs_mcmc_relocate), in place on the device.
    params: a dict of float32 contiguous tensors on one CUDA device, in 3DGS's raw parameterisation: "pts_xyz" [P,3],
    "rotations" [P,4] (r, x, y, z), "scales" [P,3] (log scales), "opacity" [P] or [P,1] (logits), plus up to 16 further
    per-Gaussian rows [P, ...] (SH, features).  n: the new count (None: P); n > P appends n - P rows.
    Dead Gaussians (opacity logit <= fp32(logit(min_opacity))) and the appended rows are the destinations.  Each draws a
    live source with probability proportional to floor(2^24 opacity); each source that k destinations picked splits its
    opacity o and scales s over its n = min(k + 1, 51) copies (o' = 1 - (1 - o)^(1/n), s' from gsplat's formula in fp64),
    and every destination becomes a copy of its source's new row.
    optimizer: a torch.optim optimizer over (some of) the params, or None.  Every state tensor shaped like its parameter
    (Adam's exp_avg, exp_avg_sq, max_exp_avg_sq) is zeroed at every source and destination (gsplat zeroes the sources
    only).  On growth, the params dict, the optimizer's param groups and its state get new, longer tensors (as gsplat's
    _update_param_with_optimizer does); without growth every tensor is updated in place.
    rng: int64 [2] = {seed, offset} on the params' device; the offset advances by one on the device per call.
    Returns {"source": [n] int64, each slot's source or -1, "relocated": [1] int64, the destinations filled} on the device.
    With nothing alive no row is written (appended rows are zero with a dead opacity).  The result is bitwise repeatable.
    Nothing is read back to the host: without growth a call can be captured in a CUDA graph.  Not differentiable.
    Raises ValueError on a missing key, a bad shape, dtype, device or contiguity, rows of different lengths, n < P, too
    many rows or moments, min_opacity outside (0, 1), a bad rng, and non-leaf params with an optimizer."""
    where = "mcmc_relocate"
    if not isinstance(params, dict) or any(k not in params for k, _ in _MCMC_BASE):
        raise ValueError(f"{where}: params: expected a dict with keys {', '.join(k for k, _ in _MCMC_BASE)} (and any further rows)")
    x = params["pts_xyz"]
    _mcmc_tensor(where, "params['pts_xyz']", x, None, None, 3)
    P, device = int(x.shape[0]), x.device
    widths = dict(_MCMC_BASE)
    for name, t in params.items():
        _mcmc_tensor(where, f"params[{name!r}]", t, P, device, widths.get(name))
    extra = [k for k in params if k not in widths]
    if len(extra) > _MCMC_MAX_ROWS:
        raise ValueError(f"{where}: params: at most {_MCMC_MAX_ROWS} rows besides the four parameters, got {len(extra)}")
    n = P if n is None else n
    if isinstance(n, bool) or not isinstance(n, int) or n < P:
        raise ValueError(f"{where}: n must be an int >= P = {P}, got {n!r}")
    if isinstance(min_opacity, bool) or not isinstance(min_opacity, (int, float)) or not 0.0 < min_opacity < 1.0:
        raise ValueError(f"{where}: min_opacity must be a number in (0, 1), got {min_opacity!r}")
    _mcmc_rng(where, rng, device)
    if optimizer is not None:
        _check_leaves(where, params)
    if n > P:
        grown = {}
        for name, p in params.items():
            ext = torch.zeros((n - P,) + tuple(p.shape[1:]), dtype=p.dtype, device=device)
            if name == "opacity":
                ext.fill_(_mcmc_logit(min_opacity))
            grown[name] = torch.cat([p.detach(), ext])
        _swap_params(params, optimizer, grown, lambda name, key, v: torch.cat(
            [v, torch.zeros((n - P,) + tuple(v.shape[1:]), dtype=v.dtype, device=v.device)]))
    moments = []
    if optimizer is not None:
        for name, p in params.items():
            for key, v in optimizer.state.get(p, {}).items():
                if torch.is_tensor(v) and v.shape == p.shape:
                    _mcmc_tensor(where, f"optimizer state {key!r} of params[{name!r}]", v, n, device)
                    moments.append(v)
    if len(moments) > _MCMC_MAX_MOMENTS:
        raise ValueError(f"{where}: optimizer: at most {_MCMC_MAX_MOMENTS} moment tensors, got {len(moments)}")
    from .rasterizer import mcmc_relocate_raw
    d = {k: v.detach() for k, v in params.items()}
    source, relocated = mcmc_relocate_raw(P, d["pts_xyz"], d["rotations"], d["scales"], d["opacity"], [d[k] for k in extra],
                                          moments, rng, float(min_opacity))
    return {"source": source, "relocated": relocated}


def mcmc_perturb(pts_xyz, rotations, scales, opacity, scale, rng):
    """MCMC position noise (INTEGRATION.md §23; include/mgs_rasterizer.h, mgs_mcmc_perturb), in place: per Gaussian,
    pts_xyz += Sigma z g(o) scale with Sigma = R(q/|q|) diag(exp(scales)^2) R^T, z ~ N(0, I3) from rng, o = sigmoid(opacity)
    and g(o) = 1 / (1 + exp(-100 ((1 - o) - 0.995))), so only nearly transparent Gaussians move far.  Raw parameters as
    mcmc_relocate takes them: pts_xyz [P,3] (written), rotations [P,4], scales [P,3] (log), opacity [P] or [P,1] (logits).
    scale: lr_means * noise_lr (gsplat: noise_lr = 5e5) as a float32 tensor of one element on the device (a captured
    graph then follows the learning-rate schedule), or a number.  rng: int64 [2] = {seed, offset}, advanced by one on the
    device.  Only pts_xyz is written.  Nothing is read back to the host, so a call can be captured in a CUDA graph.  Not
    differentiable.  Returns pts_xyz.  Raises ValueError on a bad shape, dtype, device, contiguity, scale or rng."""
    where = "mcmc_perturb"
    _mcmc_tensor(where, "pts_xyz", pts_xyz, None, None, 3)
    P, device = int(pts_xyz.shape[0]), pts_xyz.device
    for name, t, w in (("rotations", rotations, 4), ("scales", scales, 3), ("opacity", opacity, 1)):
        _mcmc_tensor(where, name, t, P, device, w)
    if torch.is_tensor(scale):
        if scale.dtype != torch.float32 or scale.numel() != 1 or scale.device != device:
            raise ValueError(f"{where}: scale: expected a float32 tensor of one element on {device}, got "
                             f"{scale.dtype} {tuple(scale.shape)} on {scale.device}")
    elif isinstance(scale, bool) or not isinstance(scale, (int, float)) or not math.isfinite(scale):
        raise ValueError(f"{where}: scale: expected a finite number or a device tensor, got {scale!r}")
    else:
        scale = torch.full((1,), float(scale), dtype=torch.float32, device=device)
    _mcmc_rng(where, rng, device)
    from .rasterizer import mcmc_perturb_raw
    mcmc_perturb_raw(pts_xyz.detach(), rotations.detach(), scales.detach(), opacity.detach(), scale.detach(), rng)
    return pts_xyz


def densify_state(P, device):
    """Zeroed statistics for densify_stats / densify_and_prune: {"grad2d": [P] float32, "count": [P] int32, "radius": [P]
    float32} on `device`."""
    return {"grad2d": torch.zeros(P, dtype=torch.float32, device=device),
            "count": torch.zeros(P, dtype=torch.int32, device=device),
            "radius": torch.zeros(P, dtype=torch.float32, device=device)}


_DENSIFY_STATS = (("grad2d", torch.float32), ("count", torch.int32), ("radius", torch.float32))


def _densify_check_stats(where, stats, P, device):
    if not isinstance(stats, dict) or any(k not in stats for k, _ in _DENSIFY_STATS):
        raise ValueError(f"{where}: stats: expected a dict with keys grad2d, count and radius (densify_state makes one)")
    for k, dt in _DENSIFY_STATS:
        t = stats[k]
        if not torch.is_tensor(t) or tuple(t.shape) != (P,) or t.dtype != dt or t.device != device or not t.is_contiguous():
            got = (t.dtype, tuple(t.shape), str(t.device)) if torch.is_tensor(t) else type(t)
            raise ValueError(f"{where}: stats[{k!r}]: expected a contiguous {dt} [{P}] tensor on {device}, got {got}")


def _densify_sizes(where, sizes, V):
    """each view's max(W, H) as V host ints, from ints, a CameraBatch or a sequence of rasterization settings"""
    if isinstance(sizes, CameraBatch):
        out = [max(int(sizes.width), int(sizes.height))] * len(sizes)
    elif isinstance(sizes, int) and not isinstance(sizes, bool):
        out = [sizes] * V
    else:
        try:
            out = [max(int(s.image_width), int(s.image_height)) if hasattr(s, "image_width") else s for s in sizes]
        except TypeError:
            raise ValueError(f"{where}: sizes: expected ints, a CameraBatch or a sequence of settings, got {type(sizes)}") from None
    if len(out) != V or any(isinstance(s, bool) or not isinstance(s, int) or s <= 0 for s in out):
        raise ValueError(f"{where}: sizes: expected {V} positive ints (each view's max(W, H)), got {out!r}")
    return out


def densify_stats(stats, viewspace_grad, radii, sizes, scale=1.0):
    """Accumulate the statistics of default density control (3DGS's adaptive density control as gsplat's DefaultStrategy
    runs it; INTEGRATION.md §24; definition in include/mgs_rasterizer.h, mgs_densify_stats), in place, once per step.
    stats: densify_state(P, device)'s dict.  viewspace_grad: [V,P,3] (render_views' viewspace_points.grad) or [P,3]
    (render's), float32; radii: [V,P] or [P] int32, the renders' "radii".  sizes: each view's max(W, H): ints (one int for
    every view), a CameraBatch, or a sequence of GaussianRasterizationSettings.  For each Gaussian, over the views in order
    where its radius is > 0: grad2d += |(gx, gy)| scale, count += 1, radius = max(radius, radii / max(W, H)), every
    operation in fp32 without FMA.  scale: a number or a float32 device tensor of one element; a loss averaged over V
    views has per-view gradients 1/V as large, so pass V (gsplat's n_cameras factor).
    One thread per Gaussian and no atomics: bitwise repeatable.  Nothing is read back to the host, so the call can be
    captured in a CUDA graph beside the training step.  Returns stats.  Raises ValueError on a bad stats dict, shape,
    dtype, device, size or scale."""
    where = "densify_stats"
    if not torch.is_tensor(viewspace_grad) or viewspace_grad.dim() not in (2, 3) or viewspace_grad.shape[-1] != 3:
        got = tuple(viewspace_grad.shape) if torch.is_tensor(viewspace_grad) else type(viewspace_grad)
        raise ValueError(f"{where}: viewspace_grad: expected [V,P,3] or [P,3] (viewspace_points.grad), got {got}")
    if viewspace_grad.dtype != torch.float32:
        raise ValueError(f"{where}: viewspace_grad: expected float32, got {viewspace_grad.dtype}")
    g = viewspace_grad.detach()
    g = g if g.dim() == 3 else g[None]
    V, P, device = int(g.shape[0]), int(g.shape[1]), g.device
    if not torch.is_tensor(radii) or tuple(radii.shape) not in ((V, P),) + (((P,),) if viewspace_grad.dim() == 2 else ()):
        got = tuple(radii.shape) if torch.is_tensor(radii) else type(radii)
        raise ValueError(f"{where}: radii: expected [{V},{P}]" + (f" or [{P}]" if viewspace_grad.dim() == 2 else "") + f", got {got}")
    if radii.dtype != torch.int32 or radii.device != device:
        raise ValueError(f"{where}: radii: expected int32 on {device}, got {radii.dtype} on {radii.device}")
    _densify_check_stats(where, stats, P, device)
    sz = _densify_sizes(where, sizes, V)
    if torch.is_tensor(scale):
        if scale.dtype != torch.float32 or scale.numel() != 1 or scale.device != device:
            raise ValueError(f"{where}: scale: expected a float32 tensor of one element on {device}, got "
                             f"{scale.dtype} {tuple(scale.shape)} on {scale.device}")
        scale = scale.detach()
    elif isinstance(scale, bool) or not isinstance(scale, (int, float)) or not math.isfinite(scale):
        raise ValueError(f"{where}: scale: expected a finite number or a device tensor, got {scale!r}")
    from .rasterizer import densify_stats_raw
    densify_stats_raw(g.contiguous(), radii.detach().reshape(V, P).contiguous(), sz, stats["grad2d"], stats["count"],
                      stats["radius"], scale)
    return stats


def _positive(where, name, v):
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not (math.isfinite(v) and v > 0):
        raise ValueError(f"{where}: {name} must be a finite number > 0, got {v!r}")


def densify_and_prune(params, stats, optimizer=None, *, scene_scale, grad_threshold=2e-4, grow_scale3d=0.01, grow_scale2d=None,
                      prune_opacity=0.005, prune_scale3d=0.1, prune_scale2d=None, prune_too_big=False, rng):
    """One refinement of default density control (INTEGRATION.md §24; definition in include/mgs_rasterizer.h,
    mgs_densify_count / mgs_densify_emit): gsplat's DefaultStrategy duplicate, then split, then prune, on the device.
    params: mcmc_relocate's dict ("pts_xyz" [P,3], "rotations" [P,4], "scales" [P,3] log, "opacity" [P] or [P,1] logits,
    plus up to 16 further rows [P, ...]); stats: densify_stats' dict for the same P.
    With L the largest log scale and g = grad2d / max(count, 1): g > grad_threshold clones a Gaussian whose
    exp(L) <= grow_scale3d * scene_scale and splits the others; with grow_scale2d (None: off) a radius above it also splits.
    A split Gaussian is replaced by two children with scales / 1.6 and means drawn from its own Gaussian (Philox from rng).
    Every row (original, clone, child) with opacity below prune_opacity is removed, and with prune_too_big also one with
    exp(L) > prune_scale3d * scene_scale or (with prune_scale2d) a radius above prune_scale2d.  Rows come out as
    [kept originals] ++ [kept clones] ++ [kept first children] ++ [kept second children], each in ascending index.
    optimizer: a torch.optim optimizer over (some of) the params, or None: each state tensor shaped like its parameter
    (Adam's moments) keeps its rows for the kept originals and is zero for new rows; the params dict, the optimizer's param
    groups and state and `stats` get new tensors of the new length, and `stats` is zeroed (gsplat resets it after each
    refinement).  When nothing is cloned, split or pruned no tensor is replaced and only `stats` is zeroed.
    rng: int64 [2] = {seed, offset} on the params' device; the offset advances by one on the device per call.
    Returns {"source": [n_new] int64, each row's parent index (for labels and neighbour lists), "counts": {"n_new",
    "cloned", "split", "pruned"} host ints} with n_new = P + cloned + split - pruned.  The result is bitwise repeatable,
    so the ranks of a view-parallel run that reduce their statistics (INTEGRATION.md §24) make the same refinement.
    One device->host read per call, of the four totals that size the new tensors.  Not differentiable.
    Raises ValueError on a bad params or stats dict, shape, dtype, device or contiguity, a threshold out of range, too many
    rows or moments, a bad rng, and non-leaf params with an optimizer; RuntimeError when n_new would exceed 2^31 - 1."""
    where = "densify_and_prune"
    if not isinstance(params, dict) or any(k not in params for k, _ in _MCMC_BASE):
        raise ValueError(f"{where}: params: expected a dict with keys {', '.join(k for k, _ in _MCMC_BASE)} (and any further rows)")
    x = params["pts_xyz"]
    _mcmc_tensor(where, "params['pts_xyz']", x, None, None, 3)
    P, device = int(x.shape[0]), x.device
    widths = dict(_MCMC_BASE)
    for name, t in params.items():
        _mcmc_tensor(where, f"params[{name!r}]", t, P, device, widths.get(name))
    extra = [k for k in params if k not in widths]
    if len(extra) > _MCMC_MAX_ROWS:
        raise ValueError(f"{where}: params: at most {_MCMC_MAX_ROWS} rows besides the four parameters, got {len(extra)}")
    _densify_check_stats(where, stats, P, device)
    for name, v in (("scene_scale", scene_scale), ("grow_scale3d", grow_scale3d), ("prune_scale3d", prune_scale3d)):
        _positive(where, name, v)
    if isinstance(prune_opacity, bool) or not isinstance(prune_opacity, (int, float)) or not 0.0 < prune_opacity < 1.0:
        raise ValueError(f"{where}: prune_opacity must be a number in (0, 1), got {prune_opacity!r}")
    if isinstance(grad_threshold, bool) or not isinstance(grad_threshold, (int, float)) or math.isnan(grad_threshold):
        raise ValueError(f"{where}: grad_threshold must be a number, got {grad_threshold!r}")
    for name, v in (("grow_scale2d", grow_scale2d), ("prune_scale2d", prune_scale2d)):
        if v is not None and (isinstance(v, bool) or not isinstance(v, (int, float)) or math.isnan(v)):
            raise ValueError(f"{where}: {name} must be a number or None, got {v!r}")
    _mcmc_rng(where, rng, device)
    if optimizer is not None:
        _check_leaves(where, params)
    moments, keys = [], []
    if optimizer is not None:
        for name, p in params.items():
            for key, v in optimizer.state.get(p, {}).items():
                if torch.is_tensor(v) and v.shape == p.shape:
                    _mcmc_tensor(where, f"optimizer state {key!r} of params[{name!r}]", v, P, device)
                    moments.append(v)
                    keys.append((name, key))
    if len(moments) > _MCMC_MAX_MOMENTS:
        raise ValueError(f"{where}: optimizer: at most {_MCMC_MAX_MOMENTS} moment tensors, got {len(moments)}")
    from .rasterizer import densify_and_prune_raw
    d = {k: v.detach() for k, v in params.items()}
    totals, out = densify_and_prune_raw(
        d["pts_xyz"], d["rotations"], d["scales"], d["opacity"], [d[k] for k in extra], moments, stats["grad2d"],
        stats["count"], stats["radius"], rng, float(scene_scale), float(grad_threshold), float(grow_scale3d),
        math.inf if grow_scale2d is None else float(grow_scale2d), float(prune_opacity), float(prune_scale3d),
        math.inf if prune_scale2d is None else float(prune_scale2d), bool(prune_too_big))
    counts = dict(zip(("n_new", "cloned", "split", "pruned"), totals))
    if out is None:
        rng[1:].add_(1)  # what the emit would have done
        for t in stats.values():
            t.zero_()
        return {"source": torch.arange(P, dtype=torch.int64, device=device), "counts": counts}
    means, quats, log_scales, opacity, new_rows, new_moments, source = out
    new = dict(zip(("pts_xyz", "rotations", "scales", "opacity"), (means, quats, log_scales, opacity)))
    new.update(zip(extra, new_rows))
    by_key = dict(zip(keys, new_moments))
    _swap_params(params, optimizer, new, lambda name, key, v: by_key[(name, key)])
    stats.update(densify_state(counts["n_new"], device))
    return {"source": source, "counts": counts}


def densify_reset_opacity(params, optimizer=None, value=0.01):
    """Default density control's opacity reset (INTEGRATION.md §24), in place: params["opacity"] (logits) becomes
    min(opacity, fp32(logit(value))) and that parameter's optimizer moments (state tensors shaped like it) are zeroed, as
    gsplat's reset_opa does.  Two torch ops per tensor, no kernel of its own and no host read.  Returns params["opacity"].
    Raises ValueError on a missing or bad "opacity" tensor and a value outside (0, 1)."""
    where = "densify_reset_opacity"
    if not isinstance(params, dict) or "opacity" not in params:
        raise ValueError(f"{where}: params: expected a dict with key opacity")
    x = params["opacity"]
    if not torch.is_tensor(x) or x.dtype != torch.float32:
        raise ValueError(f"{where}: params['opacity']: expected a float32 tensor, got {x.dtype if torch.is_tensor(x) else type(x)}")
    if isinstance(value, bool) or not isinstance(value, (int, float)) or not 0.0 < value < 1.0:
        raise ValueError(f"{where}: value must be a number in (0, 1), got {value!r}")
    with torch.no_grad():
        x.clamp_(max=_mcmc_logit(value))
    if optimizer is not None:
        for v in optimizer.state.get(x, {}).values():
            if torch.is_tensor(v) and v.shape == x.shape:
                v.zero_()
    return x


_CLOUD_INPUTS = 8  # per cloud: means3D, means2D [V,P,3], sh, colors, feature, opacities, scales, rotations


class _RasterizeClouds(torch.autograd.Function):
    """render_clouds' node.  meta = (views per cloud, return_depth, targets per cloud or None, return_alpha, antialiasing,
    ssim, camera, return_median, return_normal, flow[, views_call, sync_gradients]).  flow: None, or per cloud None or its next-frame poses (a list of
    (viewmatrix, projmatrix) or None per view, or None for the views' own cameras) with that cloud's flow_xyz among the inputs,
    behind every other input.  Outputs per cloud: (color, feature image, radii, depth, alpha, median depth, median id, normal,
    flow), or
    with targets (loss_rgb, loss_embed, color, feature image, radii, loss_depth, loss_mask, depth_pixels, loss_l1, ssim) with
    gradients through the losses only.  views_call: one cloud, rendered by the views calls (render_views').
    sync_gradients (with views_call): None, True or a process group; the
    backward then sums the per-Gaussian gradients over the ranks in one packed all-reduce, started as soon as the blend stage
    has made the feature gradients final."""

    @staticmethod
    def forward(ctx, meta, *flat):
        cloud_views, return_depth, targets, return_alpha, antialiasing, ssim, camera, return_median, return_normal = meta[:9]
        flows = meta[9]
        B, dev = len(cloud_views), flat[0].device
        flow_in = [t.detach() if t is not None else None for t in flat[len(flat) - B:]] if flows is not None else [None] * B
        opts = dict(dtype=torch.float32, device=dev)
        clouds, results, frozen, cots, dms, ssims, images = [], [], [], [], [], [], []
        for b, views in enumerate(cloud_views):
            means3D, _, sh, colors, feature, opacities, scales, rotations = (_prep(t, dev) for t in flat[_CLOUD_INPUTS * b:_CLOUD_INPUTS * (b + 1)])
            V, H, W = len(views), int(views[0].image_height), int(views[0].image_width)
            F = int(feature.shape[1]) if feature is not None else 0
            color = torch.empty((V, 3, H, W), **opts)
            feat_img = torch.empty((V, F, H, W), **opts) if F else None
            depth = torch.empty((V, H, W), **opts) if return_depth else None
            alpha = torch.empty((V, H, W), **opts) if return_alpha else None
            med_depth = torch.empty((V, H, W), **opts) if return_median else None
            med_id = torch.empty((V, H, W), dtype=torch.int32, device=dev) if return_median else None
            normal = torch.empty((V, 3, H, W), **opts) if return_normal else None
            flow = torch.empty((V, 3, H, W), **opts) if flow_in[b] is not None else None
            c = dict(views=views, means3D=means3D, sh=sh, colors=colors, feature=feature, opacity=opacities, scales=scales,
                     rotations=rotations, out_buffers=(color, feat_img, depth, alpha, med_depth, med_id, normal, flow))
            if flow is not None:
                c["flow_means3D"], c["flow_poses"] = flow_in[b], flows[b]
            if targets is None:
                # the id, normal and flow planes are outputs: saved for backward, never kept on ctx
                images += [med_id if return_median else torch.empty(0, device=dev),
                           normal if return_normal else torch.empty(0, device=dev),
                           flow if flow is not None else torch.empty(0, device=dev)]
            if targets is not None:
                t_rgb = _prep(targets[b]["rgb"], dev)
                t_emb = _prep(targets[b].get("embed"), dev) if F else None
                if tuple(t_rgb.shape) != (V, 3, H, W) or (t_emb is not None and tuple(t_emb.shape) != (V, F, H, W)):
                    raise ValueError(f"cloud {b}: targets must be [V,3,H,W] and [V,F,H,W]")
                cot_rgb = torch.empty((V, 3, H, W), **opts)
                cot_emb = torch.empty((V, F, H, W), **opts) if t_emb is not None else (torch.zeros((V, F, H, W), **opts) if F else None)
                loss_acc = torch.empty((V, 2), **opts)
                c["loss_heads"] = (t_rgb, t_emb, cot_rgb, cot_emb, loss_acc)
                c["depth_mask"] = _depth_mask_heads(targets[b].get("depth"), targets[b].get("mask"), V, H, W, dev, f"cloud {b}")
                c["ssim"] = _ssim_head(V, H, W, dev) if ssim else None
                cots.append((cot_rgb, cot_emb))
                dms.append(c["depth_mask"])
                # the SSIM head's planes and the colour target (an input); the image, an output, is saved for backward
                ssims.append(c["ssim"] + (t_rgb,) if ssim else None)
                images.append(color if ssim else torch.empty(0, device=dev))
            clouds.append(c)
        degree = cloud_views[0][0].sh_degree
        include = clouds[0]["feature"] is not None
        outs, streams = rasterize_clouds_raw(clouds, degree, include, cloud_views[0][0].scale_modifier, return_depth=return_depth,
                                             debug=cloud_views[0][0].debug, return_alpha=return_alpha, antialiasing=antialiasing,
                                             return_median=return_median, return_normal=return_normal,
                                             views_call=len(meta) > 10 and meta[10])
        for b, c in enumerate(clouds):
            color, feat_img, depth, alpha, med_depth, med_id, normal, flow = c["out_buffers"]
            radii = torch.stack([o[3] for o in outs[b]])
            empty = lambda: torch.empty(0, device=dev)
            if targets is not None:
                N = float(color.shape[2] * color.shape[3])
                loss_acc = c["loss_heads"][4]
                loss_rgb = loss_acc[:, 0] / (3.0 * N)
                loss_embed = 1.0 - loss_acc[:, 1] / N if c["loss_heads"][1] is not None else torch.zeros((len(c["views"]),), **opts)
                loss_depth, loss_mask, depth_pixels = _depth_mask_losses(c["depth_mask"], N, dev)
                loss_l1, ssim_v = _ssim_losses(c["ssim"], 3.0 * N, dev)
                results += [loss_rgb, loss_embed, color, feat_img if feat_img is not None else empty(), radii, loss_depth, loss_mask,
                            depth_pixels, loss_l1, ssim_v]
                frozen += [radii, color, depth_pixels] + ([feat_img] if feat_img is not None else [])
            else:
                results += [color, feat_img if feat_img is not None else empty(), radii, depth if depth is not None else empty(),
                            alpha if alpha is not None else empty(), med_depth if med_depth is not None else empty(),
                            med_id if med_id is not None else empty(), normal if normal is not None else empty(),
                            flow[:, :2] if flow is not None else empty()]
                frozen += [radii] + ([med_id] if med_id is not None else [])
        ctx.meta, ctx.streams, ctx.degree, ctx.include, ctx.cots, ctx.dms, ctx.ssims = meta, streams, degree, include, cots, dms, ssims
        # capacity, radii and the state buffers per view -- never an output (an output kept on ctx is a reference cycle)
        ctx.state = [[(o[0], o[3], o[4], o[5], o[6]) for o in co] for co in outs]
        ctx.opac_shapes = [flat[_CLOUD_INPUTS * b + 5].shape for b in range(B)]
        e = torch.empty(0, device=dev)
        ctx.save_for_backward(*[x if x is not None else e for c in clouds for x in
                                (c["means3D"], c["sh"], c["colors"], c["feature"], c["scales"], c["rotations"])], *images,
                              *[t if t is not None else e for t in flow_in])
        ctx.mark_non_differentiable(*frozen)  # ONE call: a second one replaces the first
        return tuple(results)

    @staticmethod
    def backward(ctx, *grads):
        cloud_views, return_depth, targets, return_alpha, antialiasing, ssim, camera, return_median, return_normal = ctx.meta[:9]
        flows = ctx.meta[9]
        views_call, group = ctx.meta[10:] if len(ctx.meta) > 10 else (False, None)
        saved = ctx.saved_tensors
        dev = saved[0].device
        B = len(cloud_views)
        flow_in = saved[len(saved) - B:]
        # per cloud: the image (targets with ssim), or the median ids, the normal plane and the flow plane
        images = saved[6 * B:len(saved) - B]
        per = 10 if targets is not None else 9
        clouds = []
        for b, views in enumerate(cloud_views):
            means3D, sh, colors, feature, scales, rotations = (t if t.numel() else None for t in saved[6 * b:6 * b + 6])
            V, H, W = len(views), int(views[0].image_height), int(views[0].image_width)
            F = int(feature.shape[1]) if feature is not None else 0
            g = grads[per * b:per * (b + 1)]
            c = dict(views=views, means3D=means3D, sh=sh, colors=colors, feature=feature, scales=scales, rotations=rotations,
                     want_feature=bool(ctx.needs_input_grad[1 + _CLOUD_INPUTS * b + 4]))
            if targets is not None:
                c["cot_scale"] = _pair_scale(g[0], g[1], V, dev)
                c["grad_color"], c["grad_feature"] = ctx.cots[b]
                if ctx.dms[b] is not None:
                    c["depth_mask"] = ctx.dms[b]
                    c["depth_mask_scale"] = _depth_mask_scale(ctx.dms[b], g[5], g[6], V, dev)
                if ssim:
                    c["ssim"] = ctx.ssims[b][:3] + (images[b], ctx.ssims[b][3])
                    c["ssim_scale"] = _pair_scale(g[8], g[9], V, dev)
            else:
                c["grad_color"] = g[0] if g[0] is not None else torch.zeros((V, 3, H, W), dtype=torch.float32, device=dev)
                if F:
                    c["grad_feature"] = g[1] if g[1] is not None else torch.zeros((V, F, H, W), dtype=torch.float32, device=dev)
                if return_depth and g[3] is not None:
                    c["grad_depth"] = g[3]
                if return_alpha and g[4] is not None:
                    c["grad_alpha"] = g[4]
                if return_median and g[5] is not None:
                    c["grad_median"], c["median_id"] = g[5], images[3 * b]
                if return_normal and g[7] is not None:
                    c["grad_normal"], c["normal"] = g[7], images[3 * b + 1]
                if flow_in[b].numel():
                    c["flow_means3D"], c["flow_poses"], c["flow"] = flow_in[b], flows[b], images[3 * b + 2]
                    c["grad_flow"] = g[8] if g[8] is not None else torch.zeros((V, 2, H, W), dtype=torch.float32, device=dev)
            clouds.append(c)
        # the raw call reads only the blend inputs of the views, their capacity and state (`outs`)
        outs = [[(R, None, None, radii, geom, binb, img) for (R, radii, geom, binb, img) in st] for st in ctx.state]
        after_blend = None
        if group is not None:
            # view-parallel multi-GPU: the one exchange of the path, a SUM all-reduce of the packed buffer; the feature field
            # (final after the blend stage) is already travelling while the per-Gaussian kernel produces the other fields.
            # A view's camera gradients are complete on the rank that rendered it.
            c = clouds[0]
            P, M = c["means3D"].shape[0], c["sh"].shape[1] if c["sh"] is not None else 0
            F = int(c["feature"].shape[1]) if c["feature"] is not None else 0
            pk = PackedGradients(P, F, M, dev, colors=c["colors"] is not None, zero=False)  # every row is written
            grp = None if group is True else group
            c["accumulate_into"] = pk.views
            after_blend = lambda: pk.all_reduce_begin(grp)  # noqa: E731
        res = rasterize_clouds_backward_raw(clouds, outs, ctx.streams, ctx.degree, ctx.include, cloud_views[0][0].scale_modifier,
                                            debug=cloud_views[0][0].debug, antialiasing=antialiasing, camera_grads=camera,
                                            after_blend=after_blend, views_call=views_call)
        if group is not None:
            pk.all_reduce_finish(grp)
        ret = [None]
        for b, r in enumerate(res):
            P = clouds[b]["means3D"].shape[0]
            M = clouds[b]["sh"].shape[1] if clouds[b]["sh"] is not None else 0
            ret += [r["dL_dmeans3D"], r["dL_dmeans2D"], r["dL_dsh"].view(P, M, 3) if M else None, r["dL_dcolors"], r["dL_dfeature"],
                    r["dL_dopacity"].view(ctx.opac_shapes[b]), r["dL_dscales"], r["dL_drotations"]]
        if camera:  # the stacked camera tensors of every cloud behind its Gaussian inputs, four per cloud
            first = 1 + _CLOUD_INPUTS * len(cloud_views)
            for b, r in enumerate(res):
                cam = (r["dL_dviewmatrix"], r["dL_dprojmatrix"], r["dL_dcampos"], r.get("dL_dtan_fov"))
                ret += _camera_outputs(ctx, cam, first + 4 * b)
        if flows is not None:  # every cloud's flow_xyz, behind the camera inputs
            ret += [r.get("dL_dflow_means3D") for r in res]
        return tuple(ret)


def render_clouds(clouds, bg_color=(0.0, 0.0, 0.0), return_depth=False, normalize_feature=True, return_alpha=False,
                  antialiasing=False, ssim=False, return_median_depth=False, return_normal=False, planar_depth=False):
    """Render several Gaussian clouds, each with its own cameras, in one autograd node: e.g. the current and the deformed
    next frame of ManiGaussian's dynamic-field step (neural_rendering.py:283, :324) for every sample of the batch.

    clouds: sequence of dicts with the keyword names of render_views -- "cameras", optional "view_ids", "pts_xyz",
    "rotations", "scales", "opacity", "features_color" or "pts_rgb", optional "features_language" and optional "targets".
    The clouds share the SH degree, the feature width F and the colour mode (ValueError naming the field otherwise); within a
    cloud all views share one image size, different clouds may differ.  Targets are given on all clouds or on none.
    Returns one dict per cloud with the keys and shapes render_views returns for it ("loss_rgb" / "loss_embed" with targets,
    and "loss_depth" / "depth_pixels" / "loss_mask" with "depth" / "mask" targets; "depth" / "alpha" [V,H,W] when asked for).
    A cloud whose "features_language" does not require grad gets no feature gradient computed (e.g. the next frame of the
    dyna step, which renders the detached current features); its feature cotangents still reach its other gradients.
    antialiasing: every cloud renders with the anti-aliased projection, as in render_views.
    Camera gradients: as in render_views, per cloud (with the field of view of cameras from a learnable intr); clouds that
    share camera tensors (the dyna pair) receive the sum.
    ssim: every cloud also returns "loss_l1" and "ssim" [V], as in render_views; needs targets.
    return_median_depth: every cloud also returns "median_depth" and "median_id" [V,H,W], as in render_views; not with targets.
    return_normal: every cloud also returns "normal" [V,3,H,W], as in render_views; not with targets.
    planar_depth: every cloud's depth follows each Gaussian's tilt, as in render_views.
    A cloud's optional "flow_xyz" [P,3] (its next-frame means) and "flow_cameras" render its "flow" [V,2,H,W], as
    render_views' flow_xyz and flow_cameras.  For the dyna pair pass the next cloud's pts_xyz tensor as the current cloud's
    flow_xyz: autograd sums both of its uses.  Not with targets, return_normal or planar_depth."""
    if not clouds:
        raise ValueError("render_clouds needs at least one cloud")
    with_targets = [c.get("targets") is not None for c in clouds]
    if any(with_targets) and not all(with_targets):
        raise ValueError("targets must be given on all clouds or on none")
    if ssim and not all(with_targets):
        raise ValueError("ssim=True needs targets on every cloud (the colour target \"rgb\")")
    if all(with_targets) and return_depth:
        raise ValueError("targets and return_depth cannot be combined")
    if all(with_targets) and return_alpha:
        raise ValueError("targets and return_alpha cannot be combined")
    if all(with_targets) and return_median_depth:
        raise ValueError("targets and return_median_depth cannot be combined")
    if all(with_targets) and return_normal:
        raise ValueError("targets and return_normal cannot be combined")
    if len({c.get("features_color") is None for c in clouds}) > 1:
        raise ValueError("clouds disagree on the colour mode (SHs or precomputed colors)")
    device = clouds[0]["pts_xyz"].device
    cloud_views, batches = [], []
    for b, c in enumerate(clouds):
        include = c.get("features_language") is not None
        sh_degree = 3 if c.get("features_color") is None else 1
        cameras, view_ids = c["cameras"], c.get("view_ids")
        if isinstance(cameras, CameraBatch):
            ids = list(range(len(cameras))) if view_ids is None else list(view_ids)
            views = tuple(cameras.settings(i, _background(bg_color, device), sh_degree, include) for i in ids)
            batches.append(_batch_cameras(cameras, ids) if ids else None)
        else:
            views = tuple(cameras if view_ids is None else [cameras[i] for i in view_ids])
            batches.append(None)
        if not views:
            raise ValueError(f"cloud {b} has no views")
        if c.get("features_color") is None and c.get("pts_rgb") is None:
            raise ValueError("Please provide excatly one of either SHs or precomputed colors!")
        if any((int(s.image_height), int(s.image_width)) != (int(views[0].image_height), int(views[0].image_width)) for s in views):
            raise ValueError(f"cloud {b}: all views of a cloud need one image size")
        cloud_views.append(views)
    if len({int(s.sh_degree) for views in cloud_views for s in views}) > 1:
        raise ValueError("clouds disagree on the SH degree")
    _prep_clouds([dict(means3D=c["pts_xyz"], sh=c.get("features_color"), colors=c.get("pts_rgb") if c.get("features_color") is None else None,
                       feature=c.get("features_language")) for c in clouds], device, True)
    if planar_depth:
        cloud_views = [tuple(_with_planar_depth(s) for s in views) for views in cloud_views]
    flat, vsps = [], []
    for c, views in zip(clouds, cloud_views):
        f = c.get("features_language")
        if f is not None and normalize_feature:
            f = normalize_features(f)
        # its .grad receives each view's screen-space mean gradients, as in render_views
        vsps.append(torch.zeros((len(views), c["pts_xyz"].shape[0], 3), dtype=torch.float32, device=device, requires_grad=True))
        flat += [c["pts_xyz"], vsps[-1], c.get("features_color"), c.get("pts_rgb") if c.get("features_color") is None else None, f,
                 c["opacity"], c["scales"], c["rotations"]]
    targets = [c["targets"] for c in clouds] if all(with_targets) else None
    flows = None
    if any(c.get("flow_xyz") is not None for c in clouds):
        for bad, what in ((targets is not None, "targets"), (return_normal, "return_normal"),
                          (any(bool(getattr(s, "planar_depth", False)) for views in cloud_views for s in views), "planar_depth")):
            if bad:
                raise ValueError(f"flow_xyz cannot be combined with {what}")
        flows = []
        for c, views in zip(clouds, cloud_views):
            if c.get("flow_xyz") is None:
                flows.append(None)
                continue
            sh_degree = 3 if c.get("features_color") is None else 1
            poses = _flow_inputs(views, c["pts_xyz"], c["flow_xyz"], c.get("flow_cameras"), c.get("view_ids"),
                                 _background(bg_color, device), sh_degree, c.get("features_language") is not None)
            flows.append(poses)
        flows = tuple(flows)
    aa = bool(antialiasing) or any(bool(getattr(s, "antialiasing", False)) for views in cloud_views for s in views)
    cams = [_camera_inputs(views, batch=bt) for views, bt in zip(cloud_views, batches)]
    camera = any(c[0] is not None for c in cams)
    if camera:  # every cloud's stacked cameras, as explicit inputs (the dyna pair's shared tensors get both frames' sums)
        cams = [c if c[0] is not None else _camera_inputs(views, force=True, batch=bt)
                for c, views, bt in zip(cams, cloud_views, batches)]
        flat += [t for c in cams for t in c]
    if flows is not None:
        flat += [c.get("flow_xyz") for c in clouds]
    out = _RasterizeClouds.apply((tuple(cloud_views), bool(return_depth), targets, bool(return_alpha), aa, bool(ssim), camera,
                                  bool(return_median_depth), bool(return_normal), flows), *flat)
    ret = []
    for b, c in enumerate(clouds):
        include, vsp = c.get("features_language") is not None, vsps[b]
        if targets is not None:
            loss_rgb, loss_embed, color, feat_img, radii, loss_depth, loss_mask, depth_pixels, loss_l1, ssim_v = out[10 * b:10 * b + 10]
            r = {"render": color, "render_embed": feat_img if include else None, "viewspace_points": vsp, "radii": radii,
                 "loss_rgb": loss_rgb, "loss_embed": loss_embed}
            if targets[b].get("depth") is not None:
                r["loss_depth"], r["depth_pixels"] = loss_depth, depth_pixels
            if targets[b].get("mask") is not None:
                r["loss_mask"] = loss_mask
            if ssim:
                r["loss_l1"], r["ssim"] = loss_l1, ssim_v
            ret.append(r)
        else:
            color, feat_img, radii, depth, alpha, med_depth, med_id, normal, flow = out[9 * b:9 * b + 9]
            r = {"render": color, "render_embed": feat_img if include else None, "viewspace_points": vsp, "radii": radii}
            if return_depth:
                r["depth"] = depth
            if return_alpha:
                r["alpha"] = alpha
            if return_median_depth:
                r["median_depth"], r["median_id"] = med_depth, med_id
            if return_normal:
                r["normal"] = normal
            if c.get("flow_xyz") is not None:
                r["flow"] = flow
            ret.append(r)
    return ret

"""Host-side mirror of the reference's Python operator for the rasterizer hot path.

Same names, argument order, return values and error behaviour as
DGR/diff_gaussian_rasterization/__init__.py (GaussianRasterizationSettings :166-179,
GaussianRasterizer :181-233, _RasterizeGaussians :46-164) and the pybind functions of DGR/ext.cpp:14-18
(rasterize_gaussians / rasterize_gaussians_backward / mark_visible, DGR/rasterize_points.cu:36-247), so that
ManiGaussian's agents/manigaussian_bc/gaussian_renderer/__init__.py:14-94 runs unchanged.  PyTorch is used for
device memory, streams and autograd plumbing only; all computation happens in the sm_90a library behind
include/mgs_rasterizer.h.

Supersets of the reference: the feature width F is read from the tensor at run time (0..512) instead of being
compiled in (config.h:16; widths above 32 blend in groups of 32 channels), `return_depth=True` adds a view-space
depth plane, and `return_alpha=True` adds the accumulated-opacity plane 1 - final_T.  `return_median_depth=True` adds the
median-depth plane and each pixel's surface Gaussian, and `return_normal=True` the surface-normal plane.
"""
from typing import NamedTuple

import ctypes
import math
import os

import torch
import torch.nn as nn

from . import _binding as _b


def _ptr(t):
    """Device pointer of a tensor; None / empty tensor -> NULL (the reference's `data_ptr() == nullptr`)."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


def _prep(t, device):
    """float32, contiguous, on `device` (the reference calls .contiguous() on every input, rasterize_points.cu:104-125)."""
    if t is None:
        return None
    if t.numel() == 0:
        return t
    if t.dtype != torch.float32 or t.device != device or not t.is_contiguous():
        t = t.to(device=device, dtype=torch.float32).contiguous()
    return t


class _Alloc:
    """State-buffer allocation backed by torch's caching allocator (replaces resizeFunctional, rasterize_points.cu:27-33).
    One process-wide C callback serves every call; the `user` pointer selects the _Alloc instance."""
    _live = {}
    _next = [1]

    def __init__(self, device):
        self.device = device
        self.tensor = None
        self.error = None  # exception raised inside the C callback (ctypes would swallow it): re-raised by the caller
        self.key = _Alloc._next[0]
        _Alloc._next[0] += 1
        _Alloc._live[self.key] = self

    def release(self):
        _Alloc._live.pop(self.key, None)
        if self.tensor is None:
            self.tensor = torch.empty(0, dtype=torch.uint8, device=self.device)
        return self.tensor

    def alloc(self, nbytes):
        # Round large requests up to a geometric bucket (<= 25 % slack): the binning state's size follows the
        # data-dependent instance count, and near-equal sizes must hit the same cached block or the caching
        # allocator keeps falling back to cudaMalloc for many iterations.
        n = max(int(nbytes), 1)
        if n > (1 << 20):
            q = 1 << max(20, n.bit_length() - 3)
            n = (n + q - 1) // q * q
        self.tensor = torch.empty(n, dtype=torch.uint8, device=self.device)
        return self.tensor.data_ptr()


def _alloc_trampoline(user, nbytes):
    a = _Alloc._live.get(int(user or 0))
    if a is None:
        return 0
    try:
        return a.alloc(nbytes)
    except BaseException as ex:  # e.g. torch.cuda.OutOfMemoryError: hand it to the caller instead of losing it in ctypes
        a.error = ex
        return 0


def _checked(allocs, rc, what):
    """_b.check that re-raises an exception stashed by an allocator callback and always releases the allocators"""
    err = next((a.error for a in allocs if a.error is not None), None)
    if err is not None:
        for a in allocs:
            a.release()
        raise err
    try:
        return _b.check(rc, what)
    except Exception:
        for a in allocs:
            a.release()
        raise


_ALLOC_CB = _b.ALLOC_FN(_alloc_trampoline)


def _stream(device):
    return torch.cuda.current_stream(device).cuda_stream


def rasterize_gaussians_raw(bg, means3D, colors, language_feature, opacity, scales, rotations, scale_modifier,
                            cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width,
                            sh, degree, campos, prefiltered, debug, include_feature, return_depth=False):
    """Same contract as the reference's `_C.rasterize_gaussians` (DGR/rasterize_points.cu:36-128).

    Returns (num_rendered, color [3,H,W], feature [F,H,W] or [1], radii [P] int32, geomBuffer, binningBuffer,
    imgBuffer) and, when return_depth, an extra trailing depth [H,W] tensor.
    """
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    if not means3D.is_cuda:
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    L = _b.lib()
    dev = means3D.device
    P, H, W = means3D.size(0), int(image_height), int(image_width)
    means3D, colors, language_feature, opacity = (_prep(x, dev) for x in (means3D, colors, language_feature, opacity))
    scales, rotations, cov3D_precomp, sh = (_prep(x, dev) for x in (scales, rotations, cov3D_precomp, sh))
    bg, viewmatrix, projmatrix, campos = (_prep(x, dev) for x in (bg, viewmatrix, projmatrix, campos))
    F = 0
    if include_feature and language_feature is not None and language_feature.numel() > 0:
        F = language_feature.size(1)
    M = sh.size(1) if (sh is not None and sh.numel() != 0) else 0
    out_color = torch.empty((3, H, W), dtype=torch.float32, device=dev)
    out_feature = torch.empty((F, H, W), dtype=torch.float32, device=dev) if include_feature else \
        torch.zeros((1,), dtype=torch.float32, device=dev)
    out_depth = torch.empty((H, W), dtype=torch.float32, device=dev) if return_depth else None
    radii = torch.empty((P,), dtype=torch.int32, device=dev)
    ga, ba, ia = _Alloc(dev), _Alloc(dev), _Alloc(dev)
    rendered = 0
    if P != 0:
        with torch.cuda.device(dev):
            rendered = _checked((ga, ba, ia), L.mgs_forward(
                _ALLOC_CB, ga.key, _ALLOC_CB, ba.key, _ALLOC_CB, ia.key,
                P, int(degree), M, F,
                _ptr(bg), W, H,
                _ptr(means3D), _ptr(sh), _ptr(colors), _ptr(language_feature) if F else None,
                _ptr(opacity), _ptr(scales), float(scale_modifier), _ptr(rotations),
                _ptr(cov3D_precomp), _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos),
                float(tan_fovx), float(tan_fovy), int(bool(prefiltered)),
                _ptr(out_color), _ptr(out_feature) if F else None, _ptr(out_depth), _ptr(radii),
                int(bool(debug)), _stream(dev)), "mgs_forward")
    else:
        out_color.zero_()
        if include_feature:
            out_feature.zero_()
        if out_depth is not None:
            out_depth.zero_()
    ret = (rendered, out_color, out_feature, radii, ga.release(), ba.release(), ia.release())
    return ret + (out_depth,) if return_depth else ret


def rasterize_gaussians_backward_raw(bg, means3D, radii, colors, language_feature, scales, rotations, scale_modifier,
                                     cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color,
                                     dL_dout_language_feature, sh, degree, campos, geomBuffer, R, binningBuffer,
                                     imageBuffer, debug, include_feature, dL_dout_depth=None, accumulate_into=None):
    """Same contract as the reference's `_C.rasterize_gaussians_backward` (DGR/rasterize_points.cu:131-225):
    returns (dL_dmeans2D, dL_dcolors, dL_dlanguage_feature, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh,
    dL_dscales, dL_drotations).

    accumulate_into: optional dict of preallocated fp32 tensors keyed like manigaussian_b200.parallel.FIELDS
    (dL_dmeans3D, dL_dmeans2D, dL_dscales, dL_drotations, dL_dopacity, dL_dsh, dL_dfeature[, dL_dcolors]); the gradients of
    this view are then ADDED to what they hold (C ABI `accumulate=1`; calls sharing buffers must be issued on one stream)
    and the same tensors are returned.  For several views of one cloud prefer rasterize_views_backward_raw."""
    L = _b.lib()
    dev = means3D.device
    P = means3D.size(0)
    H, W = dL_dout_color.size(1), dL_dout_color.size(2)
    means3D, colors, language_feature = (_prep(x, dev) for x in (means3D, colors, language_feature))
    scales, rotations, cov3D_precomp, sh = (_prep(x, dev) for x in (scales, rotations, cov3D_precomp, sh))
    bg, viewmatrix, projmatrix, campos = (_prep(x, dev) for x in (bg, viewmatrix, projmatrix, campos))
    dL_dout_color = _prep(dL_dout_color, dev)
    dL_dout_depth = _prep(dL_dout_depth, dev)
    F = 0
    if include_feature and language_feature is not None and language_feature.numel() > 0:
        F = language_feature.size(1)
        dL_dout_language_feature = _prep(dL_dout_language_feature, dev)
    M = sh.size(1) if (sh is not None and sh.numel() != 0) else 0
    opts = dict(dtype=torch.float32, device=dev)
    acc = accumulate_into
    if acc is not None:
        need = ["dL_dmeans3D", "dL_dmeans2D", "dL_dopacity"]
        need += ["dL_dscales", "dL_drotations"] if (scales is not None and scales.numel() != 0) else []
        need += ["dL_dcolors"] if (colors is not None and colors.numel() != 0) else []
        missing = [k for k in need if acc.get(k) is None]
        if missing:
            raise ValueError(f"accumulate_into lacks {missing}: gradients of inputs of this render would be dropped")
        dL_dmeans3D, dL_dmeans2D, dL_dopacity = acc["dL_dmeans3D"], acc["dL_dmeans2D"], acc["dL_dopacity"]
        dL_dscales, dL_drotations = acc.get("dL_dscales"), acc.get("dL_drotations")
        dL_dsh = acc.get("dL_dsh") if M else torch.empty((P, 0, 3), **opts)
        dL_dfeature = acc.get("dL_dfeature") if F else torch.zeros((1,), **opts)
        dL_dcolors, dL_dcov3D = acc.get("dL_dcolors"), None
    else:
        dL_dmeans3D = torch.empty((P, 3), **opts)
        dL_dmeans2D = torch.empty((P, 3), **opts)
        dL_dcolors = torch.empty((P, 3), **opts)
        dL_dfeature = torch.empty((P, F), **opts) if F else torch.zeros((1,), **opts)
        dL_dopacity = torch.empty((P, 1), **opts)
        dL_dcov3D = torch.empty((P, 6), **opts)
        dL_dsh = torch.empty((P, M, 3), **opts)
        dL_dscales = torch.empty((P, 3), **opts)
        dL_drotations = torch.empty((P, 4), **opts)
    if P != 0:
        scratch = torch.empty((L.mgs_backward_scratch_bytes(P),), dtype=torch.uint8, device=dev)
        has_sr = scales is not None and scales.numel() != 0
        with torch.cuda.device(dev):
            _b.check(L.mgs_backward(
                P, int(degree), M, F, int(R),
                _ptr(bg), W, H,
                _ptr(means3D), _ptr(sh), _ptr(colors), _ptr(language_feature) if F else None,
                _ptr(scales), float(scale_modifier), _ptr(rotations), _ptr(cov3D_precomp),
                _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), float(tan_fovx), float(tan_fovy),
                _ptr(radii), _ptr(geomBuffer), _ptr(binningBuffer), _ptr(imageBuffer),
                _ptr(dL_dout_color), _ptr(dL_dout_language_feature) if F else None, _ptr(dL_dout_depth),
                _ptr(dL_dmeans2D), None, _ptr(dL_dopacity), _ptr(dL_dcolors), _ptr(dL_dfeature) if F else None,
                _ptr(dL_dmeans3D), _ptr(dL_dcov3D), _ptr(dL_dsh) if M else None,
                _ptr(dL_dscales) if has_sr else None, _ptr(dL_drotations) if has_sr else None,
                _ptr(scratch), int(acc is not None), int(bool(debug)), _stream(dev)), "mgs_backward")
        if not has_sr and acc is None:
            dL_dscales.zero_()
            dL_drotations.zero_()
    return (dL_dmeans2D, dL_dcolors, dL_dfeature, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations)


def mark_visible_raw(means3D, viewmatrix, projmatrix):
    """Same contract as the reference's `_C.mark_visible` (DGR/rasterize_points.cu:227-247)."""
    L = _b.lib()
    dev = means3D.device
    P = means3D.size(0)
    means3D, viewmatrix, projmatrix = (_prep(x, dev) for x in (means3D, viewmatrix, projmatrix))
    present = torch.zeros((P,), dtype=torch.uint8, device=dev)
    if P != 0:
        with torch.cuda.device(dev):
            _b.check(L.mgs_mark_visible(P, _ptr(means3D), _ptr(viewmatrix), _ptr(projmatrix), _ptr(present), _stream(dev)),
                     "mgs_mark_visible")
    return present.bool()


def state_array(which, name, state, a0, a1=0):
    """Device address of a named array inside an opaque state buffer (tests only)."""
    import ctypes
    out = ctypes.c_void_p()
    _b.check(_b.lib().mgs_state_array(which.encode(), name.encode(), state.data_ptr(), int(a0), int(a1), ctypes.byref(out)),
             "mgs_state_array")
    return out.value


def _is_device_fov(s):
    return any(torch.is_tensor(t) and t.is_cuda for t in (s.tanfovx, s.tanfovy))


def cpu_deep_copy_tuple(input_tuple):
    return tuple(item.cpu().clone() if isinstance(item, torch.Tensor) else item for item in input_tuple)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, language_feature_precomp, opacities, scales, rotations,
                        cov3Ds_precomp, raster_settings, return_depth=False, return_alpha=False, return_median_depth=False,
                        return_normal=False, flow_means3D=None, flow_pose=None):
    s = raster_settings
    # camera tensors that require grad become explicit inputs of the node, which then returns their gradients; a field of
    # view held as CUDA tensors (learnable intrinsics) joins them as two more inputs, tanfovx and tanfovy
    cam = (s.viewmatrix, s.projmatrix, s.campos)
    if _is_device_fov(s):
        cam += (s.tanfovx, s.tanfovy)
    if not any(torch.is_tensor(t) and t.requires_grad for t in cam):
        cam = ()
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, language_feature_precomp, opacities, scales,
                                     rotations, cov3Ds_precomp, raster_settings, return_depth, return_alpha,
                                     bool(return_median_depth), bool(return_normal), flow_means3D, flow_pose, *cam)


_CAM_FIRST = 16  # position of the first camera input of _RasterizeGaussians


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, language_feature_precomp, opacities, scales, rotations,
                cov3Ds_precomp, raster_settings, return_depth=False, return_alpha=False, return_median=False,
                return_normal=False, flow_means3D=None, flow_pose=None, *cam):
        s = raster_settings
        ctx.flow = flow_means3D is not None
        ctx.flow_pose = flow_pose
        flow_means3D = flow_means3D.detach() if ctx.flow else None
        flow = None
        args = (s.bg, means3D, colors_precomp, language_feature_precomp, opacities, scales, rotations, s.scale_modifier,
                cov3Ds_precomp, s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, s.image_height, s.image_width, sh,
                s.sh_degree, s.campos, s.prefiltered, s.debug, s.include_feature)
        ctx.async_view = None
        views_path = means3D.is_cuda and means3D.size(0) > 0
        aa = bool(getattr(s, "antialiasing", False))
        ctx.antialiasing = aa
        ctx.camera = len(cam) > 0
        # the device field of view, when the settings carry one (read by the kernels in place of host floats)
        tf = _fov_column([s], means3D.device) if (views_path and _is_device_fov(s)) else None
        ctx.tan_fov = tf
        alpha = med_depth = med_id = normal = None
        if return_normal and (cov3Ds_precomp is not None and cov3Ds_precomp.numel() != 0):
            raise ValueError("return_normal needs scales and rotations: a precomputed covariance has no axis to take a normal from")
        # planar depth, like the camera models, exists on the multi-view entry points only
        orth = bool(getattr(s, "orthographic", False)) or getattr(s, "fisheye", None) is not None \
            or getattr(s, "distortion", None) is not None or bool(getattr(s, "planar_depth", False))
        ctx.orthographic = orth
        if ctx.flow and not views_path:
            raise RuntimeError("the flow plane needs a CUDA cloud with at least one Gaussian")
        if (return_alpha or return_median or return_normal or aa or orth or ctx.camera or ctx.flow) and views_path:
            # the alpha plane, the median planes, the anti-aliased, orthographic, fisheye and distorted projections and the camera
            # gradients exist on
            # the multi-view entry points only: debug renders take them too, with the snapshot dump
            cpu_args = cpu_deep_copy_tuple(args) if s.debug else None
            try:
                outs, streams = rasterize_views_raw([s], means3D, colors_precomp, language_feature_precomp, opacities, scales,
                                                    rotations, s.scale_modifier, cov3Ds_precomp, sh, s.sh_degree, s.include_feature,
                                                    return_depth=return_depth, debug=s.debug, return_alpha=return_alpha,
                                                    antialiasing=aa, tan_fov=tf, return_median=return_median,
                                                    return_normal=return_normal, flow_means3D=flow_means3D,
                                                    flow_poses=[flow_pose] if ctx.flow else None)
            except Exception as ex:
                if s.debug:
                    torch.save(cpu_args, "snapshot_fw.dump")
                    print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
                raise ex
            out = outs[0]
            planes = 7 + bool(return_depth)
            alpha = out[planes] if return_alpha else None
            nf = int(ctx.flow)
            if ctx.flow:
                flow = out[-1]
            if return_normal:
                normal = out[-1 - nf]
            if return_median:
                med_depth, med_id = out[-2 - bool(return_normal) - nf], out[-1 - bool(return_normal) - nf]
            ctx.async_view = (int(out[0]), streams)  # as below: never the outputs themselves
        elif s.debug:
            cpu_args = cpu_deep_copy_tuple(args)  # copy before they can be corrupted
            try:
                out = rasterize_gaussians_raw(*args, return_depth=return_depth)
            except Exception as ex:
                torch.save(cpu_args, "snapshot_fw.dump")
                print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
                raise ex
        elif means3D.is_cuda and means3D.size(0) > 0:
            # no host synchronisation: the binning state is sized from the instance counts of earlier calls (the reference reads
            # the count back on every call, rasterizer_impl.cu:284); the operator itself never exposes the count
            outs, streams = rasterize_views_raw([s], means3D, colors_precomp, language_feature_precomp, opacities, scales, rotations,
                                                s.scale_modifier, cov3Ds_precomp, sh, s.sh_degree, s.include_feature,
                                                return_depth=return_depth, tan_fov=tf)
            out = outs[0]
            # only the capacity and the streams: the images and radii in `outs` are OUTPUTS of this node, and an output kept on
            # ctx is a reference cycle (output -> grad_fn -> ctx -> output) that no collector frees -- the state buffers and the
            # radii come back through saved_tensors in the backward
            ctx.async_view = (int(out[0]), streams)
        else:
            out = rasterize_gaussians_raw(*args, return_depth=return_depth)
            # no Gaussians: nothing covers any pixel
            hw, odev = (int(s.image_height), int(s.image_width)), out[1].device
            if return_alpha:
                alpha = torch.zeros(hw, dtype=torch.float32, device=odev)
            if return_median:
                med_depth, med_id = torch.zeros(hw, dtype=torch.float32, device=odev), torch.full(hw, -1, dtype=torch.int32, device=odev)
            if return_normal:
                normal = torch.zeros((3,) + hw, dtype=torch.float32, device=odev)
        num_rendered, color, language_feature, radii, geomBuffer, binningBuffer, imgBuffer = out[:7]
        depth = out[7] if return_depth else None
        ctx.raster_settings = s
        ctx.num_rendered = num_rendered
        ctx.return_depth = return_depth
        ctx.return_alpha = return_alpha
        ctx.return_median = return_median
        ctx.return_normal = return_normal
        # the id and normal planes are outputs: they reach the backward through save_for_backward, never through ctx (reference
        # cycle)
        ctx.save_for_backward(colors_precomp, language_feature_precomp, means3D, scales, rotations, cov3Ds_precomp, radii,
                              sh, geomBuffer, binningBuffer, imgBuffer, med_id if return_median else None,
                              normal if return_normal else None, flow, flow_means3D)
        if return_median:
            ctx.mark_non_differentiable(radii, med_id)
        else:
            ctx.mark_non_differentiable(radii)
        return (color, language_feature, radii) + ((depth,) if return_depth else ()) + ((alpha,) if return_alpha else ()) + \
            ((med_depth, med_id) if return_median else ()) + ((normal,) if return_normal else ()) + \
            ((flow[:2],) if ctx.flow else ())

    @staticmethod
    def backward(ctx, grad_out_color, grad_out_language_feature, _radii=None, *grad_planes):
        # grad_planes: the depth gradient when return_depth, then the alpha gradient when return_alpha, then the median-depth
        # gradient and the (absent) id gradient when return_median, then the normal gradient when return_normal
        grad_out_depth = grad_planes[0] if ctx.return_depth else None
        grad_out_alpha = grad_planes[int(ctx.return_depth)] if ctx.return_alpha else None
        # and the flow gradient, last, with a flow plane
        nf = int(ctx.flow)
        grad_out_median = grad_planes[-2 - int(ctx.return_normal) - nf] if ctx.return_median else None
        grad_out_normal = grad_planes[-1 - nf] if ctx.return_normal else None
        grad_out_flow = grad_planes[-1] if ctx.flow else None
        s = ctx.raster_settings
        (colors_precomp, language_feature_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer,
         binningBuffer, imgBuffer, med_id, normal, flow, flow_means3D) = ctx.saved_tensors
        if ctx.flow and grad_out_flow is None:
            grad_out_flow = torch.zeros((2, s.image_height, s.image_width), dtype=torch.float32, device=means3D.device)
        if grad_out_color is None:
            grad_out_color = torch.zeros((3, s.image_height, s.image_width), dtype=torch.float32, device=means3D.device)
        if s.include_feature and grad_out_language_feature is None:
            grad_out_language_feature = torch.zeros((language_feature_precomp.size(1), s.image_height, s.image_width),
                                                    dtype=torch.float32, device=means3D.device)
        args = (s.bg, means3D, radii, colors_precomp, language_feature_precomp, scales, rotations, s.scale_modifier,
                cov3Ds_precomp, s.viewmatrix, s.projmatrix, s.tanfovx, s.tanfovy, grad_out_color,
                grad_out_language_feature, sh, s.sh_degree, s.campos, geomBuffer, ctx.num_rendered, binningBuffer,
                imgBuffer, s.debug, s.include_feature)
        depth_grad = grad_out_depth if ctx.return_depth else None
        if ctx.async_view is not None:
            cap, streams = ctx.async_view
            outs = [ViewOut((cap, None, None, radii, geomBuffer, binningBuffer, imgBuffer))]
            cpu_args = cpu_deep_copy_tuple(args) if (s.debug and (ctx.return_alpha or ctx.return_median or ctx.return_normal or
                                                                  ctx.antialiasing or ctx.orthographic or ctx.camera)) else None
            try:
                grads = rasterize_views_backward_raw(
                    [s], outs, streams, [grad_out_color], [grad_out_language_feature] if s.include_feature else None, means3D,
                    colors_precomp, language_feature_precomp, scales, rotations, s.scale_modifier, cov3Ds_precomp, sh, s.sh_degree,
                    s.include_feature, grads_depth=[depth_grad] if depth_grad is not None else None, debug=s.debug,
                    grads_alpha=[grad_out_alpha] if grad_out_alpha is not None else None, antialiasing=ctx.antialiasing,
                    camera_grads=True if ctx.camera else None, tan_fov=ctx.tan_fov,
                    grads_median=[grad_out_median] if grad_out_median is not None else None,
                    median_ids=[med_id] if grad_out_median is not None else None,
                    grads_normal=[grad_out_normal] if (grad_out_normal is not None and normal is not None) else None,
                    normals=[normal] if (grad_out_normal is not None and normal is not None) else None,
                    flow_means3D=flow_means3D, flow_poses=[ctx.flow_pose] if ctx.flow else None,
                    grads_flow=[grad_out_flow] if ctx.flow else None, flows=[flow] if ctx.flow else None)
            except Exception as ex:
                if cpu_args is not None:
                    torch.save(cpu_args, "snapshot_bw.dump")
                    print("\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
                raise ex
        elif s.debug:
            cpu_args = cpu_deep_copy_tuple(args)
            try:
                grads = rasterize_gaussians_backward_raw(*args, dL_dout_depth=depth_grad)
            except Exception as ex:
                torch.save(cpu_args, "snapshot_bw.dump")
                print("\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
                raise ex
        else:
            grads = rasterize_gaussians_backward_raw(*args, dL_dout_depth=depth_grad)
        (grad_means2D, grad_colors_precomp, grad_language_feature_precomp, grad_opacities, grad_means3D,
         grad_cov3Ds_precomp, grad_sh, grad_scales, grad_rotations) = grads[:9]
        grad_cam = ()
        if ctx.camera:
            # zero gradients when the views path did not run (no Gaussians: nothing depends on the camera)
            z = lambda n: torch.zeros((1, n), device=means3D.device)  # noqa: E731
            cg = grads[9] if len(grads) > 9 + int(ctx.flow) else (z(16), z(16), z(3), z(2))
            dvm, dpm, dcp = cg[:3]
            gs, ts = [dvm, dpm, dcp], [s.viewmatrix, s.projmatrix, s.campos]
            if _is_device_fov(s):   # tanfovx, tanfovy: the two entries of the view's dL/dtan_fov
                dtf = cg[3] if len(cg) > 3 else z(2)
                gs += [dtf[0, 0], dtf[0, 1]]
                ts += [s.tanfovx, s.tanfovy]
            grad_cam = tuple(g.reshape(t.shape) if ctx.needs_input_grad[_CAM_FIRST + i] else None for i, (g, t) in enumerate(zip(gs, ts)))

        def _or_none(g, inp):
            return g if (inp is not None and inp.numel() != 0) else None

        return (grad_means3D, grad_means2D, _or_none(grad_sh, sh), _or_none(grad_colors_precomp, colors_precomp),
                _or_none(grad_language_feature_precomp, language_feature_precomp) if s.include_feature else None,
                grad_opacities, _or_none(grad_scales, scales), _or_none(grad_rotations, rotations),
                _or_none(grad_cov3Ds_precomp, cov3Ds_precomp), None, None, None, None, None,
                grads[-1] if ctx.flow else None, None) + grad_cam


class _Settings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool
    include_feature: bool


class GaussianRasterizationSettings(_Settings):
    """The reference's 13 fields (DGR/diff_gaussian_rasterization/__init__.py:166-179) and a 14th argument, `antialiasing`
    (default False; positional after include_feature, or by keyword): the anti-aliased projection of the 3DGS authors'
    current rasterizer (Mip-Splatting's 2D filter; INTEGRATION.md §5).  `antialiasing` is an attribute, not a tuple field:
    the settings still unpack into the reference's own 13-field NamedTuple, and `_fields` is the reference's.
    `orthographic` (default False; keyword, or positional after antialiasing) is an attribute in the same way: True makes the
    view orthographic, with tanfovx / tanfovy its half-width and half-height in view-space units and projmatrix an
    orthographic matrix (cameras.projection_orthographic; include/mgs_rasterizer.h, mgs_render_options.ortho).
    `fisheye` (default None; keyword, or positional after orthographic) is an attribute in the same way: the view's
    Kannala-Brandt parameters (cx, cy, k1, k2, k3, k4, theta_max), or a dict with those keys, make it a fisheye view, with
    tanfovx / tanfovy holding W / (2 fx) and H / (2 fy) (fx, fy in pixels per radian; include/mgs_rasterizer.h,
    mgs_render_options.fisheye; cameras.build_fisheye_cameras).  It cannot be combined with orthographic=True.
    `distortion` (default None; keyword, or positional after fisheye) is an attribute in the same way: the view's OpenCV
    parameters (cx, cy, k1, k2, p1, p2, k3, k4, k5, k6, r_max), or a dict with those keys, make it a distorted-pinhole view,
    with tanfovx / tanfovy holding W / (2 fx) and H / (2 fy) (include/mgs_rasterizer.h, mgs_render_options.distortion;
    cameras.build_distorted_cameras).  It cannot be combined with orthographic=True or fisheye.
    `planar_depth` (default False; keyword, or positional after distortion) is an attribute in the same way: True makes the
    depth plane, the depth head and the median depth take each Gaussian's depth along the pixel's ray, affine in the pixel
    offset, instead of its centre depth (include/mgs_rasterizer.h, mgs_render_options.planar_depth).  It is a per-call setting: the
    views of one call must agree."""
    antialiasing = False
    orthographic = False
    fisheye = None
    distortion = None
    planar_depth = False

    def __new__(cls, image_height, image_width, tanfovx, tanfovy, bg, scale_modifier, viewmatrix, projmatrix, sh_degree, campos,
                prefiltered, debug, include_feature, antialiasing=False, orthographic=False, fisheye=None, distortion=None,
                planar_depth=False):
        self = super().__new__(cls, image_height, image_width, tanfovx, tanfovy, bg, scale_modifier, viewmatrix, projmatrix,
                               sh_degree, campos, prefiltered, debug, include_feature)
        self.antialiasing = bool(antialiasing)
        self.orthographic = bool(orthographic)
        self.fisheye = _fisheye_params(fisheye)
        if self.orthographic and self.fisheye is not None:
            raise ValueError("a view cannot be both orthographic and fisheye")
        self.distortion = _distortion_params(distortion)
        if self.distortion is not None and (self.orthographic or self.fisheye is not None):
            raise ValueError("a distorted view cannot also be orthographic or fisheye")
        self.planar_depth = bool(planar_depth)
        return self

    @classmethod
    def _make(cls, iterable):
        return cls(*iterable)

    def _replace(self, **kw):
        aa = kw.pop("antialiasing", self.antialiasing)
        orth = kw.pop("orthographic", self.orthographic)
        fe = kw.pop("fisheye", self.fisheye)
        dc = kw.pop("distortion", self.distortion)
        pd = kw.pop("planar_depth", self.planar_depth)
        return type(self)(*super()._replace(**kw), antialiasing=aa, orthographic=orth, fisheye=fe, distortion=dc, planar_depth=pd)

    def __repr__(self):
        return super().__repr__()[:-1] + (f", antialiasing={self.antialiasing}, orthographic={self.orthographic}, "
                                          f"fisheye={self.fisheye}, distortion={self.distortion}, "
                                          f"planar_depth={self.planar_depth})")


FISHEYE_KEYS = ("cx", "cy", "k1", "k2", "k3", "k4", "theta_max")


def _fisheye_params(x):
    """A view's fisheye parameters as a tuple of 7 floats (FISHEYE_KEYS order) from such a sequence or a dict, or None"""
    if x is None:
        return None
    vals = [x[k] for k in FISHEYE_KEYS] if isinstance(x, dict) else list(x)
    if len(vals) != len(FISHEYE_KEYS):
        raise ValueError(f"fisheye: expected {FISHEYE_KEYS}, got {x!r}")
    return tuple(float(v) for v in vals)


DISTORTION_KEYS = ("cx", "cy", "k1", "k2", "p1", "p2", "k3", "k4", "k5", "k6", "r_max")


def _distortion_params(x):
    """A view's distortion parameters as a tuple of 11 floats (DISTORTION_KEYS order) from such a sequence or a dict, or None"""
    if x is None:
        return None
    vals = [x[k] for k in DISTORTION_KEYS] if isinstance(x, dict) else list(x)
    if len(vals) != len(DISTORTION_KEYS):
        raise ValueError(f"distortion: expected {DISTORTION_KEYS}, got {x!r}")
    return tuple(float(v) for v in vals)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings, return_depth=False, return_alpha=False, return_median_depth=False, return_normal=False):
        """return_depth / return_alpha: forward() also returns the depth plane [H,W] and / or the alpha plane [H,W]
        (accumulated opacity 1 - final_T), in that order after radii.  return_median_depth: it then also returns the
        median-depth plane [H,W] (differentiable) and the median contributor's Gaussian id [H,W] int32 (-1 where nothing
        covers the pixel; include/mgs_rasterizer.h, mgs_view_median), behind the other planes.  return_normal: it then also
        returns, last, the surface-normal plane [3,H,W] (world space, camera facing, not normalised, differentiable;
        mgs_view_normal); needs scales and rotations."""
        super().__init__()
        self.raster_settings = raster_settings
        self.return_depth = return_depth
        self.return_alpha = return_alpha
        self.return_median_depth = return_median_depth
        self.return_normal = return_normal

    def markVisible(self, positions):
        # Mark visible points (based on frustum culling for camera) with a boolean
        with torch.no_grad():
            s = self.raster_settings
            return mark_visible_raw(positions, s.viewmatrix, s.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, language_feature_precomp=None,
                scales=None, rotations=None, cov3D_precomp=None, flow_means3D=None, flow_pose=None):
        """flow_means3D [P,3]: the cloud's next-frame means; the outputs then end with the flow plane [2,H,W] (include/mgs_rasterizer.h,
        flow plane), with flow_pose (the next frame's (viewmatrix, projmatrix), or None for the view's own camera)."""
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        empty = torch.Tensor([])
        shs = empty if shs is None else shs
        colors_precomp = empty if colors_precomp is None else colors_precomp
        language_feature_precomp = empty if language_feature_precomp is None else language_feature_precomp
        scales = empty if scales is None else scales
        rotations = empty if rotations is None else rotations
        cov3D_precomp = empty if cov3D_precomp is None else cov3D_precomp
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, language_feature_precomp, opacities, scales,
                                   rotations, cov3D_precomp, self.raster_settings, self.return_depth, self.return_alpha,
                                   self.return_median_depth, self.return_normal, flow_means3D, flow_pose)


# ----------------------------------------------------------------------------------------------------------------------
# Multi-view batches (SURVEY.md 8(f) row f1; no counterpart in the reference, which renders one view per call and
# blocks the host on every view's instance count, rasterizer_impl.cu:284).  All views share one Gaussian cloud.  One C
# call (mgs_forward_views / mgs_backward_views) enqueues every view on its own CUDA stream, forks from and joins back
# into the caller's current stream, and NEVER synchronises with the host: the per-view binning state is sized from the
# instance counts observed on earlier calls (plus slack), the real count stays on the device, and {count, overflow flag}
# come back asynchronously through pinned memory to be looked at on a LATER call.  A step built from these calls
# allocates through torch's caching allocator only and can be captured in a CUDA graph.
import warnings

_VIEW_STREAMS = {}
_CAPACITY = {}        # (device index, P, W, H, slot) -> instance capacity to use for the next call
_PENDING_STATUS = []  # [(key, pinned int32[2], cuda event, capacity used)] of forwards whose status has not been read yet
_SIZES = {}
_STATUS_RING = {"buf": None, "next": 0}   # pinned {count, overflow} slots, handed out round-robin (pin_memory() per call would
_STATUS_SLOTS = 4096                       # cost a cudaHostAlloc and a device synchronisation each time)


def _status_slots(n):
    """n consecutive pinned int32[2] slots.  A slot is reused after _STATUS_SLOTS later views: by then its forward finished."""
    if _STATUS_RING["buf"] is None:
        _STATUS_RING["buf"] = torch.zeros((_STATUS_SLOTS, 2), dtype=torch.int32).pin_memory()
    i = _STATUS_RING["next"]
    if i + n > _STATUS_SLOTS:
        i = 0
    _STATUS_RING["next"] = i + n
    return _STATUS_RING["buf"][i:i + n]


def _view_streams(device, n):
    if os.environ.get("MGS_ONE_STREAM"):  # measurement hook: every view on the caller's stream (no overlap between views)
        return [torch.cuda.current_stream(device)] * n
    key = (device.index if device.index is not None else torch.cuda.current_device())
    pool = _VIEW_STREAMS.setdefault(key, [])
    while len(pool) < n:
        pool.append(torch.cuda.Stream(device=device))
    return pool[:n]


def _round_capacity(n):
    """geometric buckets (<= 12.5 % slack) so that slowly varying counts keep hitting the same cached allocation"""
    n = max(int(n), 4096)
    q = 1 << max(10, n.bit_length() - 4)
    return (n + q - 1) // q * q


def _poll_status(block=False):
    """Fold the instance counts of finished forwards into the capacity table (never waits unless block=True)."""
    keep = []
    for key, st, ev, cap in _PENDING_STATUS:
        if block:
            ev.synchronize()
        if not ev.query():
            keep.append((key, st, ev, cap))
            continue
        R, over = int(st[0]), int(st[1])
        want = _round_capacity(R * 1.25 + 4096)
        if over:
            warnings.warn(f"manigaussian_b200: a view produced {R} tile instances but its binning state held {cap}; the farthest "
                          f"{R - cap} instances were dropped from that render (capacity raised for the next call)")
            want = _round_capacity(R * 1.5 + 4096)
        cur = _CAPACITY.get(key, 0)
        # grow at once; shrink only when the state is more than twice too large (stable sizes keep hitting the same cached
        # allocation, and a render with few instances must not starve the next one)
        if want > cur or want < cur // 2:
            _CAPACITY[key] = want
    _PENDING_STATUS[:] = keep


def reset_capacity_estimates():
    """Forget the instance-count history (tests; or after a drastic scene change to force re-calibration)."""
    _poll_status(block=True)
    _CAPACITY.clear()


class ViewOut(tuple):
    """Result of one view of rasterize_views_raw: (capacity, color, feature, radii, geomBuffer, binningBuffer, imgBuffer
    [, depth]) -- the layout of rasterize_gaussians_raw with the binning CAPACITY in place of the instance count, which is
    what the backward needs.  `.num_rendered()` waits for the forward and returns the true count; `.status` is the pinned
    {count, overflow} pair."""
    status = None
    event = None

    def num_rendered(self):
        self.event.synchronize()
        return int(self.status[0])

    def overflowed(self):
        self.event.synchronize()
        return bool(self.status[1])


def _state_sizes(L, P, W, H, normal=False):
    """(geometry state, image state, backward scratch) bytes; `normal`: with the normal plane's per-Gaussian arrays"""
    key = (P, W, H, bool(normal))
    s = _SIZES.get(key)
    if s is None:
        if normal:
            s = (int(L.mgs_geometry_state_bytes_normal(P)), int(L.mgs_image_state_bytes(W, H)),
                 int(L.mgs_backward_scratch_bytes_normal(P)))
        else:
            s = (int(L.mgs_geometry_state_bytes(P)), int(L.mgs_image_state_bytes(W, H)), int(L.mgs_backward_scratch_bytes(P)))
        _SIZES[key] = s
    return s


def _check_flow(flow_means3D, normal, planar, depth_mask):
    """The flow plane's call-wide argument errors (ValueError): it takes the normal plane's tile columns, and has no kernel
    beside the depth / mask heads."""
    if flow_means3D is None:
        return
    if normal:
        raise ValueError("flow cannot be combined with a normal plane (return_normal): both take the same tile columns")
    if planar:
        raise ValueError("flow cannot be combined with planar_depth: both take the same tile columns")
    if depth_mask is not None:
        raise ValueError("flow cannot be combined with the depth / mask heads")


def _planar_flag(views, planar_depth=None, normal=False):
    """The call's planar-depth flag: `planar_depth` when given, else the views' `planar_depth` attribute (every view of one
    call must agree).  Raises ValueError beside a normal plane (both take the same columns of the blend's channel tile)."""
    if planar_depth is None:
        flags = {bool(getattr(s, "planar_depth", False)) for s in views}
        if len(flags) > 1:
            raise ValueError("planar_depth is a per-call setting: every view of one call must have the same value")
        planar_depth = flags.pop() if flags else False
    planar_depth = bool(planar_depth)
    if planar_depth and normal:
        raise ValueError("planar_depth cannot be combined with a normal plane (return_normal) in the same call")
    return planar_depth


def _flow_array(views, flow_means3D, flow_poses, P, dev, keep, planes=None, grads=None):
    """ViewFlow array of the views' flow planes (C ABI mgs_view_flow), or None without `flow_means3D`.  flow_poses: None, or
    per view None (the view's own camera) or (viewmatrix, projmatrix) of its next frame.  planes / grads: the backward's
    forward planes and cotangents (per view [3,H,W] or [2,H,W]).  The tensors that must stay alive go to `keep`."""
    if flow_means3D is None:
        return None
    if tuple(flow_means3D.shape) != (P, 3) or flow_means3D.dtype != torch.float32 or flow_means3D.device != dev:
        raise ValueError(f"flow_means3D: expected [{P},3] fp32 on {dev}, got {tuple(flow_means3D.shape)} {flow_means3D.dtype} "
                         f"on {flow_means3D.device}")
    V = len(views)
    if flow_poses is not None and len(flow_poses) != V:
        raise ValueError(f"flow_poses: expected {V} entries, got {len(flow_poses)}")
    arr = (_b.ViewFlow * V)()
    for v in range(V):
        pose = flow_poses[v] if flow_poses is not None else None
        if pose is not None:
            vm, pm = (_prep(torch.as_tensor(x, dtype=torch.float32, device=dev).detach().reshape(4, 4), dev) for x in pose)
            arr[v].next_viewmatrix, arr[v].next_projmatrix = _ptr(vm), _ptr(pm)
            keep += [vm, pm]
        if planes is not None:
            arr[v].out_flow = _ptr(planes[v])
        if grads is not None and grads[v] is not None:
            g = grads[v]
            if g.shape[0] == 2:  # the plane's third channel carries no cotangent
                g = torch.cat([g, torch.zeros_like(g[:1])])
            g = _prep(g, dev)
            arr[v].dL_dpix_flow = _ptr(g)
            keep.append(g)
    return arr


def _ortho_flags(views, ortho=None):
    """Per-view camera models: `ortho` (V truthy values) when given, else each view's `orthographic` attribute; a ctypes int
    array for mgs_render_options.ortho, or None when every view is perspective."""
    flags = [bool(o) for o in ortho] if ortho is not None else [bool(getattr(s, "orthographic", False)) for s in views]
    if len(flags) != len(views):
        raise ValueError(f"ortho: expected {len(views)} flags, got {len(flags)}")
    return (ctypes.c_int * len(flags))(*flags) if any(flags) else None


def _fisheye_array(views, fisheye=None):
    """Per-view fisheye parameters: `fisheye` (V entries, each None or parameters) when given, else each view's `fisheye`
    attribute; a ctypes ViewFisheye array for mgs_render_options.fisheye, or None when no view is fisheye."""
    fe = [_fisheye_params(f) for f in fisheye] if fisheye is not None else [getattr(s, "fisheye", None) for s in views]
    if len(fe) != len(views):
        raise ValueError(f"fisheye: expected {len(views)} entries, got {len(fe)}")
    if all(f is None for f in fe):
        return None
    arr = (_b.ViewFisheye * len(fe))()
    for v, f in enumerate(fe):
        if f is not None:
            arr[v].fisheye = 1
            for k, x in zip(FISHEYE_KEYS, f):
                setattr(arr[v], k, x)
    return arr


def _distortion_array(views, distortion=None):
    """Per-view distortion parameters: `distortion` (V entries, each None or parameters) when given, else each view's
    `distortion` attribute; a ctypes ViewDistortion array for mgs_render_options.distortion, or None when no view is distorted."""
    dc = [_distortion_params(d) for d in distortion] if distortion is not None else \
        [getattr(s, "distortion", None) for s in views]
    if len(dc) != len(views):
        raise ValueError(f"distortion: expected {len(views)} entries, got {len(dc)}")
    if all(d is None for d in dc):
        return None
    arr = (_b.ViewDistortion * len(dc))()
    for v, d in enumerate(dc):
        if d is not None:
            arr[v].distorted = 1
            for k, x in zip(DISTORTION_KEYS, d):
                setattr(arr[v], k, x)
    return arr


def _lens_arrays(views, ortho=None, fisheye=None, distortion=None):
    """The views' camera models as the C ABI takes them: (_ortho_flags, _fisheye_array, _distortion_array)"""
    return _ortho_flags(views, ortho), _fisheye_array(views, fisheye), _distortion_array(views, distortion)


def _calibrate(L, views, keys, dev, P, degree, M, means3D, sh, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, debug,
               ortho=None, fisheye=None, distortion=None):
    """First call for a (cloud size, image size): one projection + scan per view with a host read of the instance count
    (the reference does this on EVERY call), only to seed the capacity table.  An orthographic view (`ortho`: the views'
    flags, or None) is counted by a weight-only lift with one binning slot, whose status holds the full count: the
    single-view mgs_forward_begin has no camera model, and the lift is the cheapest call that takes one.  Its weights are
    discarded.  A fisheye view (`fisheye`: the views' ViewFisheye array, or None) and a distorted view (`distortion`: the
    views' ViewDistortion array, or None) are counted the same way."""
    counts = torch.zeros(len(views), dtype=torch.int32).pin_memory()
    st = torch.cuda.current_stream(dev)
    keep, ortho_status = [], {}
    for v, s in enumerate(views):
        if keys[v] in _CAPACITY:
            continue
        fe = fisheye[v] if fisheye is not None and fisheye[v].fisheye else None
        dc = distortion[v] if distortion is not None and distortion[v].distorted else None
        if (ortho is not None and ortho[v]) or fe is not None or dc is not None:
            ortho_status[v], k = _count_ortho(L, s, dev, P, means3D, colors, opacity, scales, rotations, scale_modifier,
                                              cov3D_precomp, debug, st, fe, dc)
            keep.append(k)
            continue
        H, W = int(s.image_height), int(s.image_width)
        ga, ia = _Alloc(dev), _Alloc(dev)
        radii = torch.empty((P,), dtype=torch.int32, device=dev)
        vm, pm, cp = (_prep(x, dev) for x in (s.viewmatrix, s.projmatrix, s.campos))
        _checked((ga, ia), L.mgs_forward_begin(_ALLOC_CB, ga.key, _ALLOC_CB, ia.key, P, int(degree), M, W, H, _ptr(means3D), _ptr(sh), _ptr(colors),
                                     _ptr(opacity), _ptr(scales), float(scale_modifier), _ptr(rotations), _ptr(cov3D_precomp), _ptr(vm),
                                     _ptr(pm), _ptr(cp), float(s.tanfovx), float(s.tanfovy), _ptr(radii), counts.data_ptr() + 4 * v,
                                     int(bool(debug)), st.cuda_stream), "mgs_forward_begin")
        keep.append((ga.release(), ia.release(), radii, vm, pm, cp))
    st.synchronize()
    for v in range(len(views)):
        if keys[v] not in _CAPACITY:
            n = int(ortho_status[v][0]) if v in ortho_status else int(counts[v])
            _CAPACITY[keys[v]] = _round_capacity(n * 1.25 + 4096)


def _count_ortho(L, s, dev, P, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, debug, st, fisheye=None,
                 distortion=None):
    """Enqueues orthographic view `s`'s projection and binning on `st` with one binning slot, fisheye view `s`'s with
    `fisheye` its ViewFisheye entry, or distorted view `s`'s with `distortion` its ViewDistortion entry.  Returns its pinned status {instance count, overflow}, valid once `st` is synchronised,
    and what must stay alive until then."""
    H, W = int(s.image_height), int(s.image_width)
    gbytes, ibytes, _ = _state_sizes(L, P, W, H)
    geom = torch.empty(gbytes, dtype=torch.uint8, device=dev)
    img = torch.empty(ibytes, dtype=torch.uint8, device=dev)
    binb = torch.empty(int(L.mgs_binning_state_bytes(1)), dtype=torch.uint8, device=dev)
    radii = torch.empty((P,), dtype=torch.int32, device=dev)
    weight = torch.empty((P,), dtype=torch.float32, device=dev)
    status = torch.zeros((2,), dtype=torch.int32).pin_memory()
    vm, pm = _prep(s.viewmatrix, dev), _prep(s.projmatrix, dev)
    tf = _device_fov([s], None, dev)
    colors = colors if _nonempty(colors) else torch.zeros((P, 3), dtype=torch.float32, device=dev)
    w = (_b.View * 1)()
    w[0].viewmatrix, w[0].projmatrix = _ptr(vm), _ptr(pm)
    w[0].tan_fovx, w[0].tan_fovy, w[0].width, w[0].height = _host_tan(s.tanfovx), _host_tan(s.tanfovy), W, H
    w[0].geometry_state, w[0].binning_state, w[0].image_state, w[0].binning_capacity = geom.data_ptr(), binb.data_ptr(), img.data_ptr(), 1
    w[0].radii, w[0].status, w[0].stream = radii.data_ptr(), status.data_ptr(), st.cuda_stream
    iarr = _intrinsics_array(tf, None) if tf is not None else None
    rest = (P, 0, 0, 0, _ptr(means3D), None, _ptr(colors), _ptr(opacity), _ptr(scales), float(scale_modifier), _ptr(rotations),
            _ptr(cov3D_precomp), None, _ptr(weight), int(bool(debug)), st.cuda_stream)
    dcarr = (_b.ViewDistortion * 1)(distortion) if distortion is not None else None
    farr = (_b.ViewFisheye * 1)(fisheye) if fisheye is not None and dcarr is None else None
    oarr = (ctypes.c_int * 1)(1) if farr is None and dcarr is None else None
    _b.check(L.mgs_lift_views(1, w, None, 0, iarr, oarr, farr, dcarr, *rest), "mgs_lift_views")
    return status, (geom, img, binb, radii, weight, vm, pm, tf, colors)


def rasterize_views_raw(views, means3D, colors, language_feature, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                        sh, degree, include_feature, return_depth=False, debug=False, out_buffers=None, capacities=None,
                        loss_heads=None, return_alpha=False, depth_mask=None, antialiasing=False, ssim=None, tan_fov=None,
                        return_median=False, return_normal=False, ortho=None, fisheye=None, distortion=None, planar_depth=None,
                        flow_means3D=None, flow_poses=None):
    """Forward of V views of one Gaussian cloud.  `views` is a sequence of GaussianRasterizationSettings (bg, viewmatrix,
    projmatrix, tanfov*, image size, campos are read per view).  Returns (outs, streams): outs[v] is a ViewOut; all work
    is joined into the caller's current stream before the call returns (`streams` are the per-view streams used).
    `out_buffers` = (color [V,3,H,W], feature [V,F,H,W] or None, depth [V,H,W] or None[, alpha [V,H,W] or None]): render
    straight into slices of caller-owned batch tensors instead of per-view allocations.  `return_alpha` appends the alpha
    plane 1 - final_T [H,W] to every ViewOut (after depth, when that is asked for too).  `capacities` (per-view instance capacities) overrides
    the history-based sizing of the binning state.  `loss_heads` = (target_rgb [V,3,H,W], target_embed [V,F,H,W] or None,
    cot_rgb [V,3,H,W], cot_embed [V,F,H,W] or None, loss_acc [V,2]): the forward blend's epilogue also evaluates the L2 colour
    head and the cosine embedding head against the targets (C ABI mgs_view.target_*), leaving the loss sums in loss_acc and
    the cotangent planes ready for rasterize_views_backward_raw.  `depth_mask` = (target_depth [V,H,W] or None, target_mask
    [V,H,W] or None, cot_depth, cot_alpha_depth (both [V,H,W], with target_depth), cot_alpha_mask [V,H,W] (with target_mask),
    loss_acc [V,3]), with `loss_heads` only: the same epilogue also evaluates the expected-depth L1 head and the alpha mask
    head (C ABI mgs_view_depth_mask), leaving {sum |d - g|, valid pixels, sum BCE} in loss_acc.  `antialiasing`: the
    anti-aliased projection (C ABI mgs_render_options.antialiasing); pass the same value to the backward.  `ssim` = (ssim_terms
    [V,9,H,W], loss_acc [V,4], cot_color [V,3,H,W]), with `loss_heads` only: behind each view's blend, the L1 + SSIM head
    (C ABI mgs_view_ssim) leaves {sum |x - g|, sum S} in loss_acc[:, :2] and the partials of S in ssim_terms.  `tan_fov`
    [V,2] (device): every view's {tan_fovx, tan_fovy}, read by the kernels in place of the settings' host floats (C ABI
    mgs_render_options.intrinsics); views whose tanfovx / tanfovy are CUDA tensors use it without being asked.  Pass the same to
    the backward.  `return_median` appends the median-depth plane [H,W] and the median contributor's Gaussian id [H,W] int32
    (-1 where nothing covers the pixel) to every ViewOut, behind the other planes (C ABI mgs_view_median); with `out_buffers`
    they go to out_buffers[4] and out_buffers[5] ([V,H,W] each) when those are given.  `return_normal` appends, last, the
    surface-normal plane [3,H,W] to every ViewOut (C ABI mgs_view_normal; out_buffers[6] [V,3,H,W] when given); it needs scales
    and rotations, and cannot be combined with `depth_mask`.  `ortho` (V flags) marks the orthographic views; by default each
    view's `orthographic` attribute does.  They go to mgs_render_options.ortho; pass the same
    flags (or views) to the backward.  `fisheye` (V entries, each None or a view's fisheye parameters, as the settings'
    `fisheye` attribute) marks the fisheye views, by default each view's `fisheye` attribute; they go to
    mgs_render_options.fisheye.  `distortion` (V entries, each None or a view's distortion parameters, as the settings'
    `distortion` attribute) marks the distorted-pinhole views, by default each view's `distortion` attribute; they go to
    mgs_render_options.distortion.  `planar_depth` (default: the views' `planar_depth` attribute):
    each Gaussian's depth follows its tilt across its footprint, in the depth plane, the depth head and the median depth
    (C ABI mgs_render_options.planar_depth); it cannot be combined with `return_normal`.  `flow_means3D` [P,3] (the cloud's
    next-frame means, paired by index) appends, last, every view's flow plane [3,H,W] (channels: x and y screen displacement
    in pixels, blended with the colour's weights; channel 2 is 0; C ABI mgs_render_options.flow; out_buffers[7] [V,3,H,W]
    when given), with `flow_poses` (per view None or the next frame's (viewmatrix, projmatrix)) the pose each view projects
    the next means with.  Not with `return_normal`, `planar_depth` or `depth_mask`."""
    if not means3D.is_cuda:
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    if means3D.size(0) == 0:
        raise RuntimeError("rasterize_views_raw needs at least one Gaussian")
    cloud = dict(views=views, means3D=means3D, sh=sh, colors=colors, feature=language_feature, opacity=opacity, scales=scales,
                 rotations=rotations, cov3D_precomp=cov3D_precomp, out_buffers=out_buffers, capacities=capacities,
                 loss_heads=loss_heads, depth_mask=depth_mask, ssim=ssim, tan_fov=tan_fov, ortho=ortho, fisheye=fisheye,
                 distortion=distortion, flow_means3D=flow_means3D, flow_poses=flow_poses)
    outs, streams = rasterize_clouds_raw([cloud], degree, include_feature, scale_modifier, return_depth, debug, return_alpha,
                                         antialiasing, return_median, return_normal, planar_depth, views_call=True)
    return outs[0], streams


def lift_views_raw(views, means3D, opacity, scales, rotations, scale_modifier, cov3D_precomp, maps, antialiasing=False,
                   tan_fov=None, debug=False, ortho=None, fisheye=None, distortion=None):
    """Lift one 2D map per view onto the Gaussians (C ABI mgs_lift_views): lifted [P,C] = sum over the views and pixels of
    the forward blend's weights w = alpha T times the map, weight [P] = the sum of the weights.  `maps`: [V,C,H,W] or a
    sequence of V [C,H,W] fp32 tensors on the cloud's device (each view's own H, W), or None for weight only.  `views`,
    `antialiasing`, `tan_fov`, `ortho`, `fisheye` and `distortion` as in rasterize_views_raw; the binning state is sized
    from the same capacity table (a steady-state call reads nothing back to the host).  Returns (lifted, weight); neither is differentiable.  The projection
    needs colours, which the lift never reads: a zero [P,3] buffer stands in for them."""
    L = _b.lib()
    dev = means3D.device
    if not means3D.is_cuda:
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    P = means3D.size(0)
    if P == 0:
        raise RuntimeError("lift_views_raw needs at least one Gaussian")
    means3D, opacity, scales, rotations, cov3D_precomp = (_prep(x, dev) for x in (means3D, opacity, scales, rotations, cov3D_precomp))
    V = len(views)
    oarr, farr, dcarr = _lens_arrays(views, ortho, fisheye, distortion)
    C = int(maps[0].shape[0]) if maps is not None else 0
    colors = torch.zeros((P, 3), dtype=torch.float32, device=dev)
    main = torch.cuda.current_stream(dev)
    streams = _view_streams(dev, V) if V > 1 else [main]
    di = dev.index if dev.index is not None else torch.cuda.current_device()
    keys = [(di, P, int(s.image_width), int(s.image_height), v) for v, s in enumerate(views)]
    capturing = torch.cuda.is_current_stream_capturing()
    with torch.cuda.device(dev):
        if not capturing:
            _poll_status()
        if any(k not in _CAPACITY for k in keys):
            if capturing:
                raise RuntimeError("lift the views once before capturing them in a CUDA graph (the binning capacity is learned "
                                   "from an eager call)")
            _calibrate(L, views, keys, dev, P, 0, 0, means3D, None, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                       debug, oarr, farr, dcarr)
        arr = (_b.View * V)()
        larr = (_b.ViewLift * V)()
        status = _status_slots(V)
        keep, outs = [colors], []
        for v, s in enumerate(views):
            H, W = int(s.image_height), int(s.image_width)
            gbytes, ibytes, _ = _state_sizes(L, P, W, H)
            cap = _CAPACITY[keys[v]]
            geom = torch.empty(gbytes, dtype=torch.uint8, device=dev)
            img = torch.empty(ibytes, dtype=torch.uint8, device=dev)
            binb = torch.empty(int(L.mgs_binning_state_bytes(cap)), dtype=torch.uint8, device=dev)
            radii = torch.empty((P,), dtype=torch.int32, device=dev)
            vm, pm = _prep(s.viewmatrix, dev), _prep(s.projmatrix, dev)
            w = arr[v]
            w.viewmatrix, w.projmatrix = _ptr(vm), _ptr(pm)
            w.tan_fovx, w.tan_fovy, w.width, w.height = _host_tan(s.tanfovx), _host_tan(s.tanfovy), W, H
            w.geometry_state, w.binning_state, w.image_state, w.binning_capacity = geom.data_ptr(), binb.data_ptr(), img.data_ptr(), cap
            w.radii = radii.data_ptr()
            w.status = status.data_ptr() + 8 * v
            w.stream = streams[v].cuda_stream
            if C:
                m = _prep(maps[v], dev)
                larr[v].map = m.data_ptr()
                keep.append(m)
            keep += [geom, img, binb, radii, vm, pm]
            outs.append(ViewOut((cap,)))
        lifted = torch.empty((P, C), dtype=torch.float32, device=dev)
        weight = torch.empty((P,), dtype=torch.float32, device=dev)
        tf = _device_fov(views, tan_fov, dev)
        keep.append(tf)
        iarr = _intrinsics_array(tf, None) if tf is not None else None
        rest = (P, 0, 0, C, _ptr(means3D), None, _ptr(colors), _ptr(opacity), _ptr(scales), float(scale_modifier), _ptr(rotations),
                _ptr(cov3D_precomp), _ptr(lifted) if C else None, _ptr(weight), int(bool(debug)), main.cuda_stream)
        _b.check(L.mgs_lift_views(V, arr, larr, int(bool(antialiasing)), iarr, oarr, farr, dcarr, *rest), "mgs_lift_views")
        _track_status(outs, keys, status, main, not capturing)
    return lifted, weight


def visibility_views_raw(views, means3D, opacity, scales, rotations, scale_modifier, cov3D_precomp, points, antialiasing=False,
                         tan_fov=None, debug=False, ortho=None, fisheye=None, distortion=None, keep_state=False):
    """Project Q points into every view with occlusion (C ABI mgs_visibility_views): per view and point the screen position
    uv [V,Q,2] (pixel centres at integers), the view-space depth [V,Q], in_view [V,Q] (uint8) and the transmittance [V,Q] the
    cloud leaves in front of the point, with the blend's own tile lists, depth order, thresholds and early stop.  `points`
    [Q,3] fp32 on the cloud's device.  `views`, `antialiasing`, `tan_fov`, `ortho`, `fisheye` and `distortion` as in
    lift_views_raw; the binning state is sized from the same capacity table, so a steady-state call reads nothing back to the
    host and can be captured in a CUDA graph.  Returns (uv, depth, in_view, T); none is differentiable.  `keep_state`: also
    return, fifth, what visibility_views_backward_raw needs (the views' state buffers, point scratch and streams; None for
    Q = 0)."""
    L = _b.lib()
    dev = means3D.device
    if not means3D.is_cuda:
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    P = means3D.size(0)
    if P == 0:
        raise RuntimeError("visibility_views_raw needs at least one Gaussian")
    means3D, opacity, scales, rotations, cov3D_precomp, points = (
        _prep(x, dev) for x in (means3D, opacity, scales, rotations, cov3D_precomp, points))
    V, Q = len(views), int(points.shape[0])
    oarr, farr, dcarr = _lens_arrays(views, ortho, fisheye, distortion)
    colors = torch.zeros((P, 3), dtype=torch.float32, device=dev)
    main = torch.cuda.current_stream(dev)
    streams = _view_streams(dev, V) if V > 1 else [main]
    di = dev.index if dev.index is not None else torch.cuda.current_device()
    keys = [(di, P, int(s.image_width), int(s.image_height), v) for v, s in enumerate(views)]
    capturing = torch.cuda.is_current_stream_capturing()
    uv = torch.empty((V, Q, 2), dtype=torch.float32, device=dev)
    depth = torch.empty((V, Q), dtype=torch.float32, device=dev)
    in_view = torch.empty((V, Q), dtype=torch.uint8, device=dev)
    T = torch.empty((V, Q), dtype=torch.float32, device=dev)
    if Q == 0:
        return (uv, depth, in_view, T) + ((None,) if keep_state else ())
    with torch.cuda.device(dev):
        if not capturing:
            _poll_status()
        if any(k not in _CAPACITY for k in keys):
            if capturing:
                raise RuntimeError("query the views once before capturing them in a CUDA graph (the binning capacity is learned "
                                   "from an eager call)")
            _calibrate(L, views, keys, dev, P, 0, 0, means3D, None, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                       debug, oarr, farr, dcarr)
        arr = (_b.View * V)()
        status = _status_slots(V)
        keep, outs = [colors], []
        for v, s in enumerate(views):
            H, W = int(s.image_height), int(s.image_width)
            gbytes, ibytes, _ = _state_sizes(L, P, W, H)
            cap = _CAPACITY[keys[v]]
            geom = torch.empty(gbytes, dtype=torch.uint8, device=dev)
            img = torch.empty(ibytes, dtype=torch.uint8, device=dev)
            binb = torch.empty(int(L.mgs_binning_state_bytes(cap)), dtype=torch.uint8, device=dev)
            scratch = torch.empty(int(L.mgs_visibility_scratch_bytes(Q, W, H)), dtype=torch.uint8, device=dev)
            radii = torch.empty((P,), dtype=torch.int32, device=dev)
            vm, pm = _prep(s.viewmatrix, dev), _prep(s.projmatrix, dev)
            w = arr[v]
            w.viewmatrix, w.projmatrix = _ptr(vm), _ptr(pm)
            w.tan_fovx, w.tan_fovy, w.width, w.height = _host_tan(s.tanfovx), _host_tan(s.tanfovy), W, H
            w.geometry_state, w.binning_state, w.image_state, w.binning_capacity = geom.data_ptr(), binb.data_ptr(), img.data_ptr(), cap
            w.blend_scratch = scratch.data_ptr()
            w.radii = radii.data_ptr()
            w.status = status.data_ptr() + 8 * v
            w.stream = streams[v].cuda_stream
            keep += [geom, img, binb, scratch, radii, vm, pm]
            outs.append(ViewOut((cap,)))
        tf = _device_fov(views, tan_fov, dev)
        keep.append(tf)
        iarr = _intrinsics_array(tf, None) if tf is not None else None
        _b.check(L.mgs_visibility_views(V, arr, int(bool(antialiasing)), iarr, oarr, farr, dcarr, P, 0, 0, Q, _ptr(points),
                                        _ptr(means3D), None, _ptr(colors), _ptr(opacity), _ptr(scales), float(scale_modifier),
                                        _ptr(rotations), _ptr(cov3D_precomp), _ptr(uv), _ptr(depth), _ptr(in_view), _ptr(T),
                                        int(bool(debug)), main.cuda_stream), "mgs_visibility_views")
        _track_status(outs, keys, status, main, not capturing)
    if not keep_state:
        return uv, depth, in_view, T
    state = dict(arr=arr, keep=keep, tf=tf, lens=(oarr, farr, dcarr), P=P, Q=Q, aa=bool(antialiasing), debug=bool(debug),
                 colors=colors, streams=streams)
    return uv, depth, in_view, T, state


def visibility_views_backward_raw(state, points, means3D, opacity, scales, rotations, scale_modifier, cov3D_precomp, T, grad_T,
                                  grad_uv, grad_depth, want_points=True, want_cloud=True, camera_grads=False,
                                  return_scratch=False):
    """Backward of visibility_views_raw (C ABI mgs_visibility_views_backward).  `state`: the fifth result of that call with
    keep_state=True; points, the cloud and `T` (its transmittance) as given to and returned by it.  grad_T [V,Q], grad_uv
    [V,Q,2] and grad_depth [V,Q]: the cotangents, each None for none.  Returns (dL_dpoints [Q,3], dL_dmeans3D [P,3],
    dL_dopacity [P,1], dL_dscales [P,3], dL_drotations [P,4], camera), each gradient None where not wanted: `want_points`, and
    `want_cloud`, a bool or four in that order (scales and rotations are None without scales too).  camera is None, or with
    camera_grads=True (dL_dviewmatrix [V,16], dL_dprojmatrix [V,16], dL_dcampos [V,3], dL_dtan_fov [V,2], None without a
    device field of view).  Nothing is read back to the host.  `return_scratch`: also return, seventh, the per-view backward
    scratch [V, bytes] the call wrote (its "visibility_backward" arrays of state_array)."""
    L = _b.lib()
    dev = means3D.device
    P, Q = state["P"], state["Q"]
    arr = state["arr"]
    V = len(arr)
    means3D, opacity, scales, rotations, cov3D_precomp, points, T = (
        _prep(x, dev) for x in (means3D, opacity, scales, rotations, cov3D_precomp, points, T))
    grad_T, grad_uv, grad_depth = (_prep(x, dev) if x is not None else None for x in (grad_T, grad_uv, grad_depth))
    opts = dict(dtype=torch.float32, device=dev)
    main = torch.cuda.current_stream(dev)
    dpts = torch.empty((Q, 3), **opts) if want_points else None
    has_sr = scales is not None and scales.numel() != 0
    want = tuple(want_cloud) if isinstance(want_cloud, (tuple, list)) else (bool(want_cloud),) * 4
    cloud = tuple(torch.empty(shape, **opts) if (w and (has_sr or i < 2)) else None
                  for i, (w, shape) in enumerate(zip(want, ((P, 3), (P, 1), (P, 3), (P, 4)))))
    tf = state["tf"]
    cam, carr = None, None
    if camera_grads:
        cam = (torch.empty((V, 16), **opts), torch.empty((V, 16), **opts), torch.empty((V, 3), **opts),
               torch.empty((V, 2), **opts) if tf is not None else None)
        carr = (_b.ViewCameraGrad * V)()
        for v in range(V):
            carr[v].dL_dviewmatrix = cam[0].data_ptr() + 64 * v
            carr[v].dL_dprojmatrix = cam[1].data_ptr() + 64 * v
            carr[v].dL_dcampos = cam[2].data_ptr() + 12 * v
    iarr = _intrinsics_array(tf, cam[3] if cam is not None else None) if tf is not None else None
    scratch = torch.empty((V, int(L.mgs_visibility_backward_scratch_bytes(P, Q))), dtype=torch.uint8, device=dev)
    for v in range(V):
        arr[v].dL_dmean2D = scratch[v].data_ptr()
    oarr, farr, dcarr = state["lens"]
    with torch.cuda.device(dev):
        _b.check(L.mgs_visibility_views_backward(
            V, arr, int(state["aa"]), iarr, oarr, farr, dcarr, P, 0, 0, Q, _ptr(points), _ptr(means3D), None, _ptr(state["colors"]),
            _ptr(opacity), _ptr(scales), float(scale_modifier), _ptr(rotations), _ptr(cov3D_precomp), _ptr(T), _ptr(grad_T),
            _ptr(grad_uv), _ptr(grad_depth), _ptr(dpts), _ptr(cloud[0]), _ptr(cloud[1]), _ptr(cloud[2]), _ptr(cloud[3]), None,
            carr, int(state["debug"]), main.cuda_stream), "mgs_visibility_views_backward")
    return (dpts,) + tuple(cloud) + (cam,) + ((scratch,) if return_scratch else ())


def _ray_call(views, pixels, tan_fov, ortho, fisheye, distortion):
    """(device, Q, pixels or None, mgs_view array, intrinsics array or None, lens arrays, tensors to keep alive) of a camera_rays
    call: every view's viewmatrix, projmatrix, field of view and size"""
    dev = pixels.device if pixels is not None else torch.as_tensor(views[0].viewmatrix).device
    if not dev.type == "cuda":
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    V = len(views)
    Q = int(pixels.shape[1]) if pixels is not None else int(views[0].image_width) * int(views[0].image_height)
    pixels = _prep(pixels, dev) if pixels is not None else None
    arr = (_b.View * V)()
    keep = [pixels]
    for v, s in enumerate(views):
        vm, pm = _prep(s.viewmatrix, dev), _prep(s.projmatrix, dev)
        w = arr[v]
        w.viewmatrix, w.projmatrix = _ptr(vm), _ptr(pm)
        w.tan_fovx, w.tan_fovy = _host_tan(s.tanfovx), _host_tan(s.tanfovy)
        w.width, w.height = int(s.image_width), int(s.image_height)
        keep += [vm, pm]
    tf = _device_fov(views, tan_fov, dev)
    keep.append(tf)
    return dev, Q, pixels, arr, tf, _lens_arrays(views, ortho, fisheye, distortion), keep


def camera_rays_raw(views, pixels=None, tan_fov=None, ortho=None, fisheye=None, distortion=None, debug=False):
    """The ray of each pixel of every view (C ABI mgs_camera_rays): the world points p(z) = origin + z direction whose screen
    position under the view's camera model is the pixel, z their view-space depth (direction's view-space z is 1).  pixels
    [V,Q,2] fp32 on the views' device (pixel centres at integers), or None for every pixel centre of the views' shared
    W x H grid, ray i at (i % W, i // W).  `views`, `tan_fov`, `ortho`, `fisheye` and `distortion` as in
    visibility_views_raw.  Returns (origin [V,N,3], direction [V,N,3], valid [V,N] uint8), origin and direction NaN where
    invalid; not differentiable (camera_rays_backward_raw is the backward).  Nothing is read back to the host."""
    L = _b.lib()
    dev, Q, pixels, arr, tf, (oarr, farr, dcarr), keep = _ray_call(views, pixels, tan_fov, ortho, fisheye, distortion)
    V = len(views)
    origin = torch.empty((V, Q, 3), dtype=torch.float32, device=dev)
    direction = torch.empty((V, Q, 3), dtype=torch.float32, device=dev)
    valid = torch.empty((V, Q), dtype=torch.uint8, device=dev)
    iarr = _intrinsics_array(tf, None) if tf is not None else None
    with torch.cuda.device(dev):
        _b.check(L.mgs_camera_rays(V, arr, iarr, oarr, farr, dcarr, Q, _ptr(pixels), _ptr(origin), _ptr(direction), _ptr(valid),
                                   int(bool(debug)), torch.cuda.current_stream(dev).cuda_stream), "mgs_camera_rays")
    return origin, direction, valid


def camera_rays_backward_raw(views, pixels, grad_origin, grad_direction, tan_fov=None, ortho=None, fisheye=None, distortion=None,
                             want_pixels=True, camera_grads=False, debug=False):
    """Backward of camera_rays_raw (C ABI mgs_camera_rays_backward) with the same views, pixels and camera models.
    grad_origin / grad_direction [V,N,3]: the cotangents, each None for zero.  Returns (dL_dpixels [V,Q,2] or None (with
    want_pixels and pixels), camera): camera is None, or with camera_grads=True (dL_dviewmatrix [V,16], dL_dprojmatrix [V,16],
    dL_dcampos [V,3] (zeros), dL_dtan_fov [V,2], None without a device field of view).  Deterministic; nothing is read back
    to the host."""
    L = _b.lib()
    dev, Q, pixels, arr, tf, (oarr, farr, dcarr), keep = _ray_call(views, pixels, tan_fov, ortho, fisheye, distortion)
    V = len(views)
    opts = dict(dtype=torch.float32, device=dev)
    go, gd = (_prep(g, dev) if g is not None else None for g in (grad_origin, grad_direction))
    dpix = torch.empty((V, Q, 2), **opts) if (want_pixels and pixels is not None) else None
    cam, carr = None, None
    if camera_grads:
        cam = (torch.empty((V, 16), **opts), torch.empty((V, 16), **opts), torch.empty((V, 3), **opts),
               torch.empty((V, 2), **opts) if tf is not None else None)
        rows = int(L.mgs_camera_rays_scratch_bytes(Q))
        scratch = torch.empty((V, max(rows, 4) // 4), **opts)
        carr = (_b.ViewCameraGrad * V)()
        for v in range(V):
            carr[v].dL_dviewmatrix = cam[0].data_ptr() + 64 * v
            carr[v].dL_dprojmatrix = cam[1].data_ptr() + 64 * v
            carr[v].dL_dcampos = cam[2].data_ptr() + 12 * v
            carr[v].scratch = scratch[v].data_ptr()
        keep.append(scratch)
        if Q == 0:  # the call enqueues nothing: the gradients of no rays are zero
            for t in cam:
                if t is not None:
                    t.zero_()
    iarr = _intrinsics_array(tf, cam[3] if cam is not None else None) if tf is not None else None
    with torch.cuda.device(dev):
        _b.check(L.mgs_camera_rays_backward(V, arr, iarr, oarr, farr, dcarr, Q, _ptr(pixels), _ptr(go), _ptr(gd), _ptr(dpix), carr,
                                            int(bool(debug)), torch.cuda.current_stream(dev).cuda_stream), "mgs_camera_rays_backward")
    return dpix, cam


def _fill_depth_mask(wd, depth_mask, v, scale=None):
    """Fills view v's mgs_view_depth_mask `wd` from a `depth_mask` tuple of rasterize_views_raw (and, for the backward, the
    upstream gradients `scale` [V,2])."""
    t_depth, t_mask, c_depth, c_alpha_depth, c_alpha_mask, acc = depth_mask
    if t_depth is not None:
        wd.target_depth, wd.cot_depth, wd.cot_alpha_depth = _ptr(t_depth[v]), _ptr(c_depth[v]), _ptr(c_alpha_depth[v])
    if t_mask is not None:
        wd.target_mask, wd.cot_alpha_mask = _ptr(t_mask[v]), _ptr(c_alpha_mask[v])
    wd.loss_acc = _ptr(acc[v])
    if scale is not None:
        wd.cot_scale = scale.data_ptr() + 8 * v


def _fill_ssim(ws, ssim, v, w=None, scale=None):
    """Fills view v's mgs_view_ssim `ws` from an `ssim` tuple of rasterize_views_raw.  Backward: the tuple also holds the
    forward's images and targets [V,3,H,W], which go into the view's mgs_view `w`, and `scale` [V,2] holds the upstream
    gradients {g_l1, g_ssim}."""
    ws.ssim_terms, ws.loss_acc, ws.cot_color = _ptr(ssim[0][v]), _ptr(ssim[1][v]), _ptr(ssim[2][v])
    if w is not None:
        w.out_color, w.target_color = _ptr(ssim[3][v]), _ptr(ssim[4][v])
    if scale is not None:
        ws.cot_scale = scale.data_ptr() + 8 * v


def _forward_view(L, w, s, v, dev, P, F, cap, include_feature, return_depth, out_buffers, loss_heads, wa=None, wm=None, wn=None,
                  quads=False, wf=None):
    """Allocates view v's state buffers and outputs and fills its mgs_view `w` (the caller sets status and stream) and, when
    `wa` (its mgs_view_alpha) is given, its alpha plane, when `wm` (its mgs_view_median) is given, its median planes, and when
    `wn` (its mgs_view_normal) is given, its normal plane.  `quads`: the geometry state also holds per-Gaussian quads (the
    planar-depth call), as with `wn`.  When `wf` (its mgs_view_flow) is given, its flow plane [3,H,W], last.
    Returns the ViewOut and the tensors that must stay alive until the call is enqueued."""
    H, W = int(s.image_height), int(s.image_width)
    gbytes, ibytes, _ = _state_sizes(L, P, W, H, wn is not None or quads or wf is not None)
    geom = torch.empty(gbytes, dtype=torch.uint8, device=dev)
    img = torch.empty(ibytes, dtype=torch.uint8, device=dev)
    binb = torch.empty(int(L.mgs_binning_state_bytes(cap)), dtype=torch.uint8, device=dev)
    radii = torch.empty((P,), dtype=torch.int32, device=dev)
    bg, vm, pm, cp = (_prep(x, dev) for x in (s.bg, s.viewmatrix, s.projmatrix, s.campos))
    if out_buffers is not None:
        out_color = out_buffers[0][v]
        out_feature = out_buffers[1][v] if (include_feature and F) else torch.zeros((1,), dtype=torch.float32, device=dev)
        out_depth = out_buffers[2][v] if return_depth else None
    else:
        out_color = torch.empty((3, H, W), dtype=torch.float32, device=dev)
        out_feature = torch.empty((F, H, W), dtype=torch.float32, device=dev) if include_feature else \
            torch.zeros((1,), dtype=torch.float32, device=dev)
        out_depth = torch.empty((H, W), dtype=torch.float32, device=dev) if return_depth else None
    out_alpha = None
    if wa is not None:
        ob = out_buffers[3] if (out_buffers is not None and len(out_buffers) > 3) else None
        out_alpha = ob[v] if ob is not None else torch.empty((H, W), dtype=torch.float32, device=dev)
        wa.out_alpha = _ptr(out_alpha)
    w.viewmatrix, w.projmatrix, w.cam_pos, w.background = _ptr(vm), _ptr(pm), _ptr(cp), _ptr(bg)
    w.tan_fovx, w.tan_fovy, w.width, w.height = _host_tan(s.tanfovx), _host_tan(s.tanfovy), W, H
    w.geometry_state, w.binning_state, w.image_state, w.binning_capacity = geom.data_ptr(), binb.data_ptr(), img.data_ptr(), cap
    w.out_color, w.out_feature, w.out_depth, w.radii = _ptr(out_color), (_ptr(out_feature) if F else None), _ptr(out_depth), _ptr(radii)
    if loss_heads is not None:
        t_rgb, t_emb, c_rgb, c_emb, l_acc = loss_heads
        w.target_color, w.cot_color, w.loss_acc = _ptr(t_rgb[v]), _ptr(c_rgb[v]), _ptr(l_acc[v])
        if t_emb is not None and F:
            w.target_feature, w.cot_feature = _ptr(t_emb[v]), _ptr(c_emb[v])
    ret = (cap, out_color, out_feature, radii, geom, binb, img) + ((out_depth,) if return_depth else ())
    ret += (out_alpha,) if wa is not None else ()
    if wm is not None:
        ob = out_buffers if (out_buffers is not None and len(out_buffers) > 5) else (None,) * 6
        med_depth = ob[4][v] if ob[4] is not None else torch.empty((H, W), dtype=torch.float32, device=dev)
        med_id = ob[5][v] if ob[5] is not None else torch.empty((H, W), dtype=torch.int32, device=dev)
        wm.out_median_depth, wm.median_id = _ptr(med_depth), _ptr(med_id)
        ret += (med_depth, med_id)
    if wn is not None:
        ob = out_buffers[6] if (out_buffers is not None and len(out_buffers) > 6) else None
        normal = ob[v] if ob is not None else torch.empty((3, H, W), dtype=torch.float32, device=dev)
        wn.out_normal = _ptr(normal)
        ret += (normal,)
    if wf is not None:
        ob = out_buffers[7] if (out_buffers is not None and len(out_buffers) > 7) else None
        flow = ob[v] if ob is not None else torch.empty((3, H, W), dtype=torch.float32, device=dev)
        wf.out_flow = _ptr(flow)
        ret += (flow,)
    return ViewOut(ret), (bg, vm, pm, cp)


def _host_tan(x):
    """mgs_view.tan_fov* of a view: its host float, or 0 for a CUDA tensor (the call then reads the device value through
    mgs_view_intrinsics; no device->host read)"""
    return 0.0 if (torch.is_tensor(x) and x.is_cuda) else float(x)


def _device_fov(views, tan_fov, dev):
    """The views' device field of view {tan_fovx, tan_fovy} [V,2] (fp32, contiguous, detached): `tan_fov` when given, else
    stacked from views whose tanfovx / tanfovy are CUDA tensors; None when neither (the host floats serve)."""
    if tan_fov is None:
        if not any(torch.is_tensor(t) and t.is_cuda for s in views for t in (s.tanfovx, s.tanfovy)):
            return None
        return _fov_column(views, dev)
    tan_fov = tan_fov.detach()
    if tuple(tan_fov.shape) != (len(views), 2):
        raise ValueError(f"tan_fov: expected [{len(views)},2], got {tuple(tan_fov.shape)}")
    return _prep(tan_fov, dev)


def _fov_column(views, dev):
    """[V,2] fp32 device tensor of the views' {tanfovx, tanfovy}: device values are copied on the device, host floats are
    written by fill kernels -- no host->device copy from pageable memory, so it can be captured in a CUDA graph."""
    out = torch.empty((len(views), 2), dtype=torch.float32, device=dev)
    with torch.no_grad():
        for v, s in enumerate(views):
            for i, t in enumerate((s.tanfovx, s.tanfovy)):
                if torch.is_tensor(t) and t.is_cuda:
                    out[v, i].copy_(t.reshape(()))
                else:
                    out[v, i].fill_(float(t))
    return out


def _intrinsics_array(tf, dtf):
    """ViewIntrinsics array of the views' device field of view tf [V,2] and its gradient output dtf [V,2] (or None)."""
    V = tf.shape[0]
    iarr = (_b.ViewIntrinsics * V)()
    for v in range(V):
        iarr[v].tan_fov = tf.data_ptr() + 8 * v
        iarr[v].dL_dtan_fov = dtf.data_ptr() + 8 * v if dtf is not None else None
    return iarr


def _track_status(outs, keys, status, main, pending):
    """Hands each ViewOut its pinned status pair and, when `pending`, queues the pair for the capacity table."""
    ev = torch.cuda.Event()
    ev.record(main)
    for v, o in enumerate(outs):
        o.status, o.event = status[v], ev
        if pending:
            _PENDING_STATUS.append((keys[v], status[v], ev, o[0]))


def rasterize_views_backward_raw(views, outs, streams, grads_color, grads_feature, means3D, colors, language_feature, scales,
                                 rotations, scale_modifier, cov3D_precomp, sh, degree, include_feature, grads_depth=None,
                                 debug=False, accumulate_into=None, means2D_per_view=None, accumulate=False, after_blend=None,
                                 cot_scale=None, grads_alpha=None, depth_mask=None, depth_mask_scale=None, antialiasing=False,
                                 ssim=None, ssim_scale=None, camera_grads=None, tan_fov=None, grads_median=None, median_ids=None,
                                 grads_normal=None, normals=None, ortho=None, fisheye=None, distortion=None, planar_depth=None,
                                 flow_means3D=None, flow_poses=None, grads_flow=None, flows=None):
    """Backward of the V views rendered by rasterize_views_raw: every view's blend backward on its stream, then ONE
    per-Gaussian chain-rule kernel that sums over the views (mgs_backward_views).  Returns the 9-tuple of
    rasterize_gaussians_backward_raw holding the SUMS over the views (dL_dmeans2D: `means2D_per_view` [V,P,3] when given,
    else the sum).  `accumulate_into`: dict of preallocated fp32 tensors keyed like manigaussian_b200.parallel.FIELDS that
    receive the sums (e.g. the views of a PackedGradients buffer -- the all-reduce message); rows are overwritten unless
    accumulate=True.  `after_blend()` is called between the blend stage and the per-Gaussian stage, when dL_dfeature is final
    (multi-GPU: start its all-reduce there; it overlaps the per-Gaussian kernel).  `cot_scale` [V,2] (device): upstream
    gradients of the fused loss heads' two scalars per view, multiplied onto the colour / feature cotangent planes as they
    are loaded.  `grads_alpha` (per view [H,W] or None): cotangents of the alpha planes of a `return_alpha` forward.  The
    caller's current stream holds the result on return.  `depth_mask`: the tuple given to the forward, whose cotangent planes
    are read back with `depth_mask_scale` [V,2] (device; the upstream gradients {g_depth, g_mask} of the depth and mask losses,
    or None for 1).  `antialiasing`: the value the forward was given (C ABI mgs_render_options.antialiasing).  `ssim`: the tuple given to
    the forward plus the forward's images and colour targets (both [V,3,H,W]); each view's L1 + SSIM head then writes its
    complete colour cotangent, with `ssim_scale` [V,2] (device; the upstream gradients {g_l1, g_ssim}, or None for 1), before
    its blend backward reads it.  `camera_grads`: True, or a tuple (dL_dviewmatrix [V,16], dL_dprojmatrix [V,16], dL_dcampos
    [V,3]) of fp32 device tensors or None each, asks for the gradients with respect to each view's viewmatrix, projmatrix and
    campos (C ABI mgs_render_options.camera_grad; written, or added to with accumulate=True); the return value then gains that tuple
    (allocated for True) as a 10th element.  `tan_fov`: as given to the forward (views with CUDA-tensor tanfov* imply it);
    it goes to mgs_render_options.intrinsics, and `camera_grads` gains a 4th entry, dL_dtan_fov [V,2] (the gradient with
    respect to each view's {tan_fovx, tan_fovy}; allocated for True, or named in a 4-tuple).  `grads_median` (per view [H,W]
    or None): cotangents of the median-depth planes of a `return_median` forward, with `median_ids` (per view [H,W] int32)
    the id planes that forward returned (C ABI mgs_view_median).  `grads_normal` (per view [3,H,W] or None):
    cotangents of the normal planes of a `return_normal` forward, with `normals` (per view [3,H,W]) the planes that forward
    returned (C ABI mgs_view_normal); their rotation gradient is added to dL_drotations.  `ortho`: as given to the
    forward (by default the views' `orthographic` attributes); C ABI mgs_render_options.ortho.
    `fisheye`: as given to the forward (by default the views' `fisheye` attributes); C ABI
    mgs_render_options.fisheye.  `distortion`: likewise, mgs_render_options.distortion.  `planar_depth`:
    as given to the forward (mgs_render_options.planar_depth).  `flow_means3D` and `flow_poses`: as given to the forward, with
    `flows` (per view [3,H,W]) the flow planes it returned and `grads_flow` (per view [3,H,W] or [2,H,W], or None) their
    cotangents (C ABI mgs_render_options.flow and flow_next); the return value then gains, last, dL_dflow_means3D [P,3]."""
    if flow_means3D is not None and flows is None:
        raise ValueError("flow cotangents need the forward's flow planes (flows)")
    cloud = dict(views=views, means3D=means3D, sh=sh, colors=colors, feature=language_feature, scales=scales, rotations=rotations,
                 cov3D_precomp=cov3D_precomp, grad_color=grads_color, grad_feature=grads_feature, grad_depth=grads_depth,
                 grad_alpha=grads_alpha, cot_scale=cot_scale, depth_mask=depth_mask, depth_mask_scale=depth_mask_scale, ssim=ssim,
                 ssim_scale=ssim_scale, tan_fov=tan_fov, grad_median=grads_median, median_id=median_ids, grad_normal=grads_normal,
                 normal=normals, ortho=ortho, fisheye=fisheye, distortion=distortion, flow_means3D=flow_means3D,
                 flow_poses=flow_poses, flow=flows, grad_flow=grads_flow, accumulate_into=accumulate_into,
                 means2D_per_view=means2D_per_view, shared_mean2D=means2D_per_view is None)
    r = rasterize_clouds_backward_raw([cloud], [outs], streams, degree, include_feature, scale_modifier, debug, antialiasing,
                                      camera_grads, planar_depth, accumulate=accumulate, after_blend=after_blend, views_call=True)[0]
    grads = tuple(r[k] for k in ("dL_dmeans2D", "dL_dcolors", "dL_dfeature", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh",
                                 "dL_dscales", "dL_drotations"))
    if camera_grads is not None and camera_grads is not False:
        grads += (tuple(r[k] for k in _CAMERA_GRADS if k in r),)
    return grads + (r["dL_dflow_means3D"],) if flow_means3D is not None else grads


_CAMERA_GRADS = ("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos", "dL_dtan_fov")


def _median_array(grads, ids, V, dev, keep):
    """ViewMedian array of V views' median-depth cotangents and id planes (per view [H,W] each, or None), or None without
    cotangents.  The tensors that must stay alive until the call is enqueued go to `keep`."""
    if grads is None:
        return None
    if ids is None:
        raise ValueError("median-depth cotangents need the forward's median ids")
    marr = (_b.ViewMedian * V)()
    for v in range(V):
        if grads[v] is None:
            continue
        g = _prep(grads[v], dev)
        i = ids[v].to(device=dev, dtype=torch.int32).contiguous()
        marr[v].median_id, marr[v].dL_dpix_median_depth = _ptr(i), _ptr(g)
        keep += [g, i]
    return marr


def _normal_array(grads, planes, V, dev, keep):
    """ViewNormal array of V views' normal cotangents and forward planes (per view [3,H,W] each, or None), or None without
    cotangents.  The tensors that must stay alive until the call is enqueued go to `keep`."""
    if grads is None:
        return None
    if planes is None:
        raise ValueError("normal cotangents need the forward's normal planes")
    narr = (_b.ViewNormal * V)()
    for v in range(V):
        if grads[v] is None:
            continue
        g = _prep(grads[v], dev)
        narr[v].out_normal, narr[v].dL_dpix_normal = _ptr(planes[v]), _ptr(g)
        keep += [g, planes[v]]
    return narr


def _camera_grads(L, camera_grads, Ps, dev, keep, intr=False):
    """(outputs, ViewCameraGrad array) for the views of clouds of Ps[v] Gaussians, or (None, None) without camera_grads.
    True allocates the three outputs [V,16], [V,16], [V,3] (and with `intr` a 4th, dL_dtan_fov [V,2]); a tuple names them
    (each a contiguous fp32 device tensor of that shape, or None)."""
    if camera_grads is None or camera_grads is False:
        return None, None
    V = len(Ps)
    opts = dict(dtype=torch.float32, device=dev)
    if camera_grads is True:
        camera_grads = (torch.empty((V, 16), **opts), torch.empty((V, 16), **opts), torch.empty((V, 3), **opts)) + \
            ((torch.empty((V, 2), **opts),) if intr else ())
    if intr and len(camera_grads) == 3:
        camera_grads = tuple(camera_grads) + (None,)
    shapes = ((V, 16), (V, 16), (V, 3), (V, 2))
    for t, shape in zip(camera_grads, shapes):
        if t is not None and (t.dtype != torch.float32 or t.device != dev or not t.is_contiguous() or t.numel() != shape[0] * shape[1]):
            raise ValueError(f"camera_grads: expected contiguous fp32 tensors of {shape} on {dev}")
    rows = [L.mgs_camera_grad_scratch_bytes(int(P)) // 4 for P in Ps]
    scratch = torch.empty((max(sum(rows), 1),), **opts)
    keep.append(scratch)
    carr = (_b.ViewCameraGrad * V)()
    off = 0
    for v in range(V):
        for name, t, n in zip(("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos"), camera_grads, (16, 16, 3)):
            setattr(carr[v], name, t.data_ptr() + 4 * n * v if t is not None else None)
        carr[v].scratch = scratch.data_ptr() + 4 * off
        off += rows[v]
    return tuple(camera_grads), carr


def _backward_view(L, w, s, o, dev, P, grad_color, grad_feature, grad_depth, normal=False):
    """Fills the backward fields of mgs_view `w` from the view's forward result `o` (a ViewOut) and its pixel gradients
    (the caller sets dL_dmean2D, stream and cot_scale); `normal`: the scratch also holds the normal gradients.  Returns the tensors that must stay alive until the call is enqueued."""
    H, W = int(s.image_height), int(s.image_width)
    bg, vm, pm, cp = (_prep(x, dev) for x in (s.bg, s.viewmatrix, s.projmatrix, s.campos))
    gc, gf, gd = (_prep(x, dev) for x in (grad_color, grad_feature, grad_depth))
    scratch = torch.empty((_state_sizes(L, P, W, H, normal)[2],), dtype=torch.uint8, device=dev)
    w.viewmatrix, w.projmatrix, w.cam_pos, w.background = _ptr(vm), _ptr(pm), _ptr(cp), _ptr(bg)
    w.tan_fovx, w.tan_fovy, w.width, w.height = _host_tan(s.tanfovx), _host_tan(s.tanfovy), W, H
    w.geometry_state, w.binning_state, w.image_state, w.binning_capacity = o[4].data_ptr(), o[5].data_ptr(), o[6].data_ptr(), int(o[0])
    w.radii = _ptr(o[3])
    w.dL_dpix, w.dL_dpix_F, w.dL_dpix_depth = _ptr(gc), _ptr(gf), _ptr(gd)
    w.blend_scratch = scratch.data_ptr()
    return (bg, vm, pm, cp, gc, gf, gd, scratch)


# ----------------------------------------------------------------------------------------------------------------------
# Several clouds in one call (DESIGN.md section 1, row f5): both frames of ManiGaussian's dynamic-field step, for every sample of
# the batch.  One C call (mgs_forward_clouds / mgs_backward_clouds) enqueues the views of ALL clouds stage by stage on their
# own streams between one fork and one join, so the clouds' chains overlap instead of queueing behind each other's blends.
_CLOUD_TENSORS = ("means3D", "sh", "colors", "feature", "opacity", "scales", "rotations", "cov3D_precomp")


def _nonempty(t):
    return t is not None and t.numel() != 0


def _prep_clouds(clouds, dev, include_feature):
    """Per cloud: its tensors as float32 contiguous on `dev`, and P, F, M.  Raises ValueError naming the field on which the
    clouds disagree (the C call shares the colour mode, the covariance mode, M and F between all clouds)."""
    out = []
    for b, c in enumerate(clouds):
        d = {k: _prep(c.get(k), dev) for k in _CLOUD_TENSORS}
        d["P"] = int(d["means3D"].size(0))
        if d["P"] == 0:
            raise ValueError(f"cloud {b} has no Gaussians (P = 0)")
        d["F"] = int(d["feature"].size(1)) if (include_feature and _nonempty(d["feature"])) else 0
        d["M"] = int(d["sh"].size(1)) if _nonempty(d["sh"]) else 0
        out.append(d)
    for field, key in (("colour mode (SHs or precomputed colours)", lambda d: _nonempty(d["colors"])),
                       ("covariance mode (scales/rotations or cov3D_precomp)", lambda d: _nonempty(d["cov3D_precomp"])),
                       ("SH degree (SH coefficients per Gaussian)", lambda d: d["M"]),
                       ("feature width F", lambda d: d["F"])):
        if len({key(d) for d in out}) > 1:
            raise ValueError(f"clouds disagree on the {field}")
    return out


def rasterize_clouds_raw(clouds, degree, include_feature, scale_modifier=1.0, return_depth=False, debug=False, return_alpha=False,
                         antialiasing=False, return_median=False, return_normal=False, planar_depth=None, views_call=False):
    """Forward of several Gaussian clouds, each with its own views, in one C call.  clouds[b] is a dict: "views" (a sequence
    of GaussianRasterizationSettings, one image size per cloud), the tensors "means3D", "sh" or "colors", "feature"
    (optional), "opacity", "scales" + "rotations" or "cov3D_precomp", and optionally "out_buffers", "loss_heads" and
    "capacities" as rasterize_views_raw takes them, and "depth_mask" and "ssim" (with "loss_heads") as its `depth_mask` and
    `ssim`.  degree, F, the
    colour and covariance modes are shared.  `return_alpha`
    appends every view's alpha plane to its ViewOut, as in rasterize_views_raw.  Returns
    (outs, streams): outs[b][v] is the ViewOut of view v of cloud b; streams are the per-view streams of all views in order.
    Capacity history is kept per (device, P, W, H, view slot across the call).  `antialiasing`: the anti-aliased projection for
    every cloud (C ABI mgs_render_options.antialiasing); pass the same value to the backward.  A cloud's optional "tan_fov" [V_b,2]
    (device) is its views' field of view, as rasterize_views_raw's `tan_fov` (C ABI mgs_render_options.intrinsics).
    `return_median` appends every view's median-depth and median-id planes to its ViewOut, as in rasterize_views_raw (C ABI
    mgs_view_median).  `return_normal` appends, last, every view's normal plane [3,H,W], as in rasterize_views_raw
    (C ABI mgs_view_normal).  A cloud's optional "ortho" (V_b flags; by default its views' `orthographic`
    attributes) marks its orthographic views (C ABI mgs_render_options.ortho); the backward reads the same entry.  A cloud's
    optional "fisheye" (V_b entries, each None or parameters; by default its views' `fisheye` attributes) marks its fisheye
    views (C ABI mgs_render_options.fisheye), likewise, and its optional "distortion" its distorted-pinhole views (C ABI
    mgs_render_options.distortion).  A cloud's optional "flow_means3D" [P,3] (its next-frame means) and "flow_poses" (as
    rasterize_views_raw takes them) append, last, its views' flow planes [3,H,W] (out_buffers[7] when given; C ABI
    mgs_render_options.flow).  `views_call`: one cloud, rendered by mgs_forward_views, the C ABI's one-cloud form (the
    backward then takes `views_call` too)."""
    L = _b.lib()
    pln = _planar_flag([s for c in clouds for s in c["views"]], planar_depth, return_normal)
    for c in clouds:
        _check_flow(c.get("flow_means3D"), return_normal, pln, c.get("depth_mask"))
    dev = clouds[0]["means3D"].device
    if not clouds[0]["means3D"].is_cuda:
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    pc = _prep_clouds(clouds, dev, include_feature)
    F, M, B = pc[0]["F"], pc[0]["M"], len(clouds)
    offsets = [0]
    for c in clouds:
        offsets.append(offsets[-1] + len(c["views"]))
    V = offsets[-1]
    main = torch.cuda.current_stream(dev)
    streams = _view_streams(dev, V) if V > 1 else [main]
    di = dev.index if dev.index is not None else torch.cuda.current_device()
    # capacity history per view of the call, g its index across the clouds: a one-cloud call keys its views as v
    keys = [[(di, d["P"], int(s.image_width), int(s.image_height), offsets[b] + v) for v, s in enumerate(c["views"])]
            for b, (c, d) in enumerate(zip(clouds, pc))]
    capturing = torch.cuda.is_current_stream_capturing()
    with torch.cuda.device(dev):
        if not capturing:
            _poll_status()
        for b, (c, d) in enumerate(zip(clouds, pc)):
            if c.get("capacities") is None and any(k not in _CAPACITY for k in keys[b]):
                if capturing:
                    raise RuntimeError("render the views once before capturing them in a CUDA graph (the binning capacity is "
                                       "learned from an eager call) or pass `capacities`")
                _calibrate(L, c["views"], keys[b], dev, d["P"], degree, M, d["means3D"], d["sh"], d["colors"], d["opacity"],
                           d["scales"], d["rotations"], scale_modifier, d["cov3D_precomp"], debug,
                           *_lens_arrays(c["views"], c.get("ortho"), c.get("fisheye"), c.get("distortion")))
        arr, carr, offs = (_b.View * V)(), (_b.Cloud * B)(), (ctypes.c_int * (B + 1))(*offsets)
        aarr = (_b.ViewAlpha * V)() if return_alpha else None
        darr = (_b.ViewDepthMask * V)() if any(c.get("depth_mask") is not None for c in clouds) else None
        sarr = (_b.ViewSsim * V)() if any(c.get("ssim") is not None for c in clouds) else None
        marr = (_b.ViewMedian * V)() if return_median else None
        narr = (_b.ViewNormal * V)() if return_normal else None
        status = _status_slots(V)
        keep, outs = [], []
        flarr, cfarr = _clouds_flow(clouds, pc, offsets, dev, keep)
        for b, (c, d) in enumerate(zip(clouds, pc)):
            k = carr[b]
            k.P = d["P"]
            k.means3D, k.shs, k.colors_precomp, k.opacities = _ptr(d["means3D"]), _ptr(d["sh"]), _ptr(d["colors"]), _ptr(d["opacity"])
            k.feature = _ptr(d["feature"]) if F else None
            k.scales, k.rotations, k.cov3D_precomp = _ptr(d["scales"]), _ptr(d["rotations"]), _ptr(d["cov3D_precomp"])
            caps = c.get("capacities")
            cloud_outs = []
            for v, s in enumerate(c["views"]):
                g = offsets[b] + v
                cap = int(caps[v]) if caps is not None else _CAPACITY[keys[b][v]]
                if c.get("depth_mask") is not None:
                    _fill_depth_mask(darr[g], c["depth_mask"], v)
                if c.get("ssim") is not None:
                    _fill_ssim(sarr[g], c["ssim"], v)
                o, kp = _forward_view(L, arr[g], s, v, dev, d["P"], F, cap, include_feature, return_depth, c.get("out_buffers"),
                                      c.get("loss_heads"), aarr[g] if return_alpha else None, marr[g] if return_median else None,
                                      narr[g] if return_normal else None, quads=pln,
                                      wf=flarr[g] if c.get("flow_means3D") is not None else None)
                arr[g].status = status.data_ptr() + 8 * g
                arr[g].stream = streams[g].cuda_stream
                keep.append(kp)
                cloud_outs.append(o)
            outs.append(cloud_outs)
        rest = (int(degree), M, F, float(scale_modifier), 0, int(bool(debug)), main.cuda_stream)
        tf = _clouds_fov(clouds, dev)
        keep.append(tf)
        oarr, farr, dcarr = _clouds_lens(clouds)
        iarr = _intrinsics_array(tf, None) if tf is not None else None
        opts = _b.RenderOptions(alpha=aarr, depth_mask=darr, ssim=sarr, intrinsics=iarr, median=marr, normal=narr,
                                ortho=oarr, fisheye=farr, distortion=dcarr, flow=flarr,
                                flow_next=cfarr if flarr is not None else None, antialiasing=int(bool(antialiasing)),
                                planar_depth=int(pln))
        if views_call:
            k = carr[0]
            _b.check(L.mgs_forward_views(V, arr, opts, k.P, int(degree), M, F, k.means3D, k.shs, k.colors_precomp, k.feature,
                                         k.opacities, k.scales, float(scale_modifier), k.rotations, k.cov3D_precomp, *rest[4:]),
                     "mgs_forward_views")
        else:
            _b.check(L.mgs_forward_clouds(B, carr, offs, arr, opts, *rest), "mgs_forward_clouds")
        flat = [o for co in outs for o in co]
        pending = not capturing and all(c.get("capacities") is None for c in clouds)
        _track_status(flat, [k for ks in keys for k in ks], status, main, pending)
    return outs, streams


def _clouds_flow(clouds, pc, offsets, dev, keep, backward=False):
    """(ViewFlow array of every view of the call, CloudFlow array) for clouds with "flow_means3D", or (None, None) without
    any.  The backward reads each cloud's forward planes "flow" and cotangents "grad_flow" ([V_b,3 or 2,H,W]) and allocates
    its "dL_dflow_means3D" into pc[b]."""
    if all(c.get("flow_means3D") is None for c in clouds):
        return None, None
    arr, carr = (_b.ViewFlow * offsets[-1])(), (_b.CloudFlow * len(clouds))()
    for b, (c, d) in enumerate(zip(clouds, pc)):
        fm = c.get("flow_means3D")
        if fm is None:
            continue
        fm = _prep(fm.detach(), dev)
        keep.append(fm)
        planes = c.get("flow") if backward else None
        grads = c.get("grad_flow") if backward else None
        one = _flow_array(c["views"], fm, c.get("flow_poses"), d["P"], dev, keep, planes, grads)
        for v in range(len(c["views"])):
            ctypes.memmove(ctypes.addressof(arr[offsets[b] + v]), ctypes.addressof(one[v]), ctypes.sizeof(_b.ViewFlow))
        carr[b].means3D = _ptr(fm)
        if backward:
            d["dL_dflow_means3D"] = torch.empty((d["P"], 3), dtype=torch.float32, device=dev)
            carr[b].dL_dmeans3D = _ptr(d["dL_dflow_means3D"])
    return arr, carr


def _clouds_lens(clouds):
    """_lens_arrays over every view of the clouds in order: each cloud's "ortho", "fisheye" and "distortion" entries, or its
    views' attributes"""
    def entries(key, attr):
        out = []
        for c in clouds:
            e = list(c[key]) if c.get(key) is not None else [getattr(s, attr, None) for s in c["views"]]
            if len(e) != len(c["views"]):
                raise ValueError(f"{key}: expected {len(c['views'])} entries, got {len(e)}")
            out += e
        return out
    return _lens_arrays([s for c in clouds for s in c["views"]], entries("ortho", "orthographic"), entries("fisheye", "fisheye"),
                        entries("distortion", "distortion"))


def _clouds_fov(clouds, dev):
    """[V,2] device field of view of every view of the clouds in order, or None when no cloud has one (the clouds without
    one contribute their host floats)"""
    tfs = [_device_fov(c["views"], c.get("tan_fov"), dev) for c in clouds]
    if all(t is None for t in tfs):
        return None
    return torch.cat([t if t is not None else _fov_column(c["views"], dev) for t, c in zip(tfs, clouds)])


def rasterize_clouds_backward_raw(clouds, outs, streams, degree, include_feature, scale_modifier=1.0, debug=False,
                                  antialiasing=False, camera_grads=False, planar_depth=None, accumulate=False, after_blend=None,
                                  views_call=False):
    """Backward of the clouds rendered by rasterize_clouds_raw: every view's blend backward on its stream, one join, then the
    per-Gaussian stage in launches that pack whole clouds (mgs_backward_clouds).  clouds[b]: the dict given to the forward
    plus "grad_color" [V_b,3,H,W], "grad_feature" [V_b,F,H,W] (with features), optionally "grad_depth" [V_b,H,W] and
    "grad_alpha" [V_b,H,W] (the cotangent of a `return_alpha` forward's alpha planes),
    "cot_scale" [V_b,2] (device; the loss heads' upstream gradients), "depth_mask" and "depth_mask_scale" [V_b,2] (the
    forward's depth / mask heads and their upstream gradients, as rasterize_views_backward_raw takes them) and "want_feature" (default True; False: the cloud's
    dL_dfeature is not computed, but its feature cotangents still reach the other gradients), and "ssim" and "ssim_scale" [V_b,2]
    as rasterize_views_backward_raw takes them.  Returns one dict per cloud
    holding the sums over its views: dL_dmeans3D [P,3], dL_dmeans2D [V_b,P,3] (per view), dL_dopacity [P,1], dL_dscales,
    dL_drotations, dL_dsh [P,M,3], dL_dcolors, dL_dcov3D, dL_dfeature (None where not computed).  `antialiasing`: the value
    the forward was given (C ABI mgs_render_options.antialiasing).  `camera_grads=True`: every cloud's dict also holds the gradients
    with respect to its views' viewmatrix, projmatrix and campos, "dL_dviewmatrix" [V_b,16], "dL_dprojmatrix" [V_b,16] and
    "dL_dcampos" [V_b,3] (C ABI mgs_render_options.camera_grad).  Clouds with a device field of view (see rasterize_clouds_raw)
    pass it as mgs_render_options.intrinsics, and `camera_grads=True` then adds "dL_dtan_fov" [V_b,2] to every dict.  A cloud's
    "grad_median" [V_b,H,W] is the cotangent of a `return_median` forward's median-depth planes, with "median_id" [V_b,H,W]
    int32 the id planes that forward returned (C ABI mgs_view_median).  A cloud's "grad_normal" [V_b,3,H,W] is the
    cotangent of a `return_normal` forward's normal planes, with "normal" [V_b,3,H,W] the planes that forward returned (C ABI
    mgs_view_normal).  The camera models of the clouds (see rasterize_clouds_raw) go to mgs_render_options.ortho, fisheye
    and distortion.  A cloud rendered with "flow_means3D" (and "flow_poses") also takes "flow" [V_b,3,H,W],
    the planes its forward returned, and "grad_flow" [V_b,2 or 3,H,W], their cotangent (C ABI mgs_render_options.flow and flow_next);
    its dict then holds "dL_dflow_means3D" [P,3].  A cloud's "accumulate_into" (a dict as rasterize_views_backward_raw takes it)
    receives its sums, overwritten or, with `accumulate`, added to.  Its "means2D_per_view" [V_b,P,3] receives the per-view
    dL_dmeans2D, or with "shared_mean2D" True its dict holds their sum [P,3].  `camera_grads` may also be a tuple of
    caller-given outputs over every view of the call, as rasterize_views_backward_raw takes it.  `views_call`: one cloud,
    run by mgs_backward_views, the C ABI's one-cloud form, which always computes the feature gradient; only such a call takes
    `after_blend` (called when the feature gradients are final) and a shared dL_dmeans2D."""
    L = _b.lib()
    pln = _planar_flag([s for c in clouds for s in c["views"]], planar_depth, any(c.get("grad_normal") is not None for c in clouds))
    for c in clouds:
        _check_flow(c.get("flow_means3D"), c.get("grad_normal") is not None, pln, c.get("depth_mask"))
        if c.get("flow_means3D") is not None and c.get("flow") is None:
            raise ValueError("flow cotangents need the forward's flow planes (\"flow\")")
    if not views_call and (after_blend is not None or any(c.get("shared_mean2D") for c in clouds)):
        raise ValueError("after_blend and a shared dL_dmeans2D need a one-cloud views call")
    dev = clouds[0]["means3D"].device
    pc = _prep_clouds(clouds, dev, include_feature)
    F, M, B = pc[0]["F"], pc[0]["M"], len(clouds)
    offsets = [0]
    for c in clouds:
        offsets.append(offsets[-1] + len(c["views"]))
    V = offsets[-1]
    main = torch.cuda.current_stream(dev)
    opts = dict(dtype=torch.float32, device=dev)
    grads = []
    with torch.cuda.device(dev):
        arr, carr, offs = (_b.View * V)(), (_b.Cloud * B)(), (ctypes.c_int * (B + 1))(*offsets)
        aarr = (_b.ViewAlpha * V)() if any(c.get("grad_alpha") is not None for c in clouds) else None
        darr = (_b.ViewDepthMask * V)() if any(c.get("depth_mask") is not None for c in clouds) else None
        sarr = (_b.ViewSsim * V)() if any(c.get("ssim") is not None for c in clouds) else None
        keep = []
        marr = None
        if any(c.get("grad_median") is not None for c in clouds):
            gm = [c["grad_median"][v] if c.get("grad_median") is not None else None for c in clouds for v in range(len(c["views"]))]
            ids = None if any(c.get("grad_median") is not None and c.get("median_id") is None for c in clouds) else \
                [c["median_id"][v] if c.get("grad_median") is not None else None for c in clouds for v in range(len(c["views"]))]
            marr = _median_array(gm, ids, V, dev, keep)
        narr = None
        if any(c.get("grad_normal") is not None for c in clouds):
            gn = [c["grad_normal"][v] if c.get("grad_normal") is not None else None for c in clouds for v in range(len(c["views"]))]
            pl = None if any(c.get("grad_normal") is not None and c.get("normal") is None for c in clouds) else \
                [c["normal"][v] if c.get("grad_normal") is not None else None for c in clouds for v in range(len(c["views"]))]
            narr = _normal_array(gn, pl, V, dev, keep)
        flarr, cfarr = _clouds_flow(clouds, pc, offsets, dev, keep, backward=True)
        for b, (c, d) in enumerate(zip(clouds, pc)):
            P, Vb = d["P"], len(c["views"])
            has_sr = _nonempty(d["scales"])
            acc = c.get("accumulate_into")

            def out(name, shape, need=True):
                t = acc.get(name) if acc is not None else None
                if t is None and need:
                    if acc is not None and name not in ("dL_dmeans2D", "dL_dcov3D"):
                        raise ValueError(f"accumulate_into lacks '{name}', the gradient of an input of this render")
                    t = torch.empty(shape, **opts)
                return t

            shared = bool(c.get("shared_mean2D"))
            m2d = out("dL_dmeans2D", (P, 3)) if shared else c.get("means2D_per_view")
            gr = dict(dL_dmeans3D=out("dL_dmeans3D", (P, 3)), dL_dmeans2D=m2d if m2d is not None else torch.empty((Vb, P, 3), **opts),
                      dL_dopacity=out("dL_dopacity", (P, 1)), dL_dscales=out("dL_dscales", (P, 3), has_sr),
                      dL_drotations=out("dL_drotations", (P, 4), has_sr), dL_dsh=out("dL_dsh", (P, M, 3), M > 0),
                      dL_dcolors=out("dL_dcolors", (P, 3), _nonempty(d["colors"])),
                      dL_dcov3D=out("dL_dcov3D", (P, 6), _nonempty(d["cov3D_precomp"])),
                      dL_dfeature=out("dL_dfeature", (P, F), views_call or c.get("want_feature", True)) if F else None)
            if "dL_dflow_means3D" in d:
                gr["dL_dflow_means3D"] = d["dL_dflow_means3D"]
            grads.append(gr)
            k = carr[b]
            k.P = P
            k.means3D, k.shs, k.colors_precomp = _ptr(d["means3D"]), _ptr(d["sh"]), _ptr(d["colors"])
            k.feature = _ptr(d["feature"]) if F else None
            k.scales, k.rotations, k.cov3D_precomp = _ptr(d["scales"]), _ptr(d["rotations"]), _ptr(d["cov3D_precomp"])
            k.dL_dmean3D, k.dL_dopacity, k.dL_dcolor = _ptr(gr["dL_dmeans3D"]), _ptr(gr["dL_dopacity"]), _ptr(gr["dL_dcolors"])
            k.dL_dfeature, k.dL_dcov3D, k.dL_dsh = _ptr(gr["dL_dfeature"]), _ptr(gr["dL_dcov3D"]), _ptr(gr["dL_dsh"]) if M else None
            k.dL_dscale = _ptr(gr["dL_dscales"]) if has_sr else None
            k.dL_drot = _ptr(gr["dL_drotations"]) if has_sr else None
            cot = _prep(c.get("cot_scale"), dev)
            dscale = _prep(c.get("depth_mask_scale"), dev)
            sscale = _prep(c.get("ssim_scale"), dev)
            keep += [dscale, sscale]
            for v, s in enumerate(c["views"]):
                g = offsets[b] + v
                w = arr[g]
                if c.get("depth_mask") is not None:
                    _fill_depth_mask(darr[g], c["depth_mask"], v, dscale)
                keep.append(_backward_view(L, w, s, outs[b][v], dev, P, c["grad_color"][v],
                                           c["grad_feature"][v] if (F and c.get("grad_feature") is not None) else None,
                                           c["grad_depth"][v] if c.get("grad_depth") is not None else None,
                                           c.get("grad_normal") is not None or pln or c.get("flow_means3D") is not None))
                w.dL_dmean2D = _ptr(gr["dL_dmeans2D"]) if shared else _ptr(gr["dL_dmeans2D"][v])
                w.stream = streams[g].cuda_stream
                if c.get("grad_alpha") is not None:
                    ga = _prep(c["grad_alpha"][v], dev)
                    aarr[g].dL_dpix_alpha = _ptr(ga)
                    keep.append(ga)
                if cot is not None:
                    w.cot_scale = cot.data_ptr() + 8 * v
                if c.get("ssim") is not None:
                    _fill_ssim(sarr[g], c["ssim"], v, w, sscale)
            keep.append(cot)
        tf = _clouds_fov(clouds, dev)
        keep.append(tf)
        cam, camarr = _camera_grads(L, camera_grads, [d["P"] for d, c in zip(pc, clouds) for _ in c["views"]], dev, keep,
                                    tf is not None)
        if cam is not None:
            for b, gr in enumerate(grads):
                for name, t in zip(_CAMERA_GRADS, cam):
                    gr[name] = t[offsets[b]:offsets[b + 1]] if (t is not None and not views_call) else t
        rest = (int(degree), M, F, float(scale_modifier), int(bool(accumulate)), int(bool(debug)), main.cuda_stream)
        oarr, farr, dcarr = _clouds_lens(clouds)
        iarr = _intrinsics_array(tf, cam[3] if cam is not None else None) if tf is not None else None
        opts = _b.RenderOptions(alpha=aarr, depth_mask=darr, ssim=sarr, camera_grad=camarr, intrinsics=iarr, median=marr,
                                normal=narr, ortho=oarr, fisheye=farr, distortion=dcarr, flow=flarr,
                                flow_next=cfarr if flarr is not None else None, antialiasing=int(bool(antialiasing)),
                                planar_depth=int(pln))
        if views_call:
            k = carr[0]
            for stages in ((1, 2) if after_blend is not None else (3,)):
                _b.check(L.mgs_backward_views(V, arr, opts, k.P, int(degree), M, F, k.means3D, k.shs if M else None, k.colors_precomp,
                                              k.feature, k.scales, float(scale_modifier), k.rotations, k.cov3D_precomp, k.dL_dmean3D,
                                              k.dL_dopacity, k.dL_dcolor, k.dL_dfeature, k.dL_dcov3D, k.dL_dsh, k.dL_dscale, k.dL_drot,
                                              int(bool(clouds[0].get("shared_mean2D"))), *rest[4:5], stages, *rest[5:]),
                         "mgs_backward_views")
                if stages == 1:
                    after_blend()
        else:
            _b.check(L.mgs_backward_clouds(B, carr, offs, arr, opts, *rest), "mgs_backward_clouds")
    return grads


def field_query_raw(points, means3D, scales, rotations, opacity, features=None, channel_first=False, debug=False):
    """Density and features of the Gaussian field at points [Q,3] (C ABI mgs_field_query; definition in
    include/mgs_rasterizer.h).  features [P,C] or None.  Returns (density [Q], features [Q,C] ([C,Q] with channel_first) or
    None, query state, pair state, pair count); the two states serve field_query_backward_raw.  One host synchronisation."""
    if not points.is_cuda:
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    L = _b.lib()
    dev = points.device
    Q, P = points.size(0), means3D.size(0)
    points, means3D, scales, rotations, opacity = (_prep(x, dev) for x in (points, means3D, scales, rotations, opacity))
    C = features.size(1) if features is not None else 0
    features = _prep(features, dev) if C else None
    density = torch.empty((Q,), dtype=torch.float32, device=dev)
    out = torch.empty((C, Q) if channel_first else (Q, C), dtype=torch.float32, device=dev) if C else None
    sa, pa = _Alloc(dev), _Alloc(dev)
    with torch.cuda.device(dev):
        n = _checked((sa, pa), L.mgs_field_query(_ALLOC_CB, sa.key, _ALLOC_CB, pa.key, Q, P, C, _ptr(points), _ptr(means3D),
                                                 _ptr(scales), _ptr(rotations), _ptr(opacity), _ptr(features), int(bool(channel_first)),
                                                 _ptr(density), _ptr(out), int(bool(debug)), _stream(dev)), "mgs_field_query")
    return density, out, sa.release(), pa.release(), n


def field_query_backward_raw(state, pair_state, points, scales, rotations, features, grad_density, grad_features,
                             channel_first=False, needs=(True,) * 6, debug=False):
    """Gradients of a field_query_raw call (C ABI mgs_field_query_backward) from the cotangents grad_density [Q] and
    grad_features (laid out as the forward's features), each None for zero.  `needs` selects, in this order, dL/dpoints,
    dL/dmeans3D, dL/dscales, dL/drotations, dL/dopacity [P] and dL/dfeatures; each unselected one is None and not computed."""
    L = _b.lib()
    dev = points.device
    Q, P = points.size(0), scales.size(0)
    points, scales, rotations = (_prep(x, dev) for x in (points, scales, rotations))
    C = features.size(1) if features is not None else 0
    features = _prep(features, dev) if C else None
    grad_density = _prep(grad_density, dev)
    grad_features = _prep(grad_features, dev) if C else None
    shapes = ((Q, 3), (P, 3), (P, 3), (P, 4), (P,), (P, C))
    outs = [torch.empty(s, dtype=torch.float32, device=dev) if n and (k < 5 or C) else None
            for k, (s, n) in enumerate(zip(shapes, needs))]
    with torch.cuda.device(dev):
        _b.check(L.mgs_field_query_backward(_ptr(state), _ptr(pair_state), Q, P, C, _ptr(points), _ptr(scales), _ptr(rotations),
                                            _ptr(features), int(bool(channel_first)), _ptr(grad_density), _ptr(grad_features),
                                            *[_ptr(o) for o in outs], int(bool(debug)), _stream(dev)), "mgs_field_query_backward")
    return tuple(outs)


def knn_raw(points, k, queries=None, debug=False):
    """The k nearest of `points` [N,3] to each query (C ABI mgs_knn; definition in include/mgs_rasterizer.h): `queries` [Q,3],
    or None for the points themselves (each without its own index).  Returns (index [Q,k] int64, dist2 [Q,k] float32) on the
    points' device, each query's entries ascending by (d2, index), padded with index -1 and d2 = +inf.  The state is
    allocated with torch and nothing is read back, so a call can be captured in a CUDA graph.  Not differentiable."""
    if not points.is_cuda or (queries is not None and not queries.is_cuda):
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    L = _b.lib()
    dev = points.device
    points = _prep(points, dev)
    queries = _prep(queries, dev)
    N = points.size(0)
    Q = N if queries is None else queries.size(0)
    index = torch.empty((Q, k), dtype=torch.int64, device=dev)
    dist2 = torch.empty((Q, k), dtype=torch.float32, device=dev)
    if Q == 0:
        return index, dist2
    with torch.cuda.device(dev):  # the state's size depends on the device it is used on
        nbytes = int(L.mgs_knn_state_bytes(N, Q))
        if nbytes == 0:
            raise RuntimeError("mgs_knn_state_bytes: " + _b.last_error())
        state = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _b.check(L.mgs_knn(_ptr(state), N, Q, int(k), _ptr(points), _ptr(queries), _ptr(index), _ptr(dist2), int(bool(debug)),
                           _stream(dev)), "mgs_knn")
    return index, dist2


def neighbour_reg_raw(xyz, rot, xyz_next, rot_next, index, weight, debug=False):
    """The neighbour regularisers (C ABI mgs_neighbour_reg; definition in include/mgs_rasterizer.h) of a cloud xyz [P,3],
    rot [P,4] and its next frame xyz_next [P,3], rot_next [P,4] over index [P,k] int64 with constant weight [P,k].
    Returns (loss [3] = {rigid, rotation, isometry}, state) on xyz's device; the state is what neighbour_reg_backward_raw
    reads.  Nothing is read back to the host, so a call can be captured in a CUDA graph.  Not differentiable."""
    if not all(t.is_cuda for t in (xyz, rot, xyz_next, rot_next, index, weight)):
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    L = _b.lib()
    dev = xyz.device
    xyz, rot, xyz_next, rot_next, weight = (_prep(t, dev) for t in (xyz, rot, xyz_next, rot_next, weight))
    index = index.to(device=dev, dtype=torch.int64).contiguous()
    P, k = index.shape
    loss = torch.empty(3, dtype=torch.float32, device=dev)
    state = torch.empty(int(L.mgs_neighbour_reg_state_bytes(P, k)), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _b.check(L.mgs_neighbour_reg(_ptr(state), P, k, _ptr(xyz), _ptr(rot), _ptr(xyz_next), _ptr(rot_next), _ptr(index),
                                     _ptr(weight), _ptr(loss), int(bool(debug)), _stream(dev)), "mgs_neighbour_reg")
    return loss, state


def neighbour_reg_backward_raw(state, xyz, rot, xyz_next, rot_next, index, weight, grad_loss, needs=(True,) * 4, debug=False):
    """Backward of neighbour_reg_raw (C ABI mgs_neighbour_reg_backward) with the state its forward returned for the same
    inputs: grad_loss [3] on the device (read there, never by the host).  Returns (dL_dxyz, dL_drot, dL_dxyz_next,
    dL_drot_next), each None where `needs` is False."""
    L = _b.lib()
    dev = xyz.device
    xyz, rot, xyz_next, rot_next, weight = (_prep(t, dev) for t in (xyz, rot, xyz_next, rot_next, weight))
    index = index.to(device=dev, dtype=torch.int64).contiguous()
    grad_loss = _prep(grad_loss, dev)
    P, k = index.shape
    outs = [torch.empty((P, c), dtype=torch.float32, device=dev) if n else None for n, c in zip(needs, (3, 4, 3, 4))]
    with torch.cuda.device(dev):
        _b.check(L.mgs_neighbour_reg_backward(_ptr(state), P, k, _ptr(xyz), _ptr(rot), _ptr(xyz_next), _ptr(rot_next),
                                              _ptr(index), _ptr(weight), _ptr(grad_loss), *[_ptr(o) for o in outs],
                                              int(bool(debug)), _stream(dev)), "mgs_neighbour_reg_backward")
    return tuple(outs)


def deform_raw(xyz, rot, node_xyz, node_rot, node_t, index, weight, debug=False):
    """A cloud xyz [P,3], rot [P,4] deformed by control nodes node_xyz [N,3], node_rot [N,4], node_t [N,3] over index [P,k]
    int64 with weight [P,k] (C ABI mgs_deform; definition in include/mgs_rasterizer.h).  Returns (out_xyz [P,3],
    out_rot [P,4], state) on xyz's device; the state is what deform_backward_raw reads.  Nothing is read back to the host,
    so a call can be captured in a CUDA graph.  Not differentiable."""
    if not all(t.is_cuda for t in (xyz, rot, node_xyz, node_rot, node_t, index, weight)):
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    L = _b.lib()
    dev = xyz.device
    xyz, rot, node_xyz, node_rot, node_t, weight = (_prep(t, dev) for t in (xyz, rot, node_xyz, node_rot, node_t, weight))
    index = index.to(device=dev, dtype=torch.int64).contiguous()
    P, k = index.shape
    N = node_xyz.shape[0]
    out_xyz = torch.empty((P, 3), dtype=torch.float32, device=dev)
    out_rot = torch.empty((P, 4), dtype=torch.float32, device=dev)
    state = torch.empty(int(L.mgs_deform_state_bytes(P, N, k)), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _b.check(L.mgs_deform(_ptr(state), P, N, k, _ptr(xyz), _ptr(rot), _ptr(node_xyz), _ptr(node_rot), _ptr(node_t),
                              _ptr(index), _ptr(weight), _ptr(out_xyz), _ptr(out_rot), int(bool(debug)), _stream(dev)),
                 "mgs_deform")
    return out_xyz, out_rot, state


def deform_backward_raw(state, xyz, rot, node_xyz, node_rot, node_t, index, weight, grad_xyz, grad_rot, needs=(True,) * 6,
                        debug=False):
    """Backward of deform_raw (C ABI mgs_deform_backward) with the state its forward returned for the same inputs:
    grad_xyz [P,3] and grad_rot [P,4], each None for zero.  Returns (dL_dxyz, dL_drot, dL_dnode_xyz, dL_dnode_rot,
    dL_dnode_t, dL_dweight), each None where `needs` is False."""
    L = _b.lib()
    dev = xyz.device
    xyz, rot, node_xyz, node_rot, node_t, weight, grad_xyz, grad_rot = (
        _prep(t, dev) for t in (xyz, rot, node_xyz, node_rot, node_t, weight, grad_xyz, grad_rot))
    index = index.to(device=dev, dtype=torch.int64).contiguous()
    P, k = index.shape
    N = node_xyz.shape[0]
    shapes = ((P, 3), (P, 4), (N, 3), (N, 4), (N, 3), (P, k))
    outs = [torch.empty(s, dtype=torch.float32, device=dev) if n else None for n, s in zip(needs, shapes)]
    with torch.cuda.device(dev):
        _b.check(L.mgs_deform_backward(_ptr(state), P, N, k, _ptr(xyz), _ptr(rot), _ptr(node_xyz), _ptr(node_rot),
                                       _ptr(node_t), _ptr(index), _ptr(weight), _ptr(grad_xyz), _ptr(grad_rot),
                                       *[_ptr(o) for o in outs], int(bool(debug)), _stream(dev)), "mgs_deform_backward")
    return tuple(outs)


def fps_raw(points, n, lengths=None, start=None, debug=False):
    """Farthest-point sampling of n picks from each cloud of `points` [B,P,3] (C ABI mgs_fps; definition in
    include/mgs_rasterizer.h), each cloud cut to lengths[b] points ([B] int64, or None for all P) and started at start[b]
    ([B] int64, or None).  Returns (index [B,n] int64, dist2 [B,n] float32) on the points' device, padded with index -1 and
    d2 = +inf.  The state is allocated with torch and nothing is read back, so a call can be captured in a CUDA graph.  Not
    differentiable."""
    if not points.is_cuda:
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    L = _b.lib()
    dev = points.device
    points = _prep(points, dev)
    lengths, start = (None if t is None else t.to(device=dev, dtype=torch.int64).contiguous() for t in (lengths, start))
    B, P = points.shape[0], points.shape[1]
    index = torch.empty((B, n), dtype=torch.int64, device=dev)
    dist2 = torch.empty((B, n), dtype=torch.float32, device=dev)
    if B == 0 or n == 0:
        return index, dist2
    state = torch.empty(int(L.mgs_fps_state_bytes(B, P)), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):  # the cluster sizes are looked up for the device current at the call
        _b.check(L.mgs_fps(_ptr(state), B, P, int(n), _ptr(points), _ptr(lengths), _ptr(start), _ptr(index), _ptr(dist2),
                           int(bool(debug)), _stream(dev)), "mgs_fps")
    return index, dist2


def tsdf_fuse_raw(views, depth, bounds, resolution, trunc, color=None, volume=None, tan_fov=None, ortho=None, fisheye=None,
                  distortion=None, debug=False):
    """Depth images fused into a TSDF volume (C ABI mgs_tsdf_fuse; definition in include/mgs_rasterizer.h).  depth [V,H,W]
    view-space z on the views' device, every view W x H; color [V,C,H,W] or None; bounds (x0, y0, z0, x1, y1, z1) and
    resolution (X, Y, Z) as voxel_centres takes them; trunc > 0.  volume: (tsdf [X,Y,Z], weight [X,Y,Z], color [C,X,Y,Z] or
    None), updated in place, or None for a fresh one (tsdf 1, weight 0, colour 0).  `views`, `tan_fov`, `ortho`, `fisheye`
    and `distortion` as in camera_rays_raw.  Returns (tsdf, weight, color or None).  Nothing is read back to the host."""
    L = _b.lib()
    dev, _, _, arr, tf, (oarr, farr, dcarr), keep = _ray_call(views, None, tan_fov, ortho, fisheye, distortion)
    V = len(views)
    X, Y, Z = (int(n) for n in resolution)
    C = 0 if color is None else int(color.shape[1])
    depth, color = _prep(depth, dev), _prep(color, dev)
    if volume is None:
        volume = (torch.ones((X, Y, Z), dtype=torch.float32, device=dev), torch.zeros((X, Y, Z), dtype=torch.float32, device=dev),
                  torch.zeros((C, X, Y, Z), dtype=torch.float32, device=dev) if C else None)
    tsdf, weight, cvol = volume
    iarr = _intrinsics_array(tf, None) if tf is not None else None
    b = (ctypes.c_double * 6)(*[float(x) for x in bounds])
    with torch.cuda.device(dev):
        _b.check(L.mgs_tsdf_fuse(V, arr, iarr, oarr, farr, dcarr, _ptr(depth), C, _ptr(color), b, X, Y, Z, float(trunc), _ptr(tsdf),
                                 _ptr(weight), _ptr(cvol) if C else None, int(bool(debug)), _stream(dev)), "mgs_tsdf_fuse")
    return tsdf, weight, cvol


def marching_cubes_raw(values, level, bounds, weight=None, color=None, debug=False):
    """The level surface of values [X,Y,Z] (C ABI mgs_marching_cubes_count / _emit; definition in include/mgs_rasterizer.h),
    grid point (i, j, k) at its voxel centre over bounds; weight [X,Y,Z] or None (a point is valid where its weight is > 0),
    color [C,X,Y,Z] or None.  Returns (vertices [Nv,3] float32, faces [Nf,3] int64, colors [Nv,C] or None).  One
    device->host read of the two totals sizes the outputs."""
    if not values.is_cuda:
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    L = _b.lib()
    dev = values.device
    values, weight, color = _prep(values, dev), _prep(weight, dev), _prep(color, dev)
    X, Y, Z = values.shape
    C = 0 if color is None else int(color.shape[0])
    counts = torch.zeros(2, dtype=torch.int64, device=dev)
    state = torch.empty(int(L.mgs_marching_cubes_state_bytes(X, Y, Z)), dtype=torch.uint8, device=dev)
    lvl = float(level)
    with torch.cuda.device(dev):
        _b.check(L.mgs_marching_cubes_count(_ptr(state), X, Y, Z, _ptr(values), _ptr(weight), lvl, _ptr(counts), int(bool(debug)),
                                            _stream(dev)), "mgs_marching_cubes_count")
        nv, nf = (int(n) for n in counts.cpu())
        vertices = torch.empty((nv, 3), dtype=torch.float32, device=dev)
        faces = torch.empty((nf, 3), dtype=torch.int64, device=dev)
        colors = torch.empty((nv, C), dtype=torch.float32, device=dev) if C else None
        if nv or nf:
            b = (ctypes.c_double * 6)(*[float(x) for x in bounds])
            _b.check(L.mgs_marching_cubes_emit(_ptr(state), X, Y, Z, _ptr(values), lvl, b, C, _ptr(color), _ptr(vertices), _ptr(faces),
                                               _ptr(colors), int(bool(debug)), _stream(dev)), "mgs_marching_cubes_emit")
    return vertices, faces, colors


def _pointer_list(tensors):
    """host arrays (device pointers, floats per row) of a list of [P, ...] tensors, for the C ABI's generic row lists"""
    n = len(tensors)
    ptrs = (ctypes.c_void_p * max(n, 1))(*[t.data_ptr() for t in tensors])
    widths = (ctypes.c_int * max(n, 1))(*[t.numel() // max(t.shape[0], 1) for t in tensors])
    return n, ptrs, widths


def mcmc_relocate_raw(P_old, means, quats, log_scales, opacity_logit, rows, moments, rng, min_opacity=0.005, debug=False):
    """MCMC relocation and growth in place (C ABI mgs_mcmc_relocate; definition in include/mgs_rasterizer.h): means [P,3],
    quats [P,4], log_scales [P,3], opacity_logit [P] or [P,1], every tensor of `rows` and `moments` [P, ...], all float32,
    contiguous and on one device; rows [P_old, P) are newly appended.  rng: device int64 [2] = {seed, offset}, advanced by
    one on the device.  Returns (source [P] int64, relocated [1] int64) on the same device.  Nothing is read back to the
    host, so a call can be captured in a CUDA graph."""
    if not means.is_cuda:
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    L = _b.lib()
    dev = means.device
    P = means.shape[0]
    source = torch.empty(P, dtype=torch.int64, device=dev)
    relocated = torch.empty(1, dtype=torch.int64, device=dev)
    nr, rp, rw = _pointer_list(rows)
    nm, mp, mw = _pointer_list(moments)
    with torch.cuda.device(dev):  # the state's size depends on the device it is used on
        nbytes = int(L.mgs_mcmc_state_bytes(int(P_old)))
        if nbytes == 0:
            raise RuntimeError("mgs_mcmc_state_bytes: " + _b.last_error())
        state = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _b.check(L.mgs_mcmc_relocate(_ptr(state), int(P_old), P, float(min_opacity), _ptr(means), _ptr(quats), _ptr(log_scales),
                                     _ptr(opacity_logit), nr, rp, rw, nm, mp, mw, _ptr(rng), _ptr(source), _ptr(relocated),
                                     int(bool(debug)), _stream(dev)), "mgs_mcmc_relocate")
    return source, relocated


def mcmc_perturb_raw(means, quats, log_scales, opacity_logit, scale, rng, debug=False):
    """MCMC position noise in place (C ABI mgs_mcmc_perturb; definition in include/mgs_rasterizer.h): means [P,3] += the
    covariance-shaped noise of quats [P,4], log_scales [P,3] and opacity_logit [P], times scale (device float32 [1]).  rng:
    device int64 [2] = {seed, offset}, advanced by one on the device.  Only means is written; nothing is read back."""
    if not means.is_cuda:
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    L = _b.lib()
    dev = means.device
    if quats.data_ptr() % 16:  # the kernel reads each quaternion as one 16-byte load
        quats = quats.clone()
    with torch.cuda.device(dev):
        _b.check(L.mgs_mcmc_perturb(means.shape[0], _ptr(means), _ptr(quats), _ptr(log_scales), _ptr(opacity_logit), _ptr(scale),
                                    _ptr(rng), int(bool(debug)), _stream(dev)), "mgs_mcmc_perturb")
    return means


def densify_stats_raw(viewspace_grad, radii, sizes, grad2d, count, radius, scale=1.0, debug=False):
    """Density-control statistics in place (C ABI mgs_densify_stats; definition in include/mgs_rasterizer.h):
    viewspace_grad [V,P,3] float32, radii [V,P] int32, sizes: V host ints (each view's max(W, H)), grad2d [P] float32,
    count [P] int32 and radius [P] float32 (updated), all contiguous on one device.  scale: a number, or a float32 tensor of
    one element on the device.  Nothing is read back to the host, so a call can be captured in a CUDA graph."""
    if not viewspace_grad.is_cuda:
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    L = _b.lib()
    dev = viewspace_grad.device
    V, P = int(viewspace_grad.shape[0]), int(viewspace_grad.shape[1])
    sz = (ctypes.c_int * max(V, 1))(*[int(s) for s in sizes])
    dscale = scale if torch.is_tensor(scale) else None
    with torch.cuda.device(dev):
        _b.check(L.mgs_densify_stats(V, P, _ptr(viewspace_grad), _ptr(radii), sz, 1.0 if dscale is not None else float(scale),
                                     _ptr(dscale), _ptr(grad2d), _ptr(count), _ptr(radius), int(bool(debug)), _stream(dev)),
                 "mgs_densify_stats")


def densify_and_prune_raw(means, quats, log_scales, opacity_logit, rows, moments, grad2d, count, radius, rng, scene_scale,
                          grad_threshold=2e-4, grow_scale3d=0.01, grow_scale2d=math.inf, prune_opacity=0.005,
                          prune_scale3d=0.1, prune_scale2d=math.inf, prune_too_big=False, debug=False):
    """Clone, split and prune (C ABI mgs_densify_count / mgs_densify_emit; definition in include/mgs_rasterizer.h): means
    [P,3], quats [P,4], log_scales [P,3], opacity_logit [P] or [P,1], every tensor of `rows` and `moments` [P, ...], all
    float32 and contiguous, and the statistics grad2d [P], count [P] int32, radius [P] on one device; grow_scale2d and
    prune_scale2d take math.inf for no test.  rng: device int64 [2] = {seed, offset}; emit advances the offset by one on
    the device.  One device->host read of the four totals sizes the outputs.  Returns (counts (n_new, cloned, split,
    pruned) as host ints, or None when nothing is cloned, split or pruned (then nothing is enqueued after the count),
    else (new means, quats, log_scales, opacity_logit, [new rows], [new moments], source [n_new] int64))."""
    if not means.is_cuda:
        raise RuntimeError("manigaussian_b200 runs on CUDA tensors only (there is no CPU path)")
    L = _b.lib()
    dev = means.device
    P = int(means.shape[0])
    counts = torch.empty(4, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):  # the state's size depends on the device it is used on
        nbytes = int(L.mgs_densify_state_bytes(P))
        if nbytes == 0:
            raise RuntimeError("mgs_densify_state_bytes: " + _b.last_error())
        state = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _b.check(L.mgs_densify_count(_ptr(state), P, _ptr(log_scales), _ptr(opacity_logit), _ptr(grad2d), _ptr(count),
                                     _ptr(radius), float(scene_scale), float(grad_threshold), float(grow_scale3d),
                                     float(grow_scale2d), float(prune_opacity), float(prune_scale3d), float(prune_scale2d),
                                     int(bool(prune_too_big)), _ptr(counts), int(bool(debug)), _stream(dev)), "mgs_densify_count")
        totals = tuple(int(n) for n in counts.cpu())
        n_new, cloned, split, pruned = totals
        if cloned == 0 and split == 0 and pruned == 0:
            return totals, None
        if n_new > 2 ** 31 - 1:
            raise RuntimeError(f"densify_and_prune: {n_new} Gaussians after refinement exceed the 2^31 - 1 the kernels index")

        def grown(t):
            return torch.empty((n_new,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)

        new = [grown(t) for t in (means, quats, log_scales, opacity_logit)]
        new_rows, new_moments = [grown(t) for t in rows], [grown(t) for t in moments]
        source = torch.empty(n_new, dtype=torch.int64, device=dev)
        nr, rp, rw = _pointer_list(rows)
        nm, mp, mw = _pointer_list(moments)
        _, nrp, _ = _pointer_list(new_rows)
        _, nmp, _ = _pointer_list(new_moments)
        _b.check(L.mgs_densify_emit(_ptr(state), P, n_new, _ptr(means), _ptr(quats), _ptr(log_scales), _ptr(opacity_logit),
                                    nr, rp, rw, nm, mp, mw, *[_ptr(t) for t in new], nrp, nmp, _ptr(rng), _ptr(source),
                                    int(bool(debug)), _stream(dev)), "mgs_densify_emit")
    return totals, (*new, new_rows, new_moments, source)

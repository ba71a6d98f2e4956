"""ctypes binding of the C ABI in include/mgs_rasterizer.h.

The CUDA library is the product path: importing this module raises if it cannot be built or loaded.
There is no CPU or PyTorch fallback anywhere in this package.
"""
import ctypes as C
import os

from . import build as _build

_c_float_p = C.c_void_p  # device pointers are passed as integers
ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_size_t)



class View(C.Structure):
    """mirror of `mgs_view` (include/mgs_rasterizer.h)"""
    _fields_ = [("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("cam_pos", C.c_void_p), ("background", C.c_void_p),
                ("tan_fovx", C.c_float), ("tan_fovy", C.c_float), ("width", C.c_int), ("height", C.c_int),
                ("geometry_state", C.c_void_p), ("binning_state", C.c_void_p), ("image_state", C.c_void_p),
                ("binning_capacity", C.c_int),
                ("out_color", C.c_void_p), ("out_feature", C.c_void_p), ("out_depth", C.c_void_p), ("radii", C.c_void_p),
                ("status", C.c_void_p),
                ("dL_dpix", C.c_void_p), ("dL_dpix_F", C.c_void_p), ("dL_dpix_depth", C.c_void_p),
                ("blend_scratch", C.c_void_p), ("dL_dmean2D", C.c_void_p), ("stream", C.c_void_p),
                ("target_color", C.c_void_p), ("target_feature", C.c_void_p), ("cot_color", C.c_void_p),
                ("cot_feature", C.c_void_p), ("loss_acc", C.c_void_p), ("cot_scale", C.c_void_p)]


class ViewAlpha(C.Structure):
    """mirror of `mgs_view_alpha` (include/mgs_rasterizer.h): the optional alpha plane of one view"""
    _fields_ = [("out_alpha", C.c_void_p), ("dL_dpix_alpha", C.c_void_p)]


class ViewDepthMask(C.Structure):
    """mirror of `mgs_view_depth_mask` (include/mgs_rasterizer.h): the optional depth and mask heads of one view"""
    _fields_ = [(n, C.c_void_p) for n in ("target_depth", "target_mask", "cot_depth", "cot_alpha_depth", "cot_alpha_mask",
                                          "loss_acc", "cot_scale")]


class ViewSsim(C.Structure):
    """mirror of `mgs_view_ssim` (include/mgs_rasterizer.h): the optional L1 + SSIM head of one view"""
    _fields_ = [(n, C.c_void_p) for n in ("ssim_terms", "loss_acc", "cot_scale", "cot_color")]


class ViewCameraGrad(C.Structure):
    """mirror of `mgs_view_camera_grad` (include/mgs_rasterizer.h): the optional camera gradients of one view"""
    _fields_ = [(n, C.c_void_p) for n in ("dL_dviewmatrix", "dL_dprojmatrix", "dL_dcampos", "scratch")]


class ViewIntrinsics(C.Structure):
    """mirror of `mgs_view_intrinsics` (include/mgs_rasterizer.h): the optional device field of view of one view and its
    gradient"""
    _fields_ = [(n, C.c_void_p) for n in ("tan_fov", "dL_dtan_fov")]


class ViewMedian(C.Structure):
    """mirror of `mgs_view_median` (include/mgs_rasterizer.h): the optional median-depth plane and surface-Gaussian ids of
    one view"""
    _fields_ = [(n, C.c_void_p) for n in ("out_median_depth", "median_id", "dL_dpix_median_depth")]


class ViewNormal(C.Structure):
    """mirror of `mgs_view_normal` (include/mgs_rasterizer.h): the optional surface-normal plane of one view"""
    _fields_ = [(n, C.c_void_p) for n in ("out_normal", "dL_dpix_normal")]


class ViewFlow(C.Structure):
    """mirror of `mgs_view_flow` (include/mgs_rasterizer.h): the optional flow plane of one view and its next-frame pose"""
    _fields_ = [(n, C.c_void_p) for n in ("next_viewmatrix", "next_projmatrix", "out_flow", "dL_dpix_flow")]


class CloudFlow(C.Structure):
    """mirror of `mgs_cloud_flow` (include/mgs_rasterizer.h): one cloud's next-frame means and their gradient"""
    _fields_ = [(n, C.c_void_p) for n in ("means3D", "dL_dmeans3D")]


class ViewFisheye(C.Structure):
    """mirror of `mgs_view_fisheye` (include/mgs_rasterizer.h): one view's Kannala-Brandt fisheye parameters"""
    _fields_ = [("fisheye", C.c_int)] + [(n, C.c_float) for n in ("cx", "cy", "k1", "k2", "k3", "k4", "theta_max")]


class ViewDistortion(C.Structure):
    """mirror of `mgs_view_distortion` (include/mgs_rasterizer.h): one view's OpenCV distortion parameters"""
    _fields_ = [("distorted", C.c_int)] + \
        [(n, C.c_float) for n in ("cx", "cy", "k1", "k2", "p1", "p2", "k3", "k4", "k5", "k6", "r_max")]


class RenderOptions(C.Structure):
    """mirror of `mgs_render_options` (include/mgs_rasterizer.h): every optional input of the render calls; the array
    fields take ctypes arrays (kept alive by the record) or None"""
    _fields_ = [("alpha", C.POINTER(ViewAlpha)), ("depth_mask", C.POINTER(ViewDepthMask)), ("ssim", C.POINTER(ViewSsim)),
                ("camera_grad", C.POINTER(ViewCameraGrad)), ("intrinsics", C.POINTER(ViewIntrinsics)),
                ("median", C.POINTER(ViewMedian)), ("normal", C.POINTER(ViewNormal)), ("ortho", C.POINTER(C.c_int)),
                ("fisheye", C.POINTER(ViewFisheye)), ("distortion", C.POINTER(ViewDistortion)), ("flow", C.POINTER(ViewFlow)),
                ("flow_next", C.POINTER(CloudFlow)), ("antialiasing", C.c_int), ("planar_depth", C.c_int)]


class ViewLift(C.Structure):
    """mirror of `mgs_view_lift` (include/mgs_rasterizer.h): the 2D map [C,H,W] one view lifts onto the Gaussians"""
    _fields_ = [("map", C.c_void_p)]


class Cloud(C.Structure):
    """mirror of `mgs_cloud` (include/mgs_rasterizer.h)"""
    _fields_ = [("P", C.c_int)] + [(n, C.c_void_p) for n in (
        "means3D", "shs", "colors_precomp", "feature", "opacities", "scales", "rotations", "cov3D_precomp",
        "dL_dmean3D", "dL_dopacity", "dL_dcolor", "dL_dfeature", "dL_dcov3D", "dL_dsh", "dL_dscale", "dL_drot")]


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    path = _build.build()
    if not os.path.exists(path):
        raise ImportError(f"manigaussian_b200: CUDA library missing at {path}")
    L = C.CDLL(path)
    L.mgs_abi_version.restype = C.c_int
    L.mgs_last_error.restype = C.c_char_p
    for name in ("mgs_geometry_state_bytes", "mgs_binning_state_bytes", "mgs_backward_scratch_bytes", "mgs_camera_grad_scratch_bytes",
                 "mgs_geometry_state_bytes_normal", "mgs_backward_scratch_bytes_normal"):
        getattr(L, name).restype = C.c_size_t
        getattr(L, name).argtypes = [C.c_int]
    L.mgs_image_state_bytes.restype = C.c_size_t
    L.mgs_image_state_bytes.argtypes = [C.c_int, C.c_int]
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    L.mgs_forward.restype = C.c_int
    L.mgs_forward.argtypes = [ALLOC_FN, vp, ALLOC_FN, vp, ALLOC_FN, vp,
                              i, i, i, i,            # P D M F
                              vp, i, i,              # background, width, height
                              vp, vp, vp, vp,        # means3D shs colors feature
                              vp, vp, f, vp,         # opacities scales scale_modifier rotations
                              vp, vp, vp, vp,        # cov3D_precomp viewmatrix projmatrix cam_pos
                              f, f, i,               # tan_fovx tan_fovy prefiltered
                              vp, vp, vp, vp,        # out_color out_feature out_depth radii
                              i, vp]                 # debug stream
    L.mgs_forward_begin.restype = C.c_int
    L.mgs_forward_begin.argtypes = [ALLOC_FN, vp, ALLOC_FN, vp, i, i, i, i, i,
                                    vp, vp, vp, vp, vp, f, vp, vp, vp, vp, vp, f, f, vp, vp, i, vp]
    L.mgs_backward.restype = C.c_int
    L.mgs_backward.argtypes = [i, i, i, i, i,        # P D M F R
                               vp, i, i,             # background width height
                               vp, vp, vp, vp,       # means3D shs colors feature
                               vp, f, vp, vp,        # scales scale_modifier rotations cov3D_precomp
                               vp, vp, vp, f, f,     # viewmatrix projmatrix campos tan_fovx tan_fovy
                               vp, vp, vp, vp,       # radii geom binning image
                               vp, vp, vp,           # dL_dpix dL_dpix_F dL_dpix_depth
                               vp, vp, vp, vp, vp,   # dL_dmean2D dL_dconic dL_dopacity dL_dcolor dL_dfeature
                               vp, vp, vp, vp, vp,   # dL_dmean3D dL_dcov3D dL_dsh dL_dscale dL_drot
                               vp, i, i, vp]         # scratch accumulate debug stream
    opts = C.POINTER(RenderOptions)
    L.mgs_forward_views.restype = C.c_int
    L.mgs_forward_views.argtypes = [i, C.POINTER(View), opts, i, i, i, i,  # V views options P D M F
                                    vp, vp, vp, vp,                     # means3D shs colors feature
                                    vp, vp, f, vp, vp,                  # opacities scales scale_modifier rotations cov3D_precomp
                                    i, i, vp]                           # prefiltered debug join_stream
    L.mgs_backward_views.restype = C.c_int
    L.mgs_backward_views.argtypes = [i, C.POINTER(View), opts, i, i, i, i,  # V views options P D M F
                                     vp, vp, vp, vp,                    # means3D shs colors feature
                                     vp, f, vp, vp,                     # scales scale_modifier rotations cov3D_precomp
                                     vp, vp, vp, vp, vp, vp, vp, vp,    # dL: mean3D opacity color feature cov3D sh scale rot
                                     i, i, i, i, vp]                    # shared_mean2D accumulate stages debug join_stream
    L.mgs_forward_clouds.restype = C.c_int
    L.mgs_forward_clouds.argtypes = [i, C.POINTER(Cloud), C.POINTER(C.c_int), C.POINTER(View),  # B clouds view_offsets views
                                     opts, i, i, i, f,                  # options D M F scale_modifier
                                     i, i, vp]                          # prefiltered debug join_stream
    L.mgs_backward_clouds.restype = C.c_int
    L.mgs_backward_clouds.argtypes = [i, C.POINTER(Cloud), C.POINTER(C.c_int), C.POINTER(View),  # B clouds view_offsets views
                                      opts, i, i, i, f,                 # options D M F scale_modifier
                                      i, i, vp]                         # accumulate debug join_stream
    L.mgs_lift_views.restype = C.c_int
    L.mgs_lift_views.argtypes = [i, C.POINTER(View), C.POINTER(ViewLift), i, C.POINTER(ViewIntrinsics),  # V views lift aa intr
                                 C.POINTER(C.c_int), C.POINTER(ViewFisheye), C.POINTER(ViewDistortion),  # ortho fisheye distortion
                                 i, i, i, i,                        # P D M C
                                 vp, vp, vp,                        # means3D shs colors
                                 vp, vp, f, vp, vp,                 # opacities scales scale_modifier rotations cov3D_precomp
                                 vp, vp, i, vp]                     # out_lifted out_weight debug join_stream
    L.mgs_visibility_scratch_bytes.restype = C.c_size_t
    L.mgs_visibility_scratch_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    L.mgs_visibility_views.restype = C.c_int
    L.mgs_visibility_views.argtypes = [i, C.POINTER(View), i, C.POINTER(ViewIntrinsics),  # V views aa intr
                                       C.POINTER(C.c_int), C.POINTER(ViewFisheye), C.POINTER(ViewDistortion),  # ortho fisheye distortion
                                       i, i, i, i, vp,                  # P D M Q points
                                       vp, vp, vp,                      # means3D shs colors
                                       vp, vp, f, vp, vp,               # opacities scales scale_modifier rotations cov3D_precomp
                                       vp, vp, vp, vp, i, vp]           # out_uv out_depth out_in_view out_T debug join_stream
    L.mgs_visibility_backward_scratch_bytes.restype = C.c_size_t
    L.mgs_visibility_backward_scratch_bytes.argtypes = [C.c_int, C.c_int]
    L.mgs_visibility_views_backward.restype = C.c_int
    L.mgs_visibility_views_backward.argtypes = L.mgs_visibility_views.argtypes[:20] + [
        vp, vp, vp, vp,                  # out_T dL_dT dL_duv dL_ddepth
        vp, vp, vp, vp, vp, vp,          # dL_dpoints dL_dmean3D dL_dopacity dL_dscale dL_drot dL_dcov3D
        C.POINTER(ViewCameraGrad), i, vp]  # cam debug join_stream
    L.mgs_camera_rays_scratch_bytes.restype = C.c_size_t
    L.mgs_camera_rays_scratch_bytes.argtypes = [C.c_int]
    L.mgs_camera_rays.restype = C.c_int
    L.mgs_camera_rays.argtypes = [i, C.POINTER(View), C.POINTER(ViewIntrinsics),  # V views intr
                                  C.POINTER(C.c_int), C.POINTER(ViewFisheye), C.POINTER(ViewDistortion),  # ortho fisheye distortion
                                  i, vp, vp, vp, vp, i, vp]  # Q pixels out_origin out_direction out_valid debug stream
    L.mgs_camera_rays_backward.restype = C.c_int
    L.mgs_camera_rays_backward.argtypes = L.mgs_camera_rays.argtypes[:8] + [
        vp, vp, vp, C.POINTER(ViewCameraGrad), i, vp]  # dL_dorigin dL_ddirection dL_dpixels cam debug stream
    L.mgs_knn_state_bytes.restype = C.c_size_t
    L.mgs_knn_state_bytes.argtypes = [C.c_int, C.c_int]
    L.mgs_knn.restype = C.c_int
    L.mgs_knn.argtypes = [vp, i, i, i, vp, vp, vp, vp, i, vp]  # state N Q k points queries out_index out_dist2 debug stream
    L.mgs_neighbour_reg_state_bytes.restype = C.c_size_t
    L.mgs_neighbour_reg_state_bytes.argtypes = [C.c_int, C.c_int]
    L.mgs_neighbour_reg.restype = C.c_int
    L.mgs_neighbour_reg.argtypes = [vp, i, i, vp, vp, vp, vp, vp, vp,  # state P k xyz rot xyz_next rot_next index weight
                                    vp, i, vp]                         # out_loss debug stream
    L.mgs_neighbour_reg_backward.restype = C.c_int
    L.mgs_neighbour_reg_backward.argtypes = [vp, i, i, vp, vp, vp, vp, vp, vp,  # state P k xyz rot xyz_next rot_next index weight
                                             vp, vp, vp, vp, vp, i, vp]         # dL_dloss dL_d{xyz,rot,xyz_next,rot_next} debug stream
    L.mgs_deform_state_bytes.restype = C.c_size_t
    L.mgs_deform_state_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    L.mgs_deform.restype = C.c_int
    L.mgs_deform.argtypes = [vp, i, i, i, vp, vp, vp, vp, vp, vp, vp,  # state P N k xyz rot node_xyz node_rot node_t index weight
                             vp, vp, i, vp]                          # out_xyz out_rot debug stream
    L.mgs_deform_backward.restype = C.c_int
    L.mgs_deform_backward.argtypes = L.mgs_deform.argtypes[:11] + [
        vp, vp,                  # dL_dout_xyz dL_dout_rot
        vp, vp, vp, vp, vp, vp,  # dL_d{xyz,rot,node_xyz,node_rot,node_t,weight}
        i, vp]                   # debug stream
    L.mgs_fps_state_bytes.restype = C.c_size_t
    L.mgs_fps_state_bytes.argtypes = [C.c_int, C.c_int]
    L.mgs_fps.restype = C.c_int
    L.mgs_fps.argtypes = [vp, i, i, i, vp, vp, vp,  # state B P n points lengths start
                          vp, vp, i, vp]            # out_index out_dist2 debug stream
    L.mgs_mcmc_state_bytes.restype = C.c_size_t
    L.mgs_mcmc_state_bytes.argtypes = [C.c_int]
    fpp, ip = C.POINTER(C.c_void_p), C.POINTER(C.c_int)
    L.mgs_mcmc_relocate.restype = C.c_int
    L.mgs_mcmc_relocate.argtypes = [vp, i, i, f, vp, vp, vp, vp,  # state P_old P min_opacity means quats log_scales opacity_logit
                                    i, fpp, ip, i, fpp, ip,       # num_rows rows row_widths num_moments moments moment_widths
                                    vp, vp, vp, i, vp]            # rng out_source out_relocated debug stream
    L.mgs_mcmc_perturb.restype = C.c_int
    L.mgs_mcmc_perturb.argtypes = [i, vp, vp, vp, vp, vp, vp, i, vp]  # P means quats log_scales opacity_logit scale rng debug stream
    d = C.c_double
    L.mgs_densify_stats.restype = C.c_int
    L.mgs_densify_stats.argtypes = [i, i, vp, vp, ip, f, vp,  # V P viewspace_grad radii sizes scale scale_device
                                    vp, vp, vp, i, vp]        # grad2d count radius debug stream
    L.mgs_densify_state_bytes.restype = C.c_size_t
    L.mgs_densify_state_bytes.argtypes = [C.c_int]
    L.mgs_densify_count.restype = C.c_int
    L.mgs_densify_count.argtypes = [vp, i, vp, vp, vp, vp, vp,  # state P log_scales opacity_logit grad2d count radius
                                    d, f, d, f,                 # scene_scale grad_threshold grow_scale3d grow_scale2d
                                    d, d, f, i,                 # prune_opacity prune_scale3d prune_scale2d prune_too_big
                                    vp, i, vp]                  # out_counts debug stream
    L.mgs_densify_emit.restype = C.c_int
    L.mgs_densify_emit.argtypes = [vp, i, i, vp, vp, vp, vp,    # state P n_new means quats log_scales opacity_logit
                                   i, fpp, ip, i, fpp, ip,      # num_rows rows row_widths num_moments moments moment_widths
                                   vp, vp, vp, vp, fpp, fpp,    # new_{means,quats,log_scales,opacity_logit,rows,moments}
                                   vp, vp, i, vp]               # rng out_source debug stream
    L.mgs_tsdf_fuse.restype = C.c_int
    L.mgs_tsdf_fuse.argtypes = [i, C.POINTER(View), C.POINTER(ViewIntrinsics),  # V views intr
                                C.POINTER(C.c_int), C.POINTER(ViewFisheye), C.POINTER(ViewDistortion),  # ortho fisheye distortion
                                vp, i, vp, C.POINTER(C.c_double),  # depth C color bounds
                                i, i, i, f, vp, vp, vp, i, vp]     # X Y Z trunc tsdf weight color_volume debug stream
    L.mgs_marching_cubes_state_bytes.restype = C.c_size_t
    L.mgs_marching_cubes_state_bytes.argtypes = [i, i, i]
    L.mgs_marching_cubes_count.restype = C.c_int
    L.mgs_marching_cubes_count.argtypes = [vp, i, i, i, vp, vp, f, vp, i, vp]  # state X Y Z values weight level out_counts debug stream
    L.mgs_marching_cubes_emit.restype = C.c_int
    L.mgs_marching_cubes_emit.argtypes = [vp, i, i, i, vp, f, C.POINTER(C.c_double), i, vp,  # state X Y Z values level bounds C color
                                          vp, vp, vp, i, vp]  # out_vertices out_faces out_colors debug stream
    L.mgs_field_query.restype = C.c_int
    L.mgs_field_query.argtypes = [ALLOC_FN, vp, ALLOC_FN, vp, i, i, i,    # state and pair allocators, Q P C
                                  vp, vp, vp, vp, vp, vp, i,            # points means3D scales rotations opacities features channel_first
                                  vp, vp, i, vp]                        # out_density out_features debug stream
    L.mgs_field_query_backward.restype = C.c_int
    L.mgs_field_query_backward.argtypes = [vp, vp, i, i, i,             # state pair_state Q P C
                                           vp, vp, vp, vp, i, vp, vp,   # points scales rotations features channel_first dL_ddensity dL_dout_features
                                           vp, vp, vp, vp, vp, vp,      # dL: points means3D scales rotations opacities feature
                                           i, vp]                       # debug stream
    L.mgs_loss_heads.restype = C.c_int
    L.mgs_loss_heads.argtypes = [i, i, i, vp, vp, vp, vp, vp, vp, vp, vp]
    L.mgs_ssim.restype = C.c_int
    L.mgs_ssim.argtypes = [i, i, i, i, vp, vp, vp, vp, vp]                # V C H W x g ssim_terms loss_acc stream
    L.mgs_ssim_backward.restype = C.c_int
    L.mgs_ssim_backward.argtypes = [i, i, i, i, vp, vp, vp, vp, vp, vp, vp]  # V C H W x g ssim_terms scale cot_in cot_out stream
    L.mgs_mark_visible.restype = C.c_int
    L.mgs_mark_visible.argtypes = [i, vp, vp, vp, vp, vp]
    L.mgs_state_array.restype = C.c_int
    L.mgs_state_array.argtypes = [C.c_char_p, C.c_char_p, vp, i, i, C.POINTER(C.c_void_p)]
    L.mgs_profile_enable.argtypes = [i]
    L.mgs_profile_num_stages.restype = C.c_int
    L.mgs_profile_stage_name.restype = C.c_char_p
    L.mgs_profile_stage_name.argtypes = [i]
    L.mgs_profile_read.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_int)]
    L.mgs_activate.restype = C.c_int
    L.mgs_activate.argtypes = [i, i, vp, vp, vp, vp, vp, vp, vp, vp,   # P F means d_means rot d_rot scales d_scales opac feature
                               i, f, i, i, i,                           # scale_mode scale_max opacity_mode rot_normalize feature_normalize
                               vp, vp, vp, vp, vp, vp]                  # out_means out_rot out_scales out_opac out_feature stream
    L.mgs_activate_backward.restype = C.c_int
    L.mgs_activate_backward.argtypes = [i, i, vp, vp, vp, vp, vp, vp, vp, vp, i, f, i, i, i,
                                        vp, vp, vp, vp, vp,             # g_means g_rot g_scales g_opac g_feature
                                        vp, vp, vp, vp, vp, vp, vp, vp, # dL: means d_means rot d_rot scales d_scales opac feature
                                        vp]
    if L.mgs_abi_version() != 400:
        raise ImportError("manigaussian_b200: ABI version mismatch")
    _lib = L
    return L


EXPORTED_SYMBOLS = (
    "mgs_abi_version", "mgs_last_error", "mgs_geometry_state_bytes", "mgs_image_state_bytes",
    "mgs_binning_state_bytes", "mgs_backward_scratch_bytes", "mgs_forward", "mgs_forward_begin",
    "mgs_backward", "mgs_forward_views", "mgs_backward_views", "mgs_forward_clouds", "mgs_backward_clouds", "mgs_loss_heads",
    "mgs_ssim", "mgs_ssim_backward", "mgs_camera_grad_scratch_bytes",
    "mgs_geometry_state_bytes_normal", "mgs_backward_scratch_bytes_normal",
    "mgs_lift_views",
    "mgs_field_query", "mgs_field_query_backward",
    "mgs_visibility_scratch_bytes", "mgs_visibility_views",
    "mgs_visibility_backward_scratch_bytes", "mgs_visibility_views_backward",
    "mgs_camera_rays_scratch_bytes", "mgs_camera_rays", "mgs_camera_rays_backward",
    "mgs_knn_state_bytes", "mgs_knn",
    "mgs_neighbour_reg_state_bytes", "mgs_neighbour_reg", "mgs_neighbour_reg_backward",
    "mgs_deform_state_bytes", "mgs_deform", "mgs_deform_backward",
    "mgs_fps_state_bytes", "mgs_fps",
    "mgs_tsdf_fuse", "mgs_marching_cubes_state_bytes", "mgs_marching_cubes_count", "mgs_marching_cubes_emit",
    "mgs_mcmc_state_bytes", "mgs_mcmc_relocate", "mgs_mcmc_perturb",
    "mgs_densify_stats", "mgs_densify_state_bytes", "mgs_densify_count", "mgs_densify_emit",
    "mgs_activate", "mgs_activate_backward",
    "mgs_mark_visible", "mgs_state_array", "mgs_profile_enable", "mgs_profile_num_stages",
    "mgs_profile_stage_name", "mgs_profile_read",
)


def profile_enable(on=True):
    lib().mgs_profile_enable(int(bool(on)))


def profile_read():
    """{stage: (total_ms, launches)} since the last read."""
    L = lib()
    n = L.mgs_profile_num_stages()
    ms, cnt = (C.c_float * n)(), (C.c_int * n)()
    L.mgs_profile_read(ms, cnt)
    return {L.mgs_profile_stage_name(k).decode(): (float(ms[k]), int(cnt[k])) for k in range(n)}


def last_error():
    return lib().mgs_last_error().decode()


def check(rc, what):
    if rc < 0:
        raise RuntimeError(f"{what} failed ({rc}): {last_error()}")
    return rc

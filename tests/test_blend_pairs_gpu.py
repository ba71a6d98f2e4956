"""Both blend kernels, pair by pair, against the float64 blend reference (tests/blend_ref64.py).

Per scene: (a) every pair the reference puts surely inside the alpha >= 1/255 footprint is in its pixel's block list (the
cull in binning.cu / project.cu is sound); (b) our pixel masks equal the float64 decisions wherever no decision is
borderline, and block_nwalk ends at the block's last contributor; (c) with our masks as the decisions every pixel of
colour / features / depth / final_T / alpha is within its bound and n_contrib is exact; (d) every Gaussian's dL_dmeans2D,
dL_dopacity, dL_dcolors and dL_dfeature, and the blend-stage record's dL_dconic and dL_ddepth (read from the backward
scratch), is within its bound (F <= 32: the two-warp kernel; F > 32: blend_bwd_groups).  F = 12 and 28 take the padded
NFT = 2 / 4 paths, F = 16 the vectorised NFT = 2 one, and `ragged_off4` (F = 32 with the feature rows 4 bytes off a 16-byte
boundary) the NFT = 4 path without vector loads.

The scenes are built in screen space (`place`: target pixel centres and depths unprojected through the camera, shapes
given as 2D covariances through cov3D_precomp) to reach the kernels' structural edges, and each asserts the edge it was
built for.  The reference reads our projected records, so the placement only has to be approximate.

Measured on an H100 SXM 80 GB (400 W limit): worst raw ratio |x - ref64| / (u B) per scene (KAPPA = 4x the worst of
these and of the CPU-side ratios, per quantity):

| scene | colour | depth | final_T | alpha | features | dmeans2D | dopacity | dcolors | dfeature | dcov3D |
|---|---|---|---|---|---|---|---|---|---|---|
| lists (F 3 / 40) | 2.42 | 1.98 | 0.16 | 0.28 | 1.57 / 3.45 | 0.0079 | 0.043 | 0.12 | 0.24 | 0 |
| term32 / term64 | 2.56 | 2.57 | 0.37 | 0.49 | 0.76 | 0.0029 | 0.0054 | 0.017 | 0.043 | 0 |
| empty_run (F 3 / 67) | 0.64 | 0.61 | 0.31 | 0.36 | 1.26 | 0.0033 | 0.0058 | 0.056 | 0.10 | 0 |
| needles | 1.58 | 2.20 | 0.37 | 0.33 | 3.81 | 0.0033 | 0.0078 | 0.037 | 0.033 | 0 |
| offscreen | 0.79 | 0.88 | 0.21 | 0.21 | 1.43 | 0.0029 | 0.0053 | 0.029 | 0.036 | 0 |
| opacity (F 32 / 67) | 1.55 | 0.91 | 0.31 | 0.49 | 2.52 | 0.0028 | 0.049 | 0.19 | 0.17 | 0 |
| ragged (F 0-67) | 2.89 | 1.78 | 0.10 | 0.48 | 2.49 | 0.011 | 0.030 | 0.065 | 0.14 | 0 |
| ragged_f32 | 3.63 | 2.77 | 0.11 | 0.48 | 1.60 | 0.0054 | 0.010 | - | 0.072 | - |
| sh3_big | 1.48 | 1.23 | 0.19 | 0.22 | 1.60 | 0.0100 | 0.017 | - | 0.12 | - |
| ragged F 12 / 16 / 28, ragged_off4 (H100 80GB HBM3, 700 W) | 2.89 | 1.78 | 0.10 | 0.48 | 2.47 | 0.0051 | 0.016 | 0.065 | 0.14 | 0 |

gb dL_dconic / dL_ddepth (the blend-stage record) on the same H100 80GB HBM3 (700 W), all cases: at most 0.0060 / 0.15.

dcov3D: project_ref64.cov3d_grad, the raw ratio of the part the inherited conic bound does not cover, over u e.
No cull violation in any scene; borderline pixels 0.12 % (needles), 0.10 % (opacity), 0.09 % (ragged_f32), 0 elsewhere.
All 21 cases take about 15 s.
"""
import numpy as np
import pytest

import blend_ref64 as R64
import project_ref64 as P64
import util
from manigaussian_b200 import scenes

pytestmark = pytest.mark.gpu

# --------------------------------------------------------------------------- scene construction
def place(cam, px, py, z, cov2d, opac, F=3, seed=0, colors=None):
    """Gaussians whose means project near pixel (px, py) at view depth z with a screen-space covariance near cov2d
    ([n,2,2], before the 0.3 px^2 dilation)."""
    px, py, z = (np.asarray(v, np.float64).ravel() for v in (px, py, z))
    n = len(px)
    W, H = cam["W"], cam["H"]
    fx, fy = W / (2 * cam["tanfovx"]), H / (2 * cam["tanfovy"])
    V = cam["viewmatrix"].astype(np.float64).T          # world -> view
    xv = (px + 0.5 - W / 2.0) / fx * z
    yv = (py + 0.5 - H / 2.0) / fy * z
    pv = np.stack([xv, yv, z, np.ones(n)], 1)
    means = (np.linalg.inv(V) @ pv.T).T[:, :3]
    Rw = V[:3, :3]
    sv = np.zeros((n, 3, 3))
    sv[:, 0, 0] = cov2d[:, 0, 0] * (z / fx) ** 2
    sv[:, 1, 1] = cov2d[:, 1, 1] * (z / fy) ** 2
    sv[:, 0, 1] = sv[:, 1, 0] = cov2d[:, 0, 1] * z * z / (fx * fy)
    sv[:, 2, 2] = 1e-8
    sw = np.einsum("ji,njk,kl->nil", Rw, sv, Rw)
    cov3 = np.stack([sw[:, 0, 0], sw[:, 0, 1], sw[:, 0, 2], sw[:, 1, 1], sw[:, 1, 2], sw[:, 2, 2]], 1)
    rng = np.random.default_rng(seed)
    col = rng.random((n, 3)) if colors is None else colors
    feat = rng.normal(0, 1, (n, F)) if F else None
    return dict(means3D=means.astype(np.float32), opacities=np.asarray(opac, np.float32).reshape(n, 1),
                cov3D_precomp=cov3.astype(np.float32), colors_precomp=col.astype(np.float32),
                feature=None if feat is None else feat.astype(np.float32))


def iso(n, var):
    c = np.zeros((n, 2, 2))
    c[:, 0, 0] = c[:, 1, 1] = var
    return c


def _cat(parts):
    out = {}
    for k in parts[0]:
        vals = [p[k] for p in parts]
        out[k] = None if vals[0] is None else np.concatenate(vals, 0)
    return out


def _scene(W, H, parts, F, seed, bg=(0.25, 0.5, 0.75), view=0):
    cam = scenes.make_camera(W, H, view, 4)
    g = _cat([place(cam, **p, F=F, seed=seed + i) for i, p in enumerate(parts)])
    g.update(scales=None, rotations=None, shs=None, sh_degree=0)
    P = g["means3D"].shape[0]
    ct = scenes.make_cotangents(W, H, F, seed=seed, depth=True)
    ct["dL_dalpha"] = np.random.default_rng(seed + 1).normal(0, 1, (H, W)).astype(np.float32)
    return dict(cam=cam, g=g, ct=ct, bg=np.asarray(bg, np.float32), P=P, W=W, H=H, F=F)


LIST_LENGTHS = (1, 31, 32, 33, 63, 64, 65, 97, 200)


def scene_lists(F=3):
    """Block 3 (pixels x 8..15, y 4..7) of tile i holds exactly LIST_LENGTHS[i] translucent splats, all reaching every
    pixel of the block."""
    parts, W = [], 16 * 3
    for i, n in enumerate(LIST_LENGTHS):
        tx, ty = i % 3, i // 3
        rng = np.random.default_rng(100 + i)
        z = 1.0 + 0.5 * rng.permutation(n) / n
        parts.append(dict(px=np.full(n, tx * 16 + 11.0), py=np.full(n, ty * 16 + 5.0), z=z,
                          cov2d=iso(n, 3.7), opac=rng.uniform(0.03, 0.035, n)))
    return _scene(W, W, parts, F, 1)


def scene_terminate(k, F=3):
    """Every pixel terminates exactly at list entry k: wide splats (alpha nearly uniform over the image) of opacity
    o with (1 - o)^k > 1e-4 > (1 - o)^(k+1); the list goes on past the stop."""
    o = 1.0 - np.exp(np.log(1e-4) / (k + 0.5))
    n = k + 12
    z = 1.0 + 0.5 * np.arange(n) / n
    return _scene(32, 16, [dict(px=np.full(n, 15.5), py=np.full(n, 7.5), z=z, cov2d=iso(n, 300.0 ** 2),
                                opac=np.full(n, o))], F, 2)


def scene_empty_run(F=3, n_empty=75):
    """In block 0 of tile 0, n_empty listed entries with empty pixel masks between contributors in front and behind:
    faint splats (o = 1.3/255) centred between pixel centres, footprint radius ~0.4 px."""
    k = np.arange(n_empty)
    gx, gy = (k % 7) + 0.5, ((k // 7) % 3) + 0.5
    parts = [dict(px=np.full(3, 3.5), py=np.full(3, 1.5), z=np.array([0.8, 0.82, 0.84]), cov2d=iso(3, 40.0),
                  opac=np.full(3, 0.2)),
             dict(px=gx, py=gy, z=0.9 + 0.4 * k / n_empty, cov2d=iso(n_empty, 1e-4), opac=np.full(n_empty, 1.3 / 255)),
             dict(px=np.full(3, 3.5), py=np.full(3, 1.5), z=np.array([1.4, 1.42, 1.44]), cov2d=iso(3, 40.0),
                  opac=np.full(3, 0.2))]
    return _scene(32, 16, parts, F, 3)


def scene_needles(F=3):
    """45-degree needles whose conic has dq / ac around 1e-3 (the extent falls back to no cull below), plus round
    splats behind them."""
    n = 24
    ratio = np.geomspace(0.7e-3, 1.4e-3, n)
    lmin = 0.05
    lmaj = 4.0 * (lmin + 0.3) / ratio - 0.3
    c, s = np.cos(np.pi / 4), np.sin(np.pi / 4)
    cov = np.zeros((n, 2, 2))
    for i in range(n):
        Rm = np.array([[c, -s], [s, c]]) if i % 2 else np.array([[c, s], [-s, c]])
        cov[i] = Rm @ np.diag([lmaj[i], lmin]) @ Rm.T
    rng = np.random.default_rng(7)
    parts = [dict(px=rng.uniform(10, 86, n), py=rng.uniform(10, 86, n), z=1.0 + 0.3 * rng.random(n), cov2d=cov,
                  opac=rng.uniform(0.3, 0.9, n)),
             dict(px=rng.uniform(0, 96, 60), py=rng.uniform(0, 96, 60), z=1.5 + 0.3 * rng.random(60), cov2d=iso(60, 20.0),
                  opac=rng.uniform(0.1, 0.6, 60))]
    return _scene(96, 96, parts, F, 4)


def scene_offscreen(F=3):
    """Big splats whose means lie >= 1000 px off-screen and still reach the image."""
    pts = np.array([[-1000.0, 20.0], [1100.0, 10.0], [30.0, -1050.0], [20.0, 1080.0], [-1000.0, -1000.0]])
    parts = [dict(px=pts[:, 0], py=pts[:, 1], z=np.full(5, 2.0) + 0.01 * np.arange(5), cov2d=iso(5, 420.0 ** 2),
                  opac=np.full(5, 0.95)),
             dict(px=np.array([10.0, 40.0]), py=np.array([20.0, 5.0]), z=np.array([1.0, 1.1]), cov2d=iso(2, 30.0),
                  opac=np.array([0.5, 0.7]))]
    return _scene(64, 48, parts, F, 5)


OPACITIES = (np.nextafter(np.float32(1 / 255), np.float32(0)), np.float32(1 / 255),
             np.nextafter(np.float32(1 / 255), np.float32(1)), 0.98, 0.99, 0.995, 1.0, 1.5)


def scene_opacity(F=3):
    """One splat per opacity of OPACITIES, each in its own tile, with translucent splats behind them; an opaque stack
    of alpha ~ 0.98 layers; means on block and tile borders."""
    n = len(OPACITIES)
    tx = np.arange(n) % 4
    ty = np.arange(n) // 4
    # centred on a pixel centre: there power ~ 0, so the 1/255 decision turns on the opacity itself
    parts = [dict(px=tx * 16 + 8.0, py=ty * 16 + 8.0, z=np.full(n, 1.0), cov2d=iso(n, 6.0), opac=np.array(OPACITIES, np.float64)),
             dict(px=tx * 16 + 8.0, py=ty * 16 + 6.0, z=np.full(n, 1.4), cov2d=iso(n, 12.0), opac=np.full(n, 0.3)),
             # opaque stack (tile row 2)
             dict(px=np.full(8, 24.0), py=np.full(8, 40.0), z=1.0 + 0.02 * np.arange(8), cov2d=iso(8, 400.0),
                  opac=np.linspace(0.97, 0.985, 8)),
             # means on block / tile borders
             dict(px=np.array([15.5, 31.5, 47.5, 7.5]), py=np.array([3.5, 15.5, 35.5, 43.5]), z=np.full(4, 1.2),
                  cov2d=iso(4, 5.0), opac=np.full(4, 0.6))]
    return _scene(64, 48, parts, F, 6)


def scene_ragged(F):
    """A 61 x 37 image (W, H not multiples of 8 / 4) with random splats and splats on the ragged edge."""
    rng = np.random.default_rng(8)
    n = 400
    parts = [dict(px=rng.uniform(-5, 66, n), py=rng.uniform(-5, 42, n), z=0.8 + rng.random(n), cov2d=iso(n, 1.0) *
                  rng.uniform(0.5, 30, (n, 1, 1)), opac=1 / (1 + np.exp(-rng.normal(-1, 1.5, n)))),
             dict(px=np.array([60.0, 59.5, 30.0, 60.5]), py=np.array([20.0, 36.0, 36.5, 36.5]), z=np.full(4, 0.9),
                  cov2d=iso(4, 3.0), opac=np.full(4, 0.8))]
    return _scene(61, 37, parts, F, 9)


SCENES = {
    "lists": lambda F: scene_lists(F),
    "term32": lambda F: scene_terminate(32, F),
    "term64": lambda F: scene_terminate(64, F),
    "empty_run": lambda F: scene_empty_run(F),
    "needles": lambda F: scene_needles(F),
    "offscreen": lambda F: scene_offscreen(F),
    "opacity": lambda F: scene_opacity(F),
    "ragged": lambda F: scene_ragged(F),
    "ragged_off4": lambda F: dict(scene_ragged(F), feature_offset=1),
    # the existing random parity cases, so the per-element bars also cover realistic density
    "ragged_f32": lambda F: _random(dict(P=5000, W=200, H=120, F=F, seed=3, bg=(0.3, 0.6, 0.9))),
    "sh3_big": lambda F: _random(dict(P=1500, W=128, H=96, F=F, seed=5, sh_degree=3, scale0=0.04, bg=(1.0, 1.0, 1.0))),
}


def _random(kw):
    inp = util.make_inputs(**kw, depth=True)
    inp["ct"]["dL_dalpha"] = np.random.default_rng(kw["seed"] + 1).normal(0, 1, (kw["H"], kw["W"])).astype(np.float32)
    return inp


# --------------------------------------------------------------------------- running the kernels
class scratch_capture:
    """Keeps every backward view's blend_scratch alive (in call order) while in effect, so that its blend-stage records
    can be read after the call: `records(i, P)` = (gb [P,12], gn [P,4] or None) of the i-th view's scratch."""
    def __enter__(self):
        from manigaussian_b200 import rasterizer as R
        self.R, self.orig, self.views = R, R._backward_view, []

        def wrapped(*a, **kw):
            keep = self.orig(*a, **kw)
            self.views.append((keep[-1], bool(a[-1]) if len(a) > 9 else bool(kw.get("normal", False))))
            return keep
        R._backward_view = wrapped
        return self

    def __exit__(self, *exc):
        self.R._backward_view = self.orig

    def records(self, i, P):
        import torch
        torch.cuda.synchronize()
        sc, normal = self.views[i]
        out = []
        for name, n in (("gb", 12), ("gn", 4)):
            if name == "gn" and not normal:
                out.append(None)
                continue
            off = self.R.state_array("scratch", name, sc, P) - sc.data_ptr()
            out.append(sc[off:off + 4 * n * P].view(torch.float32).reshape(P, n).cpu().numpy())
        return out


def feature_tensor(feature, offset=0):
    """The feature rows as a CUDA tensor whose data start `offset` floats past a 16-byte boundary (offset 0: util._t)."""
    import torch
    if not offset:
        return util._t(feature)
    n = feature.size
    buf = torch.zeros(n + offset, dtype=torch.float32, device="cuda")
    buf[offset:] = torch.from_numpy(np.ascontiguousarray(feature, np.float32).ravel()).cuda()
    return buf[offset:].view(feature.shape)


def run_kernels(inp, planar=False, normal=False, median=False, depth_mask=False):
    """One forward and backward of the scene `inp`, and everything the checks read back.  The options (for
    tests/test_blend_planes_gpu.py): planar depth, the normal plane (cotangent inp["ct"]["dL_dnormal"]), the median depth
    (cotangent inp["ct"]["dL_dmedian"]) and the depth / mask heads (targets inp["dm_targets"], upstream gradients
    inp["dm_scale"]).  inp["lens"]: a distortion tuple for a distorted-pinhole view, inp["tanfov"] its (tan_fovx, tan_fovy)."""
    import torch
    from manigaussian_b200 import rasterizer as R
    t = util._t
    cam, g, ct = inp["cam"], inp["g"], inp["ct"]
    P, W, H, F = inp["P"], inp["W"], inp["H"], inp["F"]
    tfx, tfy = inp.get("tanfov", (cam["tanfovx"], cam["tanfovy"]))
    s = R.GaussianRasterizationSettings(H, W, tfx, tfy, t(inp["bg"]), 1.0, t(cam["viewmatrix"]),
                                        t(cam["projmatrix"]), g["sh_degree"], t(cam["campos"]), False, False, F > 0,
                                        distortion=inp.get("lens"), planar_depth=planar)
    feat = feature_tensor(g["feature"], inp.get("feature_offset", 0)) if F else None
    if feat is not None and inp.get("feature_offset"):
        assert feat.data_ptr() % 16 == 4 * inp["feature_offset"]
    args = (t(g["means3D"]), t(g["colors_precomp"]), feat, t(g["opacities"]), t(g["scales"]),
            t(g["rotations"]), 1.0, t(g["cov3D_precomp"]), t(g["shs"]), g["sh_degree"], F > 0)
    heads = dm = dm_scale = None
    if depth_mask:
        from manigaussian_b200.gaussian_renderer import _depth_mask_heads
        opts = dict(dtype=torch.float32, device="cuda")
        heads = (torch.zeros((1, 3, H, W), **opts), None, torch.empty((1, 3, H, W), **opts), None, torch.empty((1, 2), **opts))
        dm = _depth_mask_heads(t(inp["dm_targets"][0][None]), t(inp["dm_targets"][1][None]), 1, H, W, torch.device("cuda"))
        dm_scale = t(np.asarray(inp["dm_scale"], np.float32)[None])
    outs, streams = R.rasterize_views_raw([s], *args, return_depth=True, return_alpha=True, return_median=median,
                                          return_normal=normal, loss_heads=heads, depth_mask=dm)
    o = outs[0]
    Rn = o.num_rendered()
    assert not o.overflowed()
    cap = int(o[0])
    gc = [t(ct["dL_dcolor"])]
    gf = [t(ct["dL_dfeature"])] if F else None
    med = (o[-2 - int(normal)], o[-1 - int(normal)]) if median else None
    with scratch_capture() as cap_sc:
        grads = R.rasterize_views_backward_raw(
            [s], outs, streams, gc, gf, args[0], args[1], args[2], args[4], args[5], 1.0, args[7], args[8], g["sh_degree"], F > 0,
            grads_depth=[t(ct["dL_ddepth"])], grads_alpha=[t(ct["dL_dalpha"])],
            grads_median=[t(ct["dL_dmedian"])] if median else None, median_ids=[med[1]] if median else None,
            grads_normal=[t(ct["dL_dnormal"])] if normal else None, normals=[o[-1]] if normal else None,
            depth_mask=dm, depth_mask_scale=dm_scale)
    torch.cuda.synchronize()
    gb, gn = cap_sc.records(0, P)
    geomB, binB, imgB = o[4], o[5], o[6]
    T = ((W + 15) // 16) * ((H + 15) // 16)
    S = (cap + 11) & ~3

    def arr(which, name, state, a0, a1, dtype, count):
        off = R.state_array(which, name, state, a0, a1) - state.data_ptr()
        nbytes = count * torch.empty((), dtype=dtype).element_size()
        return state[off:off + nbytes].view(dtype).cpu().numpy()

    k = dict(W=W, H=H, F=F, R=Rn, color=o[1].cpu().numpy(), feature=o[2].cpu().numpy() if F else None,
             depth=o[7].cpu().numpy(), alpha=o[8].cpu().numpy())
    k["means2D"] = arr("geometry", "means2D", geomB, P, 0, torch.float32, 2 * P).reshape(P, 2)
    k["conic_opacity"] = arr("geometry", "conic_opacity", geomB, P, 0, torch.float32, 4 * P).reshape(P, 4)
    k["rgbd"] = arr("geometry", "rgbd", geomB, P, 0, torch.float32, 4 * P).reshape(P, 4)
    k["point_list"] = arr("binning", "point_list", binB, cap, 0, torch.int32, Rn).view(np.uint32)
    k["block_bits"] = arr("binning", "block_bits", binB, cap, 0, torch.uint8, Rn)
    k["block_lists"] = arr("binning", "block_lists", binB, cap, 0, torch.int32, 8 * S).view(np.uint32).reshape(8, S)
    k["pixel_masks"] = arr("binning", "pixel_masks", binB, cap, 0, torch.int32, 8 * S).view(np.uint32).reshape(8, S)
    k["ranges"] = arr("image", "ranges", imgB, W, H, torch.int32, 2 * T).view(np.uint32).reshape(T, 2)
    k["block_count"] = arr("image", "block_count", imgB, W, H, torch.int32, 8 * T).view(np.uint32).reshape(T, 8)
    k["block_nwalk"] = arr("image", "block_nwalk", imgB, W, H, torch.int32, 8 * T).view(np.uint32).reshape(T, 8)
    k["final_T"] = arr("image", "final_T", imgB, W, H, torch.float32, W * H).reshape(H, W)
    k["n_contrib"] = arr("image", "n_contrib", imgB, W, H, torch.int32, W * H).reshape(H, W)
    names = ("dL_dmeans2D", "dL_dcolors", "dL_dfeature", "dL_dopacity")
    for n, v in zip(names, grads[:4]):
        k[n] = None if v is None else v.cpu().numpy()
    k["radii"] = o[3].cpu().numpy()
    k["gb"], k["gn"] = gb, gn
    k["dL_dmeans3D"] = grads[4].cpu().numpy()
    if planar or normal:
        k["nrm"] = arr("geometry", "nrm", geomB, P, 0, torch.float32, 4 * P).reshape(P, 4)
    if normal:
        k["normal"] = o[-1].cpu().numpy()
    if median:
        k["median_depth"], k["median_id"] = med[0].cpu().numpy(), med[1].cpu().numpy()
    if depth_mask:
        k["dm_planes"] = [None if x is None else x[0].cpu().numpy() for x in dm[2:5]]
        k["dm_acc"] = dm[5][0].cpu().numpy()
    k["dL_dcov3D"] = None if grads[5] is None else grads[5].cpu().numpy()
    return k


def state_of(inp, k):
    g, ct = inp["g"], inp["ct"]
    return dict(W=k["W"], H=k["H"], ranges=k["ranges"], point_list=k["point_list"], means2D=k["means2D"],
                conic_opacity=k["conic_opacity"], colors=k["rgbd"][:, :3], depth=k["rgbd"][:, 3],
                feature=g["feature"] if k["F"] else None, bg=inp["bg"], g_color=ct["dL_dcolor"],
                g_feature=ct["dL_dfeature"] if k["F"] else None, g_depth=ct["dL_ddepth"], g_alpha=ct["dL_dalpha"])


def _where_gaussian(k, gid, n=3):
    """(tile, list position, block, block-list index, chunk) of the first block-list entries of Gaussian gid."""
    out = []
    for tile in range(k["ranges"].shape[0]):
        r0, r1 = (int(v) for v in k["ranges"][tile])
        hit = np.nonzero(k["point_list"][r0:r1] == gid)[0]
        for pos in hit:
            for s in range(8):
                cnt = int(k["block_count"][tile, s])
                e = np.nonzero(k["block_lists"][s, r0:r0 + cnt] == pos)[0]
                if len(e):
                    out.append(dict(tile=tile, pos=int(pos), block=s, entry=int(e[0]), chunk=int(e[0]) // 32,
                                    nwalk=int(k["block_nwalk"][tile, s])))
                    if len(out) >= n:
                        return out
    return out


def _where_pixel(k, x, y):
    gx = (k["W"] + 15) // 16
    tile = (y // 16) * gx + x // 16
    s, bit = R64.pixel_block_bit(x % 16, y % 16)
    nc = int(k["n_contrib"][y, x])
    return dict(x=int(x), y=int(y), tile=int(tile), block=int(s), bit=int(bit), n_contrib=nc,
                nwalk=int(k["block_nwalk"][tile, s]), chunk_of_last=(None if nc == 0 else int(nc - 1) // 32))


def _check(name, got, ref, B, where, report):
    """Worst ratio to the bound (KAPPA of the name's last word) into `report`, with the raw ratio |x - ref| / (u B)."""
    q = name.split()[-1]
    r = R64.ratio(got, ref, B, q)
    report[name] = float(r.max()) if r.size else 0.0
    report[name + " raw"] = report[name] * R64.KAPPA[q]
    if r.size and not r.max() <= 1.0:
        idx = np.argsort(r.ravel())[::-1][:5]
        rows = []
        for i in idx:
            u = np.unravel_index(i, r.shape)
            rows.append((u, float(np.asarray(got)[u]), float(ref[u]), float(r[u]), where(u)))
        return f"{name}: {int((r > 1).sum())} elements out of bound; worst: {rows}"
    return None


# --------------------------------------------------------------------------- the test
CASES = [("lists", 3), ("lists", 40), ("term32", 0), ("term64", 32), ("empty_run", 3), ("empty_run", 67),
         ("needles", 3), ("offscreen", 3), ("opacity", 32), ("opacity", 67), ("ragged", 0), ("ragged", 3), ("ragged", 12),
         ("ragged", 16), ("ragged", 28), ("ragged", 32), ("ragged_off4", 32), ("ragged", 40), ("ragged", 67), ("ragged_f32", 32),
         ("sh3_big", 8)]


@pytest.mark.parametrize("scene,F", CASES, ids=[f"{s}-F{f}" for s, f in CASES])
def test_blend_pairs(scene, F):
    inp = SCENES[scene](F)
    k = run_kernels(inp)
    st = state_of(inp, k)
    ours, ref, problems, report = check_blend(k, st, inp)
    print(f"[{scene} F={F}] " + " ".join(f"{a}={b:.3g}" for a, b in report.items()))
    _assert_edge(scene, k, st, ours)
    problems = [p for p in problems if p]
    assert not problems, "\n".join(problems)


def check_blend(k, st, inp, depth="depth", cov3d=True, records=True):
    """Checks (a) to (d) of one render `k` (run_kernels) against the reference state `st`.  Returns (our masks, the reference's
    blend(), the list of problems (None for a passed check), the report of worst ratios).  depth: the KAPPA entry of the depth
    plane; cov3d: also check dL_dcov3D (cov3D_precomp renders through a pinhole view); records: also check the blend-stage
    record's dL_dconic and dL_ddepth."""
    F = k["F"]
    W, H = k["W"], k["H"]
    T = k["ranges"].shape[0]
    ours = R64.masks_from_blocks(st, k["block_lists"], k["pixel_masks"], k["block_nwalk"])
    problems, report = [], {}
    cull_bad, border_px, mask_bad, npix = [], 0, [], 0
    for t in range(T):
        r0, r1 = (int(v) for v in k["ranges"][t])
        L = r1 - r0
        px, py, inside = R64.tile_pixels(W, H, t)
        lx, ly = np.arange(256) % 16, np.arange(256) // 16
        s, _ = R64.pixel_block_bit(lx, ly)
        if L == 0:  # an empty tile: nothing to decide, and no block walks
            npix += int(inside.sum())
            assert all(int(k["block_nwalk"][t, b]) == 0 for b in range(8) if (inside & (s == b)).any()), t
            continue
        d = R64.decide(st, t)
        bits = k["block_bits"][r0:r1].astype(np.int64)
        listed = ((bits[None, :] >> s[:, None]) & 1).astype(bool)
        # (a) cull soundness
        viol = d["foot_in"] & ~listed
        for p, j in zip(*np.nonzero(viol)):
            cull_bad.append(dict(tile=t, x=int(px[p]), y=int(py[p]), block=int(s[p]), pos=int(j),
                                 gid=int(k["point_list"][r0 + j]), power=float(d["pairs"]["power"][p, j]),
                                 alpha=float(d["pairs"]["alpha"][p, j])))
        # (b) pixel masks vs the float64 decisions, up to each pixel's first borderline decision
        fb = d["first_border"]
        npix += int(inside.sum())
        border_px += int((inside & (fb < L)).sum())
        known = np.arange(L)[None, :] < fb[:, None]
        bad = known & (ours[t] != d["mask"]) & inside[:, None]
        for p, j in list(zip(*np.nonzero(bad)))[:20]:
            mask_bad.append(dict(tile=t, x=int(px[p]), y=int(py[p]), block=int(s[p]), pos=int(j), ours=bool(ours[t][p, j])))
        # block_nwalk = the block's last contributor
        for b in range(8):
            nw = int(k["block_nwalk"][t, b])
            pix = inside & (s == b)
            if not pix.any():
                continue
            last = int(k["n_contrib"][py[pix], px[pix]].max())
            if nw == 0:
                assert last == 0, (t, b)
            else:
                assert int(k["block_lists"][b, r0 + nw - 1]) + 1 == last, (t, b, nw, last)
    report["cull_violations"] = len(cull_bad)
    report["borderline_pixel_share"] = border_px / max(npix, 1)
    if cull_bad:
        problems.append(f"(a) {len(cull_bad)} surely-contributing pairs missing from their block list: {cull_bad[:5]}")
    if mask_bad:
        problems.append(f"(b) pixel masks differ from the float64 decisions: {mask_bad[:5]}")
    assert report["borderline_pixel_share"] <= 0.02, report
    # (c) forward, per element, with our masks as the decisions
    ref = R64.blend(st, ours)
    if not np.array_equal(ref["n_contrib"], k["n_contrib"].astype(np.int64)):
        y, x = np.nonzero(ref["n_contrib"] != k["n_contrib"])
        problems.append(f"(c) n_contrib differs at {[_where_pixel(k, a, b) for a, b in zip(x[:5], y[:5])]}")
    pix = lambda u: _where_pixel(k, u[-1], u[-2])  # noqa: E731
    for name, got in (("color", k["color"]), ("depth", k["depth"]), ("final_T", k["final_T"]), ("alpha", k["alpha"])) + \
            ((("feature", k["feature"]),) if F else ()):
        q = depth if name == "depth" else name
        problems.append(_check("(c) " + q, got, ref[name], ref[name + "_B"], pix, report))
    # (d) backward, per Gaussian
    gw = lambda u: _where_gaussian(k, u[0])  # noqa: E731
    if not st.get("planar"):  # with planar depth the returned dL_dmeans2D also holds the quad's share through e
        problems.append(_check("(d) dL_dmeans2D", k["dL_dmeans2D"][:, :2], ref["dL_dmeans2D"], ref["dL_dmeans2D_B"], gw, report))
    problems.append(_check("(d) dL_dopacity", k["dL_dopacity"][:, 0], ref["dL_dopacity"], ref["dL_dopacity_B"], gw, report))
    if k["dL_dcolors"] is not None:
        problems.append(_check("(d) dL_dcolors", k["dL_dcolors"], ref["dL_dcolors"], ref["dL_dcolors_B"], gw, report))
    if F:
        problems.append(_check("(d) dL_dfeature", k["dL_dfeature"], ref["dL_dfeature"], ref["dL_dfeature_B"], gw, report))
    if records:
        # the blend-stage record (gb) itself: dL_dconic {a, b, c} in slots 2..4, dL_ddepth in slot 9
        problems.append(_check("(d) gb dL_dconic", k["gb"][:, [2, 3, 4]], ref["dL_dconic"], ref["dL_dconic_B"], gw, report))
        problems.append(_check("(d) gb dL_ddepth", k["gb"][:, 9], ref["dL_ddepth"], ref["dL_ddepth_B"], gw, report))
    if cov3d and k["dL_dcov3D"] is not None:
        # the conic gradients (GEMM 3's six moments) through the output the ABI returns for cov3D_precomp
        cam, g = inp["cam"], inp["g"]
        c3, bd = P64.cov3d_grad(ref, g, cam, live=k["radii"] > 0)
        ok = (k["radii"] > 0) & ~bd
        r = P64.raw_ratio(k["dL_dcov3D"][ok], tuple(np.broadcast_to(x, c3[0].shape)[ok] for x in c3))
        report["(d) dL_dcov3D raw"] = float(r.max()) if r.size else 0.0
        if r.size and r.max() > P64.KAPPA["dL_dcov3D"]:
            i = np.argsort(r.max(1))[::-1][:5]
            problems.append(f"(d) dL_dcov3D: {int((r > P64.KAPPA['dL_dcov3D']).any(1).sum())} Gaussians out of bound; worst "
                            f"{[(_where_gaussian(k, np.nonzero(ok)[0][j]), float(r[j].max())) for j in i]}")
    return ours, ref, problems, report


def _assert_edge(scene, k, st, ours):
    """The scene still reaches the edge it was built for."""
    cnt, nwalk = k["block_count"], k["block_nwalk"]
    if scene == "lists":
        for i, n in enumerate(LIST_LENGTHS):
            assert cnt[i, 3] == n and nwalk[i, 3] == n, (i, n, cnt[i, 3], nwalk[i, 3])
            r0 = int(k["ranges"][i][0])
            assert np.all(k["pixel_masks"][3, r0:r0 + n] != 0), (i, n)
    elif scene in ("term32", "term64"):
        want = 32 if scene == "term32" else 64
        assert np.all(k["n_contrib"] == want), np.unique(k["n_contrib"])
    elif scene == "empty_run":
        r0 = int(k["ranges"][0][0])
        nw = int(nwalk[0, 0])
        m = k["pixel_masks"][0, r0:r0 + nw]
        run = best = 0
        for v in m:
            run = run + 1 if v == 0 else 0
            best = max(best, run)
        assert best >= 70 and m[-1] != 0, (best, nw)
    elif scene == "needles":
        co = k["conic_opacity"].astype(np.float64)
        live = co[:, 0] > 0
        ac = co[:, 0] * co[:, 2]
        r = (ac - co[:, 1] ** 2) / np.where(live, ac, 1)
        assert np.any(live & (r > 1e-3) & (r < 1.1e-3)) and np.any(live & (r < 1e-3) & (r > 0.9e-3)), np.sort(r[live])[:30]
    elif scene == "offscreen":
        m2 = k["means2D"][:5]
        far = (m2[:, 0] < -1000) | (m2[:, 0] > k["W"] + 1000) | (m2[:, 1] < -1000) | (m2[:, 1] > k["H"] + 1000)
        assert far.sum() >= 3, m2
        # they contribute
        hit = np.zeros(st["means2D"].shape[0], bool)
        for t, m in enumerate(ours):
            r0, r1 = (int(v) for v in k["ranges"][t])
            hit[k["point_list"][r0:r1][m.any(0)]] = True
        assert hit[:5][far].all()
    elif scene == "opacity":
        clamped = False
        for t, m in enumerate(ours):
            p = R64._pairs(st, t)
            clamped |= bool(((p["o"] * p["G"] > R64.ALPHA_MAX) & m).any())
        assert clamped
        op = k["conic_opacity"][:len(OPACITIES), 3]
        assert np.array_equal(op, np.asarray(OPACITIES, np.float32))
        # 1/255 - ulp: alpha = min(0.99, o G) <= o < 1/255, it contributes nowhere; 1/255 and 1/255 + ulp contribute at
        # the pixel nearest their mean, unless the float64 decision there is borderline
        for gid in range(3):
            hits, border = 0, False
            for t, m in enumerate(ours):
                r0, r1 = (int(v) for v in k["ranges"][t])
                e = np.nonzero(k["point_list"][r0:r1] == gid)[0]
                if not len(e):
                    continue
                hits += int(m[:, e].sum())
                d = R64.decide(st, t)
                mx, my = np.rint(k["means2D"][gid]).astype(int)
                px, py, _ = R64.tile_pixels(k["W"], k["H"], t)
                c = np.nonzero((px == mx) & (py == my))[0]
                if len(c):
                    border |= bool(d["first_border"][c[0]] <= e[0])
                    hits_c = bool(m[c[0], e[0]])
                    if gid > 0:
                        assert hits_c or border, (gid, "does not contribute at its centre pixel")
            if gid == 0:
                assert hits == 0, "an opacity below 1/255 contributed"

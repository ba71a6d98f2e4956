"""The blend kernels' extra-column instantiations, pair by pair, against the float64 blend reference (tests/blend_ref64.py).

The normal plane (NRM), planar depth (PLN), the median depth (MED) and the depth / mask heads (DM) use columns 4..7 of the
{r,g,b,depth} tile or change the walker's prologue.  Each runs the scenes of tests/test_blend_pairs_gpu.py through checks
(a) to (d) there, and additionally every Gaussian's blend-stage records, read from the backward scratch: gb (dL_dmeans2D,
dL_dconic, dL_dopacity, dL_dcolors, dL_ddepth) and gn (dL/dn of the normal plane; planar depth's {sum w g px, sum w g py,
sum w g}).  The reference reads the kernels' own quads (geometry state "nrm").  The normal plane needs scales and rotations:
the scenes' covariances are factored into them.  DM: the heads' cotangent planes the forward wrote are folded into the depth
and alpha cotangents of the reference as the walker's prologue folds them (their values are pinned by
tests/test_depth_heads_gpu.py).  F = 12 and 16 are the NFT = 2 padded and vectorised paths, F > 32 the channel groups.

Far from the image origin: the `ragged` scene through a distortion-free distorted-pinhole view (a pinhole with a free
principal point) on a 2048 x 1536 canvas, its content moved by (1760, 1280) px -- a multiple of 16, so tiles and blocks
partition it as before -- with the focal length unchanged.  Checks (a) to (d) and the records hold with the KAPPA of the
near-origin scenes, and the per-Gaussian dL_dcov3D of the planar backward, against float64 autograd of the reference's
blend-stage gradients through the projection, has a worst error (over the norm of the Gaussian's planar part) at most 4x
that of the same scene at the origin.

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit): worst raw ratio |x - ref64| / (u B) per mode and scene (over its
F), KAPPA in blend_ref64 = 4x the worst near-origin value per quantity (normal 2.24, planar depth 2.17, planar median
0.656, dquad 0.244; dconic with the heads 0.0151 in an earlier run of DM term64, whose atomics summed in another order):

| mode | scene | color | depth | planar depth | normal | planar median | final_T | alpha | feature | dmeans2D | dconic | dconic (DM) | dopacity | dcolors | ddepth | dquad (gn) |
|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|
| NRM | lists | 2.42 | 1.98 | - | 2.04 | - | 0.158 | 0.283 | 1.57 | 0.00605 | 0.00117 | - | 0.0577 | 0.122 | 0.206 | 0.218 |
| NRM | term32 | 2.23 | 2.1 | - | 1.66 | - | 0.37 | 0.485 | - | 0.00243 | 0.000836 | - | 0.00158 | 0.00894 | 0.00625 | 0.00867 |
| NRM | term64 | 2.56 | 2.57 | - | 1.95 | - | 0.291 | 0.49 | 0.755 | 0.00182 | 0.00175 | - | 0.00503 | 0.018 | 0.0245 | 0.0188 |
| NRM | empty_run | 0.648 | 0.61 | - | 0.869 | - | 0.304 | 0.355 | 1.25 | 0.00202 | 0.0014 | - | 0.00488 | 0.0497 | 0.0131 | 0.0502 |
| NRM | needles | 1.5 | 2.22 | - | 2.24 | - | 0.349 | 0.329 | 3.75 | 0.00367 | 0.00157 | - | 0.00839 | 0.0373 | 0.0466 | 0.0398 |
| NRM | offscreen | 0.956 | 0.936 | - | 1.35 | - | 0.212 | 0.251 | 2.36 | 0.00242 | 0.00205 | - | 0.00877 | 0.0262 | 0.0211 | 0.0426 |
| NRM | opacity | 1.55 | 0.913 | - | 1.28 | - | 0.309 | 0.49 | 2.25 | 0.00231 | 0.00142 | - | 0.0139 | 0.125 | 0.136 | 0.111 |
| NRM | ragged | 2.89 | 1.78 | - | 1.94 | - | 0.11 | 0.477 | 2.23 | 0.00565 | 0.00214 | - | 0.0163 | 0.0734 | 0.144 | 0.145 |
| NRM+MED | ragged | 2.89 | 1.78 | - | 1.94 | - | 0.11 | 0.477 | 2.99 | 0.00512 | 0.00154 | - | 0.0167 | 0.0734 | 0.206 | 0.126 |
| PLN | lists | 2.42 | - | 1.88 | - | - | 0.158 | 0.283 | 1.57 | 0.00682 | 0.0021 | - | 0.0369 | 0.112 | 0.181 | 0.191 |
| PLN | term32 | 2.23 | - | 1.64 | - | - | 0.37 | 0.485 | - | 0.00301 | 0.0012 | - | 0.00151 | 0.00879 | 0.00648 | 0.00865 |
| PLN | term64 | 2.56 | - | 2.17 | - | - | 0.291 | 0.49 | 0.755 | 0.00191 | 0.00181 | - | 0.0054 | 0.018 | 0.0252 | 0.048 |
| PLN | empty_run | 0.643 | - | 0.455 | - | - | 0.305 | 0.356 | 1.26 | 0.00283 | 0.00181 | - | 0.00453 | 0.0594 | 0.0178 | 0.0412 |
| PLN | needles | 1.58 | - | 1.33 | - | - | 0.37 | 0.331 | 3.81 | 0.00323 | 0.00153 | - | 0.0079 | 0.0373 | 0.0383 | 0.0484 |
| PLN | offscreen | 0.788 | - | 0.621 | - | - | 0.212 | 0.21 | 2.33 | 0.00268 | 0.00208 | - | 0.00743 | 0.0296 | 0.0126 | 0.0356 |
| PLN | opacity | 1.55 | - | 0.673 | - | - | 0.309 | 0.49 | 2.25 | 0.00233 | 0.00153 | - | 0.0124 | 0.192 | 0.107 | 0.107 |
| PLN | ragged | 2.89 | - | 1.51 | - | - | 0.104 | 0.475 | 2.23 | 0.00502 | 0.00211 | - | 0.0143 | 0.0646 | 0.136 | 0.136 |
| PLN+MED+DM | ragged | 2.89 | - | 1.51 | - | 0.656 | 0.104 | 0.475 | 2.49 | 0.0103 | - | 0.00375 | 0.0274 | 0.0646 | 0.0726 | 0.11 |
| PLN+MED+DM | term64 | 2.56 | - | 2.17 | - | 0.00133 | 0.291 | 0.49 | - | 0.00351 | - | 0.0107 | 0.0602 | 0.0172 | 0.0036 | 0.0103 |
| DM | ragged | 2.89 | 1.78 | - | - | - | 0.104 | 0.475 | 2.47 | 0.0046 | - | 0.00139 | 0.0161 | 0.0646 | 0.0644 | - |
| DM | term64 | 2.56 | 2.57 | - | - | - | 0.291 | 0.49 | 0.487 | 0.0136 | - | 0.0108 | 0.0639 | 0.0172 | 0.0316 | - |
| PLN, distorted view, origin | ragged | 2.87 | - | 1.48 | - | - | 0.134 | 0.481 | 1.56 | 0.0097 | 0.00288 | - | 0.0361 | 0.113 | 0.0441 | 0.0684 |
| PLN, distorted view, +(1760, 1280) | ragged | 2.97 | - | 1.56 | - | - | 0.218 | 0.487 | 1.65 | 0.00907 | 0.00322 | - | 0.0317 | 0.0931 | 0.0996 | 0.0996 |

Chained planar gradient (test_planar_far_from_the_origin), worst per-Gaussian |dL_dcov3D - float64| / |planar part|, the
float64 side built from the kernels' own gb record plus the chain of the reference's dL/dquad (so the residual is the planar
path's error): 4.3e-4 at the origin, 3.9e-4 far from it (x 0.9; the bar is x 4), with gn formed relative to the mean in
block-local coordinates.  The gn records' worst raw ratio: 0.044 at the origin, 0.100 far from it.
"""
import numpy as np
import pytest

import blend_ref64 as R64
import planar_ref64 as PL64
import test_blend_pairs_gpu as BP

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fresh_capacities():
    from manigaussian_b200 import rasterizer as R
    R.reset_capacity_estimates()
    yield
    R.reset_capacity_estimates()


def scale_rotation(inp):
    """The scene with its cov3D_precomp factored into scales and rotations: eigendecomposition, scales = sqrt(eigenvalues),
    rotation = the eigenvectors with det +1 as a unit quaternion {r, x, y, z}."""
    from scipy.spatial.transform import Rotation
    g = dict(inp["g"])
    c = g["cov3D_precomp"].astype(np.float64)
    S = np.stack([np.stack([c[:, 0], c[:, 1], c[:, 2]], -1), np.stack([c[:, 1], c[:, 3], c[:, 4]], -1),
                  np.stack([c[:, 2], c[:, 4], c[:, 5]], -1)], -2)
    ev, V = np.linalg.eigh(S)
    V[np.linalg.det(V) < 0, :, 0] *= -1
    q = Rotation.from_matrix(V).as_quat()  # x, y, z, w
    g.update(scales=np.sqrt(np.maximum(ev, 1e-12)).astype(np.float32), rotations=q[:, [3, 0, 1, 2]].astype(np.float32),
             cov3D_precomp=None)
    return dict(inp, g=g)


def _with_cotangents(inp, seed, normal=False, median=False, depth_mask=False):
    rng = np.random.default_rng(seed)
    W, H = inp["W"], inp["H"]
    ct = dict(inp["ct"])
    if normal:
        ct["dL_dnormal"] = rng.normal(0, 1, (3, H, W)).astype(np.float32)
    if median:
        ct["dL_dmedian"] = rng.normal(0, 1, (H, W)).astype(np.float32)
    out = dict(inp, ct=ct)
    if depth_mask:
        tgt = rng.uniform(0.5, 2.0, (H, W)) * (rng.uniform(0, 1, (H, W)) > 0.2)
        out["dm_targets"] = (tgt.astype(np.float32), (rng.uniform(0, 1, (H, W)) > 0.5).astype(np.float32))
        out["dm_scale"] = (0.7, 1.3)
    return out


def reference_state(inp, k, planar=False, normal=False, depth_mask=False):
    """blend_ref64's state of the render k, with the quads, their cotangent planes and the heads' cotangents folded in."""
    st = BP.state_of(inp, k)
    if planar or normal:
        st["quad"] = k["nrm"]
        st["planar"] = planar
        if normal:
            st["g_quad"] = inp["ct"]["dL_dnormal"]
    if depth_mask:
        # depth_mask_cotangents (blend_bwd.cu), restated in fp32 so that the reference's cotangents are the kernels' own:
        # g_depth += s_d cot_depth, h += s_d cot_alpha_depth, h += s_m cot_alpha_mask (each one fused multiply-add),
        # s_d = scale_d / max(n, 1) with n the valid-pixel count the forward accumulated
        f = np.float32
        fma = lambda a, b, c: (a.astype(np.float64) * b + c).astype(f)  # noqa: E731  (the f32 product is exact in f64)
        cd, cad, cam = k["dm_planes"]
        sd = f(inp["dm_scale"][0]) / max(f(k["dm_acc"][1]), f(1.0))
        st["g_depth"] = fma(cd, sd, st["g_depth"].astype(f))
        st["g_alpha"] = fma(cam, f(inp["dm_scale"][1]), fma(cad, sd, st["g_alpha"].astype(f)))
    return st


def check_planes(inp, planar=False, normal=False, median=False, depth_mask=False, label=""):
    """Runs the kernels and checks (a) to (d) plus the records; returns (k, ref, report)."""
    k = BP.run_kernels(inp, planar=planar, normal=normal, median=median, depth_mask=depth_mask)
    st = reference_state(inp, k, planar, normal, depth_mask)
    ours, ref, problems, report = BP.check_blend(k, st, inp, depth="planar_depth" if planar else "depth", cov3d=False,
                                                 records=False)
    gw = lambda u: BP._where_gaussian(k, u[0])  # noqa: E731
    pix = lambda u: BP._where_pixel(k, u[-1], u[-2])  # noqa: E731
    if median:
        plane, B = R64.median_planar(st, k["median_id"], inp["ct"]["dL_dmedian"], ref)
        if planar:
            problems.append(BP._check("(c) median_planar", k["median_depth"], plane, B, pix, report))
        else:
            has = k["median_id"] >= 0
            assert np.array_equal(k["median_depth"][has], k["rgbd"][k["median_id"][has], 3])
    if normal:
        problems.append(BP._check("(c) normal", k["normal"], ref["quad"][:3], ref["quad_B"][:3], pix, report))
    # gb, element by element: {dmx, dmy, dca, dcb | dcc, dop, dr, dg | db, ddepth, 0, 0}
    gb = k["gb"]
    live = k["radii"] > 0
    problems.append(BP._check("(d) gb dL_dmeans2D", gb[:, :2], ref["dL_dmeans2D"], ref["dL_dmeans2D_B"], gw, report))
    problems.append(BP._check("(d) gb " + ("dL_dconic_heads" if depth_mask else "dL_dconic"), gb[:, 2:5], ref["dL_dconic"],
                              ref["dL_dconic_B"], gw, report))
    problems.append(BP._check("(d) gb dL_dcolors", gb[:, 6:9], ref["dL_dcolors"], ref["dL_dcolors_B"], gw, report))
    problems.append(BP._check("(d) gb dL_ddepth", gb[:, 9], ref["dL_ddepth"], ref["dL_ddepth_B"], gw, report))
    # dL_dopacity is stored as sum q / o (the kernels' dL/dopacity before the chain through the activation)
    problems.append(BP._check("(d) gb dL_dopacity", gb[live, 5], ref["dL_dopacity"][live], ref["dL_dopacity_B"][live],
                              lambda u: BP._where_gaussian(k, np.nonzero(live)[0][u[0]]), report))
    assert not gb[:, 10:].any()
    if planar or normal:
        problems.append(BP._check("(d) gn dL_dquad", k["gn"][:, :3], ref["dL_dquad"][:, :3], ref["dL_dquad_B"][:, :3], gw,
                                  report))
        assert not k["gn"][:, 3].any()
        assert np.abs(ref["dL_dquad"][:, :3]).max() > 0
    print(f"[{label}] " + " ".join(f"{a}={b:.3g}" for a, b in report.items()))
    return k, ref, [p for p in problems if p], report, ours, st


def _scene(scene, F, mode):
    inp = BP.SCENES[scene](F)
    if "NRM" in mode:
        inp = scale_rotation(inp)
    return _with_cotangents(inp, 40 + F, normal="NRM" in mode, median="MED" in mode, depth_mask="DM" in mode)


PLANE_SCENES = [("lists", 3), ("term32", 0), ("term64", 32), ("empty_run", 67), ("needles", 3), ("offscreen", 8),
                ("opacity", 40), ("ragged", 12), ("ragged", 16), ("ragged", 67)]
CASES = ([("NRM", s, f) for s, f in PLANE_SCENES] + [("NRM+MED", "ragged", 32), ("NRM+MED", "ragged", 67)] +
         [("PLN", s, f) for s, f in PLANE_SCENES] +
         [("PLN+MED+DM", "ragged", 3), ("PLN+MED+DM", "ragged", 40), ("PLN+MED+DM", "term64", 0)] +
         [("DM", "ragged", 0), ("DM", "ragged", 32), ("DM", "ragged", 67), ("DM", "term64", 3)])


@pytest.mark.parametrize("mode,scene,F", CASES, ids=[f"{m}-{s}-F{f}" for m, s, f in CASES])
def test_blend_planes(mode, scene, F):
    inp = _scene(scene, F, mode)
    k, ref, problems, report, ours, st = check_planes(inp, planar="PLN" in mode, normal="NRM" in mode, median="MED" in mode,
                                                      depth_mask="DM" in mode, label=f"{mode} {scene} F={F}")
    BP._assert_edge(scene, k, st, ours)
    if "DM" in mode:
        assert np.abs(k["dm_planes"][0]).max() > 0 and np.abs(k["dm_planes"][2]).max() > 0
    assert not problems, "\n".join(problems)


# --------------------------------------------------------------------------- far from the image origin
SHIFT = (1760, 1280)
FAR_W, FAR_H = 2048, 1536


def _placement(far, F=3):
    """The ragged scene (cov3D_precomp, planar depth) through a distortion-free distorted-pinhole view: at the origin (its own
    61 x 37 canvas, principal point at the centre) or moved by SHIFT on a FAR_W x FAR_H canvas, focal length unchanged; the
    pixel cotangents move with the content (zero elsewhere)."""
    inp = _with_cotangents(BP.SCENES["ragged"](F), 40 + F)
    W, H = inp["W"], inp["H"]
    cam = inp["cam"]
    cx, cy = (W - 1) / 2.0, (H - 1) / 2.0
    tfx, tfy = float(cam["tanfovx"]), float(cam["tanfovy"])
    if not far:
        return dict(inp, lens=(cx, cy) + (0.0,) * 8 + (float("inf"),), tanfov=(tfx, tfy))
    sx, sy = SHIFT
    ct = {}
    for name, v in inp["ct"].items():
        big = np.zeros(v.shape[:-2] + (FAR_H, FAR_W), np.float32)
        big[..., sy:sy + H, sx:sx + W] = v
        ct[name] = big
    return dict(inp, W=FAR_W, H=FAR_H, ct=ct, lens=(cx + sx, cy + sy) + (0.0,) * 8 + (float("inf"),),
                tanfov=(tfx * FAR_W / W, tfy * FAR_H / H))


def _view(inp):
    cam = inp["cam"]
    return dict(viewmatrix=np.asarray(cam["viewmatrix"], np.float64).reshape(-1),
                projmatrix=np.asarray(cam["projmatrix"], np.float64).reshape(-1), W=inp["W"], H=inp["H"],
                tanfovx=inp["tanfov"][0], tanfovy=inp["tanfov"][1], distortion=inp["lens"])


def chained_float64(inp, k, ref):
    """Per Gaussian, float64 autograd through the projection of the view of the kernels' own blend-stage record gb
    (dL/dmean2D, dL/dconic, dL/ddepth, taken as exact) and of the reference's dL/dquad: (dL_dmeans3D, dL_dcov3D), and the
    planar part alone (dL/dquad's chain).  What the kernels' result differs by is then the error of their quad gradients
    gn and of the planar terms of project_bwd, plus project_bwd's own rounding of the rest."""
    import torch
    view = _view(inp)
    live = k["radii"] > 0
    g = inp["g"]
    m = torch.tensor(g["means3D"], dtype=torch.float64, requires_grad=True)
    c6 = torch.tensor(g["cov3D_precomp"], dtype=torch.float64, requires_grad=True)
    S = PL64.packed_cov(c6)
    quad, conic = PL64.quads(m, None, None, view, cov3D=S)
    mu = PL64.screen_mean(m, view)
    vm = torch.tensor(view["viewmatrix"], dtype=torch.float64).reshape(4, 4).T
    z = m @ vm[2, :3] + vm[2, 3]
    lv = torch.tensor(live.astype(np.float64))[:, None]
    W, H = inp["W"], inp["H"]
    d = lambda x: torch.tensor(np.asarray(x, np.float64)) * lv  # noqa: E731
    gb = k["gb"].astype(np.float64)
    dm = d(gb[:, :2] / np.array([0.5 * W, 0.5 * H]))
    dc = d(gb[:, 2:5] * np.array([1.0, 2.0, 1.0]))  # the half-weight off-diagonal term
    # the reference's dL/dquad has e's share folded into a and b; quads() takes e as an output of its own
    dq = ref["dL_dquad"][:, :3].copy()
    dq[:, :2] += k["means2D"].astype(np.float64) * dq[:, 2:3]
    loss = ((mu * dm).sum() + (conic * dc).sum() + (z * d(gb[:, 9:10])[:, 0]).sum() + (quad * d(dq)).sum())
    gm, gc = torch.autograd.grad(loss, (m, c6))
    pm, pc = PL64.full_chain(g["means3D"], None, None, view, dq, live, cov3D=g["cov3D_precomp"])[:2]
    return gm.numpy(), gc.numpy(), pm, pc, live


def _chain_error(inp, k, ref):
    gm, gc, pm, pc, live = chained_float64(inp, k, ref)
    out = {}
    # dL_dmeans3D is not compared: its float64 side (gm, pm) does not yet model the kernels' mean chain -- the residual is
    # ~60x the planar part at both placements -- so it would measure that mismatch, not the planar precision
    for name, got, want, part in (("dL_dcov3D", k["dL_dcov3D"], gc, pc),):
        n = np.linalg.norm(part, axis=1)
        use = live & (n > 1e-3 * n.max())
        err = np.abs(got.astype(np.float64) - want).max(1)
        out[name] = float((err[use] / n[use]).max())
    return out


def test_planar_far_from_the_origin():
    res = {}
    for far in (False, True):
        inp = _placement(far)
        k, ref, problems, report, ours, st = check_planes(inp, planar=True, label="far" if far else "near")
        if far:
            assert float(k["means2D"][k["radii"] > 0, 0].mean()) > 1700
        assert not problems, "\n".join(problems)
        res[far] = _chain_error(inp, k, ref)
    print("chained planar gradient: worst |error| / |planar part| per Gaussian, near / far: " +
          " ".join(f"{q}={res[False][q]:.3g}/{res[True][q]:.3g} (x{res[True][q] / max(res[False][q], 1e-30):.3g})"
                   for q in res[False]))
    for q in res[False]:
        assert res[True][q] <= 4.0 * res[False][q], (q, res)

"""The float64 projection reference (tests/project_ref64.py) proves itself without a GPU.

* Against the C oracle (oracle/gs_oracle.c, fp32, built with -ffp-contract=off): its preprocess forward (every record and
  decision) and its preprocess backward fed seeded cotangents agree element by element, within the bound, on the four golden
  scenes and the edge scenes of test_project_ref64_gpu.py; the forward also agrees with the compiled reference's stored
  records in the golden fixtures.  Worst raw ratio |x - ref64| / (u e), over all those scenes (oracle / golden):
  depth 0.87 / 0.74, means2D 0.89 / 0.78, conic 0.19 / 0.14, rgb 0.79 / 0.69, cov3D 0.43 / 0.34 (the golden's rgb and
  cov3D: scenes with SH and scales), dL_dmeans3D 0.36, dL_dcov3D 0.74 (g3), dL_dsh 0.50, dL_dscales 0.12 (sh3_big),
  dL_drotations 0.093.  The C oracle writes -b^2 as (det - a c) in the conic's chain; the bound carries that cancellation.
* Against torch float64 autograd of an independent torch restatement of the forward (the reference's quirks expressed with
  `detach`): the backward matches to 1e-9 relative, for |q| != 1, degrees 0-3 with M = 16, clamped channels, Gaussians
  past the frustum clamp on both axes and AA on both sides of the 2.5e-5 threshold.
* Its bounds are tight enough to matter: on the edge scenes each mutation of the chain in project_ref64.MUTATIONS moves
  some checked element by more than twice its bound.
"""
import glob
import json
import os

import numpy as np
import pytest

import project_ref64 as P64
import util

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "g[0-9]*.npz")))
BWD = ("dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales", "dL_drotations")


def _golden(path):
    z = np.load(path)
    kw = json.loads(bytes(z["recipe"]).decode())
    if "bg" in kw:
        kw["bg"] = tuple(kw["bg"])
    return z, util.make_inputs(**kw)


def oracle_preprocess(g, cam, scale_modifier=1.0):
    from oracle import gs_oracle as O
    W, H = cam["W"], cam["H"]
    fw = O.forward(g["means3D"], g["opacities"], cam["viewmatrix"], cam["projmatrix"], cam["campos"], W, H, cam["tanfovx"],
                   cam["tanfovy"], np.zeros(3, np.float32), scales=g.get("scales"), rotations=g.get("rotations"),
                   cov3D_precomp=g.get("cov3D_precomp"), shs=g.get("shs"), sh_degree=g.get("sh_degree", 0),
                   colors_precomp=g.get("colors_precomp"), scale_modifier=scale_modifier, stages_only=True)
    return fw


def oracle_preprocess_backward(g, cam, fw, cot, scale_modifier=1.0):
    """gso_preprocess_backward on the given blend-stage cotangents (dL_dmean2D [P,2], dL_dconic [P,3], dL_dcolor [P,3])."""
    import ctypes as C
    from oracle import gs_oracle as O
    P = fw["P"]
    f32 = O._f32
    shs = g.get("shs")
    M = 0 if shs is None else np.asarray(shs).shape[1]
    m2 = np.zeros((P, 3), np.float32)
    m2[:, :2] = cot["dL_dmean2D"]
    co = np.zeros((P, 4), np.float32)
    co[:, [0, 1, 3]] = cot["dL_dconic"]
    out = dict(dL_dmeans3D=np.zeros((P, 3), np.float32), dL_dcov3D=np.zeros((P, 6), np.float32),
               dL_dsh=np.zeros((P, M, 3), np.float32), dL_dscales=np.zeros((P, 3), np.float32),
               dL_drotations=np.zeros((P, 4), np.float32))
    cov3D = f32(g["cov3D_precomp"]) if g.get("cov3D_precomp") is not None else fw["cov3D"]
    O.lib().gso_preprocess_backward(
        C.c_int(P), C.c_int(g.get("sh_degree", 0)), C.c_int(M), O._p(f32(g["means3D"])), O._p(fw["radii"]), O._p(f32(shs)),
        O._p(fw["clamped"]), O._p(f32(g.get("scales"))), O._p(f32(g.get("rotations"))), C.c_float(scale_modifier), O._p(cov3D),
        O._p(f32(cam["viewmatrix"]).reshape(-1)), O._p(f32(cam["projmatrix"]).reshape(-1)), C.c_int(cam["W"]), C.c_int(cam["H"]),
        C.c_float(cam["tanfovx"]), C.c_float(cam["tanfovy"]), O._p(f32(cam["campos"]).reshape(-1)), O._p(m2), O._p(co),
        O._p(np.ascontiguousarray(cot["dL_dcolor"], np.float32)), O._p(out["dL_dmeans3D"]), O._p(out["dL_dcov3D"]),
        O._p(out["dL_dsh"]), O._p(out["dL_dscales"]), O._p(out["dL_drotations"]))
    return out


def seeded_cotangents(P, seed, depth=False):
    rng = np.random.default_rng(seed)
    c = dict(dL_dmean2D=rng.normal(0, 1, (P, 2)), dL_dconic=rng.normal(0, 1, (P, 3)) * np.array([1.0, 0.5, 1.0]),
             dL_dopacity=rng.normal(0, 1, P), dL_dcolor=rng.normal(0, 1, (P, 3)),
             dL_ddepth=rng.normal(0, 1, P) if depth else None)
    return {k: (None if v is None else v.astype(np.float32)) for k, v in c.items()}


def compare_forward(ref, got, keep, rows, src):
    """Records of `got` (radii, means2D, depths, conic_opacity, cov3D?, rgb, clamped [P,3] or bits, tiles_touched) vs ref."""
    live = keep & ~ref["culled"]
    problems = []
    radii = np.asarray(got["radii"]).astype(np.int64)
    bad = keep & (radii != ref["radius"])
    if bad.any():
        i = np.nonzero(bad)[0][:5]
        problems.append(f"{src} radius differs at {i.tolist()}: {radii[i].tolist()} vs {ref['radius'][i].tolist()}")
    tt = np.asarray(got["tiles_touched"]).astype(np.int64)
    if (keep & (tt != ref["tiles_touched"])).any():
        problems.append(f"{src} tiles_touched differs at {np.nonzero(keep & (tt != ref['tiles_touched']))[0][:5].tolist()}")
    cl = np.asarray(got["clamped"])
    bits = (cl[:, 0] | (cl[:, 1] << 1) | (cl[:, 2] << 2)).astype(np.int64) if cl.ndim == 2 else cl.astype(np.int64)
    if ref["has_sh"] and (live & (bits != ref["clamped"])).any():
        problems.append(f"{src} clamp bits differ at {np.nonzero(live & (bits != ref['clamped']))[0][:5].tolist()}")
    co = np.asarray(got["conic_opacity"], np.float64)
    vals = dict(depth=np.asarray(got["depths"]), means2D=got["means2D"], conic=co[:, :3], rgb=got["rgb"], opacity=co[:, 3])
    if got.get("cov3D") is not None:
        vals["cov3D"] = got["cov3D"]
    if got.get("extent") is not None:
        vals["extent"] = got["extent"]
    for q, x in vals.items():
        r = P64.ratio(np.asarray(x)[live], (ref[q][live], ref[q + "_B"][live]), q, kappa=1.0)
        w = float(r.max()) if r.size else 0.0
        rows[f"{src} {q}"] = max(rows.get(f"{src} {q}", 0.0), w)
        if w > P64.KAPPA[q]:
            j = np.nonzero(live)[0][np.argmax(r.reshape(len(r), -1).max(1))]
            problems.append(f"{src} {q}: raw ratio {w:.3g} > KAPPA {P64.KAPPA[q]} at Gaussian {j}")
    return problems


def compare_backward(ref, got, keep, rows, src, names=BWD):
    problems = []
    for q in names:
        if got.get(q) is None or q not in ref or np.asarray(got[q]).size == 0:
            continue
        x = np.asarray(got[q], np.float64)
        v, e, d = (np.broadcast_to(np.asarray(a), x.shape)[keep] for a in ref[q])
        # raw ratio of the rounding part: what the inherited bound d does not cover, over u e (KAPPA scales e only)
        r = np.maximum(np.abs(x[keep] - v) - d, 0.0) / (P64.U * e + 1e-30)
        over = r > P64.KAPPA[q]
        w = float(r.max()) if r.size else 0.0
        rows[f"{src} {q}"] = max(rows.get(f"{src} {q}", 0.0), w)
        if over.any():
            idx = np.argsort(r.ravel())[::-1][:5]
            worst = [(np.unravel_index(i, r.shape), float(x[keep].ravel()[i]), float(v.ravel()[i]), float(r.ravel()[i])) for i in idx]
            problems.append(f"{src} {q}: {int(over.sum())} elements out of bound; worst (index, got, ref, raw ratio): {worst}")
    return problems


def _check_scene(g, cam, rows, src, scale_modifier=1.0, golden=None, seed=0):
    fw = oracle_preprocess(g, cam, scale_modifier)
    ref = P64.forward(g, cam, scale_modifier)
    keep = ~ref["border"]
    problems = compare_forward(ref, dict(fw, rgb=fw["rgb"] if g.get("colors_precomp") is None else g["colors_precomp"],
                                         cov3D=fw["cov3D"] if g.get("scales") is not None else None), keep, rows, "oracle")
    if golden is not None:
        z = golden
        gg = {k[3:]: z[k] for k in z.files if k.startswith("fw_")}
        if g.get("colors_precomp") is not None:
            gg["rgb"] = g["colors_precomp"]
        if g.get("scales") is None:
            gg["cov3D"] = None
        problems += compare_forward(ref, gg, keep, rows, "golden")
    cot = seeded_cotangents(fw["P"], seed)
    live = fw["radii"] > 0
    bits = (fw["clamped"][:, 0] | (fw["clamped"][:, 1] << 1) | (fw["clamped"][:, 2] << 2)).astype(np.int64)
    rb = P64.backward(g, [cam], [cot], scale_modifier, live=[live], clamped=[bits])
    ob = oracle_preprocess_backward(g, cam, fw, cot, scale_modifier)
    problems += compare_backward(rb, ob, keep & ~rb["border"], rows, "oracle")
    return problems


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_reference_matches_oracle_and_golden_per_element(path):
    z, inp = _golden(path)
    rows = {}
    problems = _check_scene(inp["g"], inp["cam"], rows, os.path.basename(path), golden=z, seed=5)
    print(os.path.basename(path), " ".join(f"{k}={v:.3g}" for k, v in rows.items()))
    assert not problems, "\n".join(problems)


def _edge_scenes():
    import test_project_ref64_gpu as S
    return S.SCENES


@pytest.mark.parametrize("scene", ["clamp_x", "clamp_y", "near", "quat_scale", "quat_scale_19", "sh0", "sh1", "sh2", "sh3",
                                   "sh3_m16", "precomp_cov", "precomp_sr", "aa1", "aa2", "aa3", "ragged_f32", "sh3_big"])
def test_reference_matches_oracle_on_edge_scenes(scene):
    sc = _edge_scenes()[scene]()
    rows = {}
    problems = _check_scene(sc["g"], sc["cam"], rows, scene, scale_modifier=sc.get("scale_modifier", 1.0), seed=9)
    print(scene, " ".join(f"{k}={v:.3g}" for k, v in rows.items()))
    assert not problems, "\n".join(problems)


# --------------------------------------------------------------------------- torch float64 autograd
def _torch_loss(g, cam, cot, mod, aa):
    """An independent torch restatement of the projection of one view; returns (loss, leaves).  The reference's quirks
    as `detach`: outside the frustum clamp t.x_c = (+-lim t.z).detach() (constant in d/dt.x and d/dt.z), the quaternion
    un-normalised, the scale leaf is scale_modifier * scale, the loss takes 2 gB on the conic's b (gB is the half-weight
    cotangent), the conic's gradient takes w = 1 / (det^2 + 1e-7), the clamp of an SH channel at 0 is a relu."""
    import torch
    d = torch.float64
    T = lambda a: torch.tensor(np.asarray(a, np.float32).astype(np.float64), dtype=d)  # noqa: E731
    p = T(g["means3D"]).requires_grad_()
    leaves = dict(dL_dmeans3D=p)
    if g.get("scales") is not None:
        se = (T(g["scales"]) * float(np.float32(mod))).detach().requires_grad_()
        q = T(g["rotations"]).requires_grad_()
        leaves.update(dL_dscales=se, dL_drotations=q)
        r, x, y, z = q.unbind(1)
        Rq = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                          2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                          2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
        Sig = Rq @ torch.diag_embed(se * se) @ Rq.transpose(1, 2)
    else:
        c6 = T(g["cov3D_precomp"]).requires_grad_()
        leaves["dL_dcov3D"] = c6
        Sig = torch.stack([c6[:, [0, 1, 2]], c6[:, [1, 3, 4]], c6[:, [2, 4, 5]]], 1)
    o = T(g["opacities"]).reshape(-1).requires_grad_()
    leaves["dL_dopacity"] = o
    vm = T(cam["viewmatrix"]).reshape(4, 4).T           # rows: world -> view
    pm = T(cam["projmatrix"]).reshape(4, 4).T
    t = p @ vm[:3, :3].T + vm[:3, 3]
    vw = P64.view_of(cam)
    fx, fy, lx, ly = vw["fx"], vw["fy"], vw["limx"], vw["limy"]
    tz = t[:, 2]
    ux, uy = t[:, 0] / tz, t[:, 1] / tz
    cx = torch.where((ux >= -lx) & (ux <= lx), t[:, 0], (ux.clamp(-lx, lx) * tz).detach())
    cy = torch.where((uy >= -ly) & (uy <= ly), t[:, 1], (uy.clamp(-ly, ly) * tz).detach())
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, zero, -fx * cx / tz ** 2], 1), torch.stack([zero, fy / tz, -fy * cy / tz ** 2], 1)], 1)
    Mx = J @ vm[:3, :3]
    cov = Mx @ Sig @ Mx.transpose(1, 2)
    h = float(np.float32(0.3))
    a, b, c = cov[:, 0, 0] + h, cov[:, 0, 1], cov[:, 1, 1] + h
    det = a * c - b * b
    # the reference's w = 1 / (det^2 + 1e-7) in place of 1 / det^2: the conic's gradient scaled by det^2 w, value unchanged
    k = (det * det / (det * det + float(np.float32(1e-7)))).detach()
    sc = lambda x: x.detach() + (x - x.detach()) * k  # noqa: E731
    hom = torch.cat([p, torch.ones_like(tz)[:, None]], 1) @ pm.T
    ndc = hom[:, :2] / (hom[:, 3:4] + float(np.float32(1e-7)))
    C_ = lambda k: torch.tensor(np.asarray(cot[k], np.float64), dtype=d)  # noqa: E731
    gco = C_("dL_dconic")
    loss = (ndc * C_("dL_dmean2D")).sum() + (sc(c / det) * gco[:, 0] + 2 * sc(-b / det) * gco[:, 1] + sc(a / det) * gco[:, 2]).sum()
    oe = o
    if aa:
        rr = (cov[:, 0, 0] * cov[:, 1, 1] - b * b) / det
        oe = o * torch.sqrt(rr.clamp_min(P64.AA_CLAMP))
    loss = loss + (oe * C_("dL_dopacity")).sum()
    if cot.get("dL_ddepth") is not None:
        loss = loss + (tz * C_("dL_ddepth")).sum()
    if g.get("shs") is not None:
        sh = T(g["shs"]).requires_grad_()
        leaves["dL_dsh"] = sh
        v = p - T(cam["campos"]).reshape(-1)
        dr = v / v.norm(dim=1, keepdim=True)
        x, y, z = dr.unbind(1)
        xx, yy, zz = x * x, y * y, z * z
        basis = [torch.full_like(x, P64.SH_C0), -P64.SH_C1 * y, P64.SH_C1 * z, -P64.SH_C1 * x]
        c2, c3 = P64.SH_C2, P64.SH_C3
        basis += [c2[0] * x * y, c2[1] * y * z, c2[2] * (2 * zz - xx - yy), c2[3] * x * z, c2[4] * (xx - yy)]
        basis += [c3[0] * y * (3 * xx - yy), c3[1] * x * y * z, c3[2] * y * (4 * zz - xx - yy), c3[3] * z * (2 * zz - 3 * xx - 3 * yy),
                  c3[4] * x * (4 * zz - xx - yy), c3[5] * z * (xx - yy), c3[6] * x * (xx - 3 * yy)]
        n = (int(g["sh_degree"]) + 1) ** 2
        rgb = sum(basis[k][:, None] * sh[:, k, :] for k in range(n)) + 0.5
        loss = loss + (torch.relu(rgb) * C_("dL_dcolor")).sum()
    return loss, leaves


AUTOGRAD = [("clamp_x", False), ("clamp_y", False), ("quat_scale", False), ("sh0_m16", False), ("sh1_m16", False),
            ("sh2_m16", False), ("sh3_m16", False), ("precomp_cov", False), ("aa1", True), ("aa3", True)]


@pytest.mark.parametrize("scene,aa", AUTOGRAD, ids=[s for s, _ in AUTOGRAD])
def test_backward_matches_torch_float64_autograd(scene, aa):
    sc = _edge_scenes()[scene]()
    g, cam, mod = sc["g"], sc["cam"], sc.get("scale_modifier", 1.0)
    ref = P64.forward(g, cam, mod, antialias=aa)
    live = ~ref["culled"]
    sel = {k: (v[live] if isinstance(v, np.ndarray) and v.ndim and len(v) == len(live) else v) for k, v in g.items()}
    cot = seeded_cotangents(int(live.sum()), 3, depth=True)
    rb = P64.backward(sel, [cam], [cot], mod, antialias=aa)
    loss, leaves = _torch_loss(sel, cam, cot, mod, aa)
    loss.backward()
    for name, leaf in leaves.items():
        want = leaf.grad.numpy().reshape(rb[name][0].shape)
        got = rb[name][0]
        # 1e-9 relative, or the float64 evaluation's own rounding (the fp32 bound e in units of 2^-53) where the
        # chain is ill-conditioned (the needles and 1e4-anisotropic splats of quat_scale)
        tol = 1e-9 * np.abs(want).max() + 16 * 2.0 ** -53 * np.broadcast_to(rb[name][1], got.shape)
        err = np.abs(got - want)
        assert np.all(err <= tol), (name, float(err.max()), np.abs(want).max())
    # the edges the scene was built for are in the comparison
    if scene in ("clamp_x", "clamp_y"):
        assert (~ref["inx" if scene == "clamp_x" else "iny"] & live).sum() >= 8
    if aa:   # Gaussians on both sides of the compensation's 2.5e-5 clamp
        S = P64.cov3d(sel, mod)[0]
        G = P64._geometry(P64._cols(sel["means3D"]), S, P64.view_of(cam))
        r = (G["a0"].v * G["c0"].v - G["b"].v ** 2) / G["det"].v
        assert (r > P64.AA_CLAMP).sum() >= 4 and (r < P64.AA_CLAMP).sum() >= 4, np.sort(r)[:8]


# --------------------------------------------------------------------------- sensitivity
SENS = ("clamp_x", "clamp_y", "quat_scale", "sh1", "sh2", "sh3", "sh1_m16", "near")


def test_every_mutation_of_the_chain_moves_a_checked_element_past_twice_its_bound():
    """Measured: every mutation in project_ref64.MUTATIONS is seen on at least one edge scene (printed: the scenes that see
    it and the largest move in units of the bound)."""
    seen = {m: [] for m in P64.MUTATIONS}
    for scene in SENS:
        sc = _edge_scenes()[scene]()
        g, cam, mod = sc["g"], sc["cam"], sc.get("scale_modifier", 1.0)
        cot = seeded_cotangents(len(g["means3D"]), 4, depth=True)
        base = P64.backward(g, [cam], [cot], mod)
        keep = ~base["border"]
        for m in P64.MUTATIONS:
            mut = P64.backward(g, [cam], [cot], mod, mutate={m})
            worst = 0.0
            for q in BWD + ("dL_dopacity", "dL_dcolors"):
                if q not in base:
                    continue
                v, e, d = (np.broadcast_to(np.asarray(a), np.shape(base[q][0])) for a in base[q])
                x = np.asarray(mut[q][0])
                r = (np.abs(x - v) / (2.0 * (P64.KAPPA[q] * P64.U * e + d) + 1e-30))[keep]
                worst = max(worst, float(r.max()) if r.size else 0.0)
            if worst > 1.0:
                seen[m].append((scene, round(worst, 1)))
    print({m: v[:3] for m, v in seen.items()})
    assert all(seen.values()), [m for m, v in seen.items() if not v]

"""The float64 blend reference's extra columns (tests/blend_ref64.py: the normal / flow planes and planar depth) prove
themselves without a GPU.

* On the four golden scenes, with the C oracle's own decisions, the extra-column planes and gradients equal the oracle's blend
  with the quads as feature channels (a feature channel has no background term, as these planes have none).  Planar depth:
  the oracle blends {z, a, b, e} as four channels with cotangents {g, g px, g py, g}; its planar plane is those channels
  combined in numpy float32 in the kernels' order.
* Planar dL/dopacity, dL/dconic, dL/dquad and dL/dmeans2D equal torch float64 autograd of a dense per-tile restatement of the
  planar blend.
* The bounds are tight enough to see each broken convention: every one of them moves some checked element past twice its
  bound.
"""
import glob
import json
import os

import numpy as np
import pytest

import blend_ref64 as R64
import util
from test_blend_ref64_cpu import oracle_state

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "g[0-9]*.npz")))


def _view_depth(g, cam):
    vm = np.asarray(cam["viewmatrix"], np.float32).reshape(-1)
    return (g["means3D"] @ np.array([vm[2], vm[6], vm[10]], np.float32) + vm[14]).astype(np.float32)


def _pixels(W, H):
    py, px = np.mgrid[0:H, 0:W]
    return px.astype(np.float32), py.astype(np.float32)


def _with_quads(path, planar, seed=5):
    """(inp, the oracle's forward and backward with the extra channels appended to the features, st, masks, ref)"""
    z = np.load(path)
    kw = json.loads(bytes(z["recipe"]).decode())
    if "bg" in kw:
        kw["bg"] = tuple(kw["bg"])
    inp = util.make_inputs(**kw, depth=True)
    g, ct, cam = inp["g"], inp["ct"], inp["cam"]
    P, W, H, F = inp["P"], inp["W"], inp["H"], inp["F"]
    rng = np.random.default_rng(seed)
    depth = _view_depth(g, cam)
    px, py = _pixels(W, H)
    gd = ct["dL_ddepth"].astype(np.float32)
    if planar:
        ab = rng.normal(0, 0.01, (P, 2)).astype(np.float32)
        e = rng.normal(0, 0.3, P).astype(np.float32)
        quad = np.stack([ab[:, 0], ab[:, 1], e, np.zeros(P, np.float32)], 1)
        extra = np.stack([depth, ab[:, 0], ab[:, 1], e], 1)
        gx = np.stack([gd, gd * px, gd * py, gd], 0)
    else:
        quad = np.concatenate([rng.normal(0, 1, (P, 3)), np.zeros((P, 1))], 1).astype(np.float32)
        extra = quad[:, :3]
        gx = rng.normal(0, 1, (3, H, W)).astype(np.float32)
    feat = extra if not F else np.concatenate([g["feature"], extra], 1)
    gf = gx if not F else np.concatenate([ct["dL_dfeature"], gx], 0)
    inp2 = dict(inp, F=feat.shape[1], g=dict(g, feature=np.ascontiguousarray(feat, np.float32)),
                ct=dict(ct, dL_dfeature=np.ascontiguousarray(gf, np.float32)))
    fw, bw = util.run_oracle(inp2)
    st = oracle_state(inp, fw, depth=depth, g_depth=gd)
    st.update(quad=quad, planar=planar)
    if not planar:
        st["g_quad"] = gx
    masks = [R64.decide_fp32(st, t) for t in range(st["ranges"].shape[0])]
    return inp, fw, bw, st, masks, R64.blend(st, masks)


def _worst(got, ref, B, q):
    r = R64.ratio(got, ref, B, q)
    return float(r.max())


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_normal_plane_matches_the_oracle_feature_channels(path):
    inp, fw, bw, st, masks, ref = _with_quads(path, planar=False)
    F = inp["F"]
    assert np.array_equal(ref["n_contrib"].ravel(), fw["n_contrib"].astype(np.int64))
    rows = dict(normal=_worst(fw["out_feature"][F:F + 3], ref["quad"][:3], ref["quad_B"][:3], "normal"),
                dL_dquad=_worst(bw["dL_dfeature"][:, F:F + 3], ref["dL_dquad"][:, :3], ref["dL_dquad_B"][:, :3], "dL_dquad"))
    print(os.path.basename(path), {k: f"{v:.3g} (raw {v * R64.KAPPA[k]:.3g})" for k, v in rows.items()})
    assert max(rows.values()) <= 1.0, rows
    assert not ref["quad"][3].any() and not ref["dL_dquad"][:, 3].any()


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_planar_depth_matches_the_oracle_feature_channels(path):
    inp, fw, bw, st, masks, ref = _with_quads(path, planar=True)
    F, W, H = inp["F"], inp["W"], inp["H"]
    assert np.array_equal(ref["n_contrib"].ravel(), fw["n_contrib"].astype(np.int64))
    f = np.float32
    of = fw["out_feature"].astype(f)
    px, py = _pixels(W, H)
    # the kernels' order: col3 + ((px col4 + py col5) + col6)
    plane = of[F] + ((px * of[F + 1] + py * of[F + 2]) + of[F + 3])
    # the reference's dL_dquad is relative to the mean ({sum w g (px - mu_x), ...}); the oracle's channels give the absolute
    # sums {sum w g px, ...}: compare those, adding mu times dL/de and its bound
    mu = st["means2D"].astype(np.float64)
    dq = ref["dL_dquad"][:, :3].copy()
    dqB = ref["dL_dquad_B"][:, :3].copy()
    dq[:, :2] += mu * dq[:, 2:3]
    dqB[:, :2] += np.abs(mu) * dqB[:, 2:3]
    rows = dict(planar_depth=_worst(plane, ref["depth"], ref["depth_B"], "planar_depth"),
                dL_dquad=_worst(bw["dL_dfeature"][:, F + 1:F + 4], dq, dqB, "dL_dquad"),
                dL_ddepth=_worst(bw["dL_dfeature"][:, F], ref["dL_ddepth"], ref["dL_ddepth_B"], "dL_ddepth"),
                dL_dmeans2D=_worst(bw["dL_dmeans2D"][:, :2], ref["dL_dmeans2D"], ref["dL_dmeans2D_B"], "dL_dmeans2D"),
                dL_dopacity=_worst(bw["dL_dopacity"][:, 0], ref["dL_dopacity"], ref["dL_dopacity_B"], "dL_dopacity"))
    print(os.path.basename(path), {k: f"{v:.3g} (raw {v * R64.KAPPA[k]:.3g})" for k, v in rows.items()})
    assert max(rows.values()) <= 1.0, rows


def test_planar_gradients_match_torch_autograd_of_a_dense_restatement():
    """Decisions held fixed: the reference's planar dL/dopacity, dL/dconic, dL/dquad and dL/dmeans2D are the float64
    derivatives of sum g_color colour + g_depth D + h alpha, D = sum w (z + a px + b py + e); dL/dquad with e's share folded
    into a and b, dL/da - mu_x dL/de and dL/db - mu_y dL/de."""
    import torch
    inp = util.make_inputs(P=300, W=40, H=24, F=0, seed=21, depth=True, bg=(0.3, 0.6, 0.9))
    fw, _ = util.run_oracle(inp, backward=False)
    rng = np.random.default_rng(3)
    H, W, P = inp["H"], inp["W"], inp["P"]
    st = oracle_state(inp, fw, depth=rng.random(P) + 1.0, g_alpha=rng.normal(0, 1, (H, W)), g_depth=rng.normal(0, 1, (H, W)))
    st.update(quad=np.concatenate([rng.normal(0, 0.02, (P, 2)), rng.normal(0, 0.5, (P, 1)), np.zeros((P, 1))], 1), planar=True)
    for k in ("means2D", "conic_opacity", "colors", "depth"):
        st[k] = np.array(st[k], np.float64)
    T = st["ranges"].shape[0]
    masks = [R64.decide(st, t)["mask"] for t in range(T)]
    ref = R64.blend(st, masks)
    D = torch.float64
    m2 = torch.tensor(st["means2D"], dtype=D, requires_grad=True)
    co = torch.tensor(st["conic_opacity"], dtype=D, requires_grad=True)
    qd = torch.tensor(st["quad"], dtype=D, requires_grad=True)
    col, z, bg = torch.tensor(st["colors"], dtype=D), torch.tensor(st["depth"], dtype=D), torch.tensor(st["bg"], dtype=D)
    loss = 0.0
    for t in range(T):
        r0, r1 = (int(v) for v in st["ranges"][t])
        if r1 == r0:
            continue
        ids = torch.tensor(st["point_list"][r0:r1].astype(np.int64))
        px, py, inside = R64.tile_pixels(W, H, t)
        pxt, pyt = torch.tensor(px, dtype=D)[:, None], torch.tensor(py, dtype=D)[:, None]
        dx, dy = m2[ids, 0][None] - pxt, m2[ids, 1][None] - pyt
        a, b, c, o = co[ids, 0], co[ids, 1], co[ids, 2], co[ids, 3]
        G = torch.exp(-0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy)
        mk = torch.tensor(masks[t])
        al = torch.where(mk, torch.clamp(o * G, max=float(R64.ALPHA_MAX)), torch.zeros_like(G))
        Tb = torch.cumprod(torch.cat([torch.ones(256, 1, dtype=D), 1 - al[:, :-1]], 1), 1)
        w = al * Tb
        Tf = Tb[:, -1] * (1 - al[:, -1])
        Dp = z[ids][None] + qd[ids, 0][None] * pxt + qd[ids, 1][None] * pyt + qd[ids, 2][None]
        x, y = np.where(inside, px, 0), np.where(inside, py, 0)
        ins = torch.tensor(inside, dtype=D)
        gc = torch.tensor(st["g_color"][:, y, x].T, dtype=D) * ins[:, None]
        gdp = torch.tensor(st["g_depth"][y, x], dtype=D) * ins
        h = torch.tensor(st["g_alpha"][y, x], dtype=D) * ins
        colour = w @ col[ids] + Tf[:, None] * bg[None]
        loss = loss + (gc * colour).sum() + (gdp * (w * Dp).sum(1)).sum() + (h * (1 - Tf)).sum()
    gm, gco, gq = torch.autograd.grad(loss, (m2, co, qd))
    gm, gco, gq = gm.numpy(), gco.numpy(), gq.numpy()
    scale = lambda x: max(float(np.abs(x).max()), 1e-30)  # noqa: E731
    assert np.abs(ref["dL_dmeans2D"] - gm * np.array([0.5 * W, 0.5 * H])).max() <= 1e-9 * scale(ref["dL_dmeans2D"])
    assert np.abs(ref["dL_dconic"] - gco[:, :3] * np.array([1.0, 0.5, 1.0])).max() <= 1e-9 * scale(ref["dL_dconic"])
    assert np.abs(ref["dL_dopacity"] - gco[:, 3]).max() <= 1e-9 * scale(ref["dL_dopacity"])
    mu = st["means2D"]
    want = np.stack([gq[:, 0] - mu[:, 0] * gq[:, 2], gq[:, 1] - mu[:, 1] * gq[:, 2], gq[:, 2], gq[:, 3]], 1)
    assert np.abs(ref["dL_dquad"] - want).max() <= 1e-9 * scale(ref["dL_dquad"])
    assert np.abs(gq[:, :3]).max(0).min() > 0


def _moves(name, mutated, ref, B, q):
    """the largest |mutated - ref| over twice the bound (KAPPA u B) of quantity q; > 1: the mutation is seen"""
    r = R64.ratio(mutated, ref, B, q) / 2.0
    print(f"{name}: {float(r.max()):.3g}")
    return float(r.max())


def test_each_broken_convention_moves_a_checked_element_past_twice_its_bound():
    path = GOLDEN[1]
    inp, fw, bw, st, masks, ref = _with_quads(path, planar=True)
    W, H = inp["W"], inp["H"]
    assert W != H
    seen = {}
    # pixel centre px + 0.5 in the planar columns: dL/da gains 0.5 dL/de, the plane 0.5 sum w a
    seen["px + 0.5"] = _moves("px + 0.5", ref["dL_dquad"][:, 0] + 0.5 * ref["dL_dquad"][:, 2], ref["dL_dquad"][:, 0],
                              ref["dL_dquad_B"][:, 0], "dL_dquad")
    # px and py swapped: dL/da becomes sum w g py
    swapped = R64.blend(dict(st, quad=st["quad"][:, [1, 0, 2, 3]]), masks)
    seen["px <-> py"] = _moves("px <-> py", swapped["depth"], ref["depth"], ref["depth_B"], "planar_depth")
    # the depth head's cotangent missing from the planar columns (present in the depth column only)
    rng = np.random.default_rng(9)
    head = rng.normal(0, 1, (H, W))
    with_head = R64.blend(dict(st, g_depth=st["g_depth"] + head), masks)
    no_head_cols = with_head["dL_dquad"][:, :3] - (R64.blend(dict(st, g_depth=head), masks)["dL_dquad"][:, :3])
    seen["head missing"] = _moves("head missing", no_head_cols, with_head["dL_dquad"][:, :3], with_head["dL_dquad_B"][:, :3],
                                  "dL_dquad")
    # planar median with (px, py) taken column-major on a W != H image
    mid = np.full((H, W), -1)
    for t, m in enumerate(masks):
        px, py, inside = R64.tile_pixels(W, H, t)
        r0, r1 = (int(v) for v in st["ranges"][t])
        has = m.any(1) & inside
        first = np.argmax(m, 1)
        mid[py[has], px[has]] = st["point_list"][r0:r1][first[has]]
    plane, B = R64.median_planar(st, mid, None, R64.new_out(st))
    p = np.arange(H * W)
    q = st["quad"][np.maximum(mid, 0)].reshape(-1, 4)
    zc = st["depth"][np.maximum(mid, 0)].ravel()
    cm = (zc + q[:, 0] * (p // H) + q[:, 1] * (p % H) + q[:, 2]).reshape(H, W)
    cm[mid < 0] = 0
    seen["median column-major"] = _moves("median column-major", cm, plane, B, "median_planar")
    # the normal plane: a background term, cot_scale on its cotangent, its cotangent counted in every channel group (G = 2)
    inp, fw, bw, st, masks, ref = _with_quads(path, planar=False)
    bgn = ref["final_T"][None] * np.asarray(inp["bg"], np.float64)[:, None, None]
    seen["background on the normal plane"] = _moves("background", ref["quad"][:3] + bgn, ref["quad"][:3], ref["quad_B"][:3],
                                                    "normal")
    seen["cot_scale on the normal cotangent"] = _moves("cot_scale", 0.5 * ref["dL_dquad"][:, :3], ref["dL_dquad"][:, :3],
                                                       ref["dL_dquad_B"][:, :3], "dL_dquad")
    seen["counted per channel group"] = _moves("groups", 2.0 * ref["dL_dquad"][:, :3], ref["dL_dquad"][:, :3],
                                               ref["dL_dquad_B"][:, :3], "dL_dquad")
    missed = [k for k, v in seen.items() if not v > 1.0]
    assert not missed, seen

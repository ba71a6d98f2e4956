"""The float64 blend reference (tests/blend_ref64.py) proves itself without a GPU.

* Fed the C oracle's own decisions on the four golden scenes, it agrees element by element, within its bound, with the C
  oracle's images and blend-stage gradients and with the stored outputs of the compiled reference.
* With the decisions held fixed the blend is smooth: its gradients match central differences of its own float64 forward.
* Its bounds are tight enough to matter: on the scenes of test_blend_pairs_gpu.py, projected and binned by the C oracle,
  removing any single contributing pair moves some checked element by more than twice its bound.
"""
import glob
import json
import os

import numpy as np
import pytest

import blend_ref64 as R64
import project_ref64 as P64
import util

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "g[0-9]*.npz")))


def oracle_state(inp, fw, depth=None, g_alpha=None, g_depth=None):
    g, ct = inp["g"], inp["ct"]
    F = inp["F"]
    return dict(W=inp["W"], H=inp["H"], ranges=fw["ranges"], point_list=fw["point_list"], means2D=fw["means2D"],
                conic_opacity=fw["conic_opacity"],
                colors=g["colors_precomp"] if g["colors_precomp"] is not None else fw["rgb"],
                feature=g["feature"] if F else None, depth=depth, bg=inp["bg"], g_color=ct["dL_dcolor"],
                g_feature=ct["dL_dfeature"] if F else None, g_depth=g_depth, g_alpha=g_alpha)


def worst(name, got, ref, B):
    """(name, worst ratio to the bound, worst raw ratio |x - ref| / (u B)); the quantity is the name's last word."""
    q = name.split()[-1]
    r = R64.ratio(got, ref, B, q)
    return name, float(r.max()) if r.size else 0.0, float(r.max()) * R64.KAPPA[q] if r.size else 0.0


def _golden(path):
    z = np.load(path)
    kw = json.loads(bytes(z["recipe"]).decode())
    if "bg" in kw:
        kw["bg"] = tuple(kw["bg"])
    inp = util.make_inputs(**kw)
    fw, bw = util.run_oracle(inp)
    return z, inp, fw, bw


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_reference_matches_oracle_and_golden_per_element(path):
    """Worst raw ratio |x - ref64| / (u B), C oracle / compiled reference: colour 0.34/1.62, final_T 0.22/1.77, features
    0.37/5.98, dL_dmeans2D 0.0048/0.057, dL_dopacity 0.019/0.17, dL_dcolors 0.069 (oracle) and 0.042/0.39 (g3),
    dL_dfeature 0.072/1.32, dL_dconic 0.0029 (oracle), dL_dcov3D 0/0 (g3); the largest of each over g1-g4.  dL_dcov3D is chained by
    project_ref64.cov3d_grad: the raw ratio of the part its inherited conic bound does not cover, over u e."""
    z, inp, fw, bw = _golden(path)
    st = oracle_state(inp, fw)
    T = st["ranges"].shape[0]
    masks = [R64.decide_fp32(st, t) for t in range(T)]
    ref = R64.blend(st, masks)
    F, W, H = inp["F"], inp["W"], inp["H"]
    # the restated fp32 decisions are the oracle's: same last contributor for every pixel
    assert np.array_equal(ref["n_contrib"].ravel(), fw["n_contrib"].astype(np.int64))
    rows = []
    for src, img, ft, g in (("oracle", fw["out_color"], fw["final_T"], bw),
                            ("golden", z["fw_out_color"], z["fw_final_T"], {k[3:]: z[k] for k in z.files if k.startswith("bw_")})):
        keep_pix = np.ones((H, W), bool)
        keep_g = np.ones(fw["means2D"].shape[0], bool)
        if src == "golden":
            # where the compiled reference (nvcc, FMA-contracted) decided a pixel differently, its values follow other decisions
            diff = (z["fw_n_contrib"].reshape(H, W) != ref["n_contrib"])
            keep_pix &= ~diff
            for t in range(T):
                px, py, inside = R64.tile_pixels(W, H, t)
                bad = inside & diff[np.where(inside, py, 0), np.where(inside, px, 0)]
                if bad.any():
                    r0, r1 = st["ranges"][t]
                    keep_g[st["point_list"][r0:r1]] = False
        rows.append(worst(src + " color", img[:, keep_pix], ref["color"][:, keep_pix], ref["color_B"][:, keep_pix]))
        rows.append(worst(src + " final_T", ft.reshape(H, W)[keep_pix], ref["final_T"][keep_pix], ref["final_T_B"][keep_pix]))
        if F:
            fimg = fw["out_feature"] if src == "oracle" else z["fw_out_feature"]
            rows.append(worst(src + " feature", fimg[:, keep_pix], ref["feature"][:, keep_pix], ref["feature_B"][:, keep_pix]))
            rows.append(worst(src + " dL_dfeature", g["dL_dfeature"][keep_g], ref["dL_dfeature"][keep_g], ref["dL_dfeature_B"][keep_g]))
        rows.append(worst(src + " dL_dmeans2D", g["dL_dmeans2D"][keep_g, :2], ref["dL_dmeans2D"][keep_g], ref["dL_dmeans2D_B"][keep_g]))
        rows.append(worst(src + " dL_dopacity", g["dL_dopacity"][keep_g, 0], ref["dL_dopacity"][keep_g], ref["dL_dopacity_B"][keep_g]))
        if src == "oracle":
            rows.append(worst(src + " dL_dconic", g["dL_dconic"][:, [0, 1, 3]], ref["dL_dconic"], ref["dL_dconic_B"]))
        if inp["g"]["cov3D_precomp"] is not None:
            # the conic gradients chained to dL_dcov3D by the projection reference (tests/project_ref64.py)
            c3, bd = P64.cov3d_grad(ref, inp["g"], inp["cam"], live=fw["radii"] > 0)
            ok = keep_g & ~bd
            r = P64.raw_ratio(g["dL_dcov3D"][ok], tuple(np.broadcast_to(x, c3[0].shape)[ok] for x in c3))
            raw = float(r.max()) if r.size else 0.0
            rows.append((src + " dL_dcov3D", raw / P64.KAPPA["dL_dcov3D"], raw))
        if inp["g"]["colors_precomp"] is not None:
            rows.append(worst(src + " dL_dcolors", g["dL_dcolors"][keep_g], ref["dL_dcolors"][keep_g], ref["dL_dcolors_B"][keep_g]))
        else:
            # the golden's colour gradient goes on into SH; the oracle keeps the blend-stage one
            if src == "oracle":
                rows.append(worst(src + " dL_dcolors", g["dL_dcolors"], ref["dL_dcolors"], ref["dL_dcolors_B"]))
    print(os.path.basename(path), " ".join(f"{k}={v:.3g}(raw {r:.3g})" for k, v, r in rows))
    bad = [(k, v) for k, v, _ in rows if not v <= 1.0]
    assert not bad, bad


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_depth_cotangent_matches_oracle_per_element(path):
    """The per-Gaussian depth cotangent dL_ddepth = w^T g_depth against the C oracle's blend backward with the view-space
    depth as its one feature channel (the oracle renders no depth plane).  Worst raw ratio |x - ref64| / (u B) over g1-g4:
    0.018 / 0.042 / 0.050 / 0.064."""
    from oracle import gs_oracle as O
    z = np.load(path)
    kw = json.loads(bytes(z["recipe"]).decode())
    if "bg" in kw:
        kw["bg"] = tuple(kw["bg"])
    kw["F"] = 0
    inp = util.make_inputs(**kw, depth=True)
    g, cam, ct = inp["g"], inp["cam"], inp["ct"]
    vm = np.asarray(cam["viewmatrix"], np.float32).reshape(-1)
    depth = (g["means3D"] @ np.array([vm[2], vm[6], vm[10]], np.float32) + vm[14]).astype(np.float32)
    okw = dict(scales=g["scales"], rotations=g["rotations"], cov3D_precomp=g["cov3D_precomp"], shs=g["shs"],
               sh_degree=g["sh_degree"], colors_precomp=g["colors_precomp"], feature=depth[:, None])
    fw = O.forward(g["means3D"], g["opacities"], cam["viewmatrix"], cam["projmatrix"], cam["campos"], inp["W"], inp["H"],
                   cam["tanfovx"], cam["tanfovy"], inp["bg"], **okw)
    bw = O.backward(fw, ct["dL_dcolor"], ct["dL_ddepth"][None], g["means3D"], cam["viewmatrix"], cam["projmatrix"],
                    cam["campos"], cam["tanfovx"], cam["tanfovy"], inp["bg"], **okw)
    st = dict(oracle_state(dict(inp, F=0), fw), depth=depth, g_depth=ct["dL_ddepth"])
    masks = [R64.decide_fp32(st, t) for t in range(st["ranges"].shape[0])]
    ref = R64.blend(st, masks)
    r = R64.ratio(bw["dL_dfeature"][:, 0], ref["dL_ddepth"], ref["dL_ddepth_B"], "dL_ddepth", kappa=1.0)
    print(os.path.basename(path), f"dL_ddepth raw {r.max():.3g}")
    assert r.max() <= R64.KAPPA["dL_ddepth"]


def _loss(st, masks):
    o = R64.blend(st, masks, backward=False)
    l = (o["color"] * st["g_color"]).sum() + (o["alpha"] * st["g_alpha"]).sum()
    if st.get("feature") is not None:
        l += (o["feature"] * st["g_feature"]).sum()
    if st.get("depth") is not None:
        l += (o["depth"] * st["g_depth"]).sum()
    return l


def test_gradients_match_central_differences_of_the_float64_forward():
    """Decisions held fixed, no clamped pair: every blend-stage gradient is the derivative of the float64 forward
    (dL_dconic.y is the reference's half-weight convention: d/d(conic b) = 2 dL_dconic.y)."""
    inp = util.make_inputs(P=300, W=40, H=24, F=5, seed=21, depth=True, bg=(0.3, 0.6, 0.9))
    fw, _ = util.run_oracle(inp, backward=False)
    rng = np.random.default_rng(3)
    H, W = inp["H"], inp["W"]
    st = oracle_state(inp, fw, depth=rng.random(inp["P"]).astype(np.float32) + 1.0,
                      g_alpha=rng.normal(0, 1, (H, W)), g_depth=rng.normal(0, 1, (H, W)))
    for k in ("means2D", "conic_opacity", "colors", "feature", "depth"):
        st[k] = np.array(st[k], np.float64)
    T = st["ranges"].shape[0]
    masks = [R64.decide(st, t)["mask"] for t in range(T)]
    ref = R64.blend(st, masks)
    clamped = np.zeros(inp["P"], bool)
    for t in range(T):
        p = R64._pairs(st, t)
        clamped[p["ids"][((p["o"] * p["G"] >= R64.ALPHA_MAX) & masks[t]).any(0)]] = True
    live = np.nonzero((np.abs(ref["dL_dopacity"]) > 1e-3) & ~clamped)[0][:8]
    assert len(live) >= 4
    fields = [("means2D", 0, "dL_dmeans2D", 0, 1.0), ("means2D", 1, "dL_dmeans2D", 1, 1.0),
              ("conic_opacity", 0, "dL_dconic", 0, 1.0), ("conic_opacity", 1, "dL_dconic", 1, 0.5),
              ("conic_opacity", 2, "dL_dconic", 2, 1.0), ("conic_opacity", 3, "dL_dopacity", None, 1.0),
              ("colors", 1, "dL_dcolors", 1, 1.0), ("feature", 4, "dL_dfeature", 4, 1.0)]
    for g in live:
        for arr, c, gname, gc, scale in fields:
            eps = 1e-5 * max(1.0, abs(st[arr][g, c]))
            base = st[arr][g, c]
            st[arr][g, c] = base + eps
            lp = _loss(st, masks)
            st[arr][g, c] = base - eps
            lm = _loss(st, masks)
            st[arr][g, c] = base
            num = (lp - lm) / (2 * eps) * scale
            ana = ref[gname][g] if gc is None else ref[gname][g, gc]
            # means2D: the reference's dL_dmeans2D is d/d(ndc) = d/d(pixel) * 0.5 W, so the pixel derivative is scaled back
            if arr == "means2D":
                num = (lp - lm) / (2 * eps)
                ana = ana / (0.5 * (W if c == 0 else H))
            assert abs(num - ana) <= 2e-8 * abs(ana) + 1e-10, (g, arr, c, num, ana)


def test_clamped_pair_gradient_is_transparent():
    """At alpha = min(0.99, o G) = 0.99 the reference's gradient acts as if unclamped: dL/dopacity = G dL/dalpha, not 0."""
    st = dict(W=1, H=1, ranges=np.array([[0, 2]], np.uint32), point_list=np.array([0, 1], np.uint32),
              means2D=np.array([[0.0, 0.0], [0.0, 0.0]]), conic_opacity=np.array([[1.0, 0.0, 1.0, 1.5], [1.0, 0.0, 1.0, 0.5]]),
              colors=np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]), feature=None, depth=None, bg=np.zeros(3),
              g_color=np.ones((3, 1, 1)), g_feature=None, g_alpha=None)
    m = [R64.decide(st, 0)["mask"]]
    assert m[0][0].tolist() == [True, True]
    o = R64.blend(st, m)
    # front pair: alpha 0.99 (clamped), T_k = 1; behind it the second pair weighs 0.5 * 0.01
    dA = 1.0 * 1.0 - (0.5 * 0.01 * 1.0) / (1 - 0.99)
    assert np.isclose(o["dL_dopacity"][0], 1.0 * dA)
    assert np.isclose(o["dL_dconic"][0, 0], 0.0) and np.isclose(o["final_T"][0, 0], 0.01 * 0.5)


SENS_SCENES = ("lists", "term32", "term64", "empty_run", "needles", "offscreen", "opacity", "ragged", "ragged_f32",
               "sh3_big")
GRADS = ("dL_dmeans2D", "dL_dopacity", "dL_dcolors", "dL_dfeature")


def _sens_state(scene):
    import test_blend_pairs_gpu as scenes_gpu
    inp = scenes_gpu.SCENES[scene](3)
    fw, _ = util.run_oracle(inp, backward=False)
    st = oracle_state(inp, fw, depth=fw["depths"], g_alpha=inp["ct"]["dL_dalpha"], g_depth=inp["ct"]["dL_ddepth"])
    T = st["ranges"].shape[0]
    masks = [R64.decide(st, t)["mask"] for t in range(T)]
    return st, masks, R64.blend(st, masks)


@pytest.mark.parametrize("scene", SENS_SCENES)
def test_image_bounds_see_every_single_pair(scene):
    """Removing any one contributing pair from a pixel moves its colour or final_T by more than twice the bound, or
    changes its n_contrib.  Measured fraction of detectable pairs: 1.0 on every scene but needles (0.986): along a needle,
    tens of pixels from its centre, the quadratic's terms reach 1e4, and the fp32 rounding of `power` they carry
    (8 |terms| u in the bound) legitimately outweighs a faint pair blended into the same pixel."""
    st, masks, ref = _sens_state(scene)
    lim_c, lim_t = 2.0 * R64.KAPPA["color"] * R64.U, 2.0 * R64.KAPPA["final_T"] * R64.U
    bg = np.asarray(st["bg"], np.float64)
    seen = total = 0
    for t, m in enumerate(masks):
        if not m.any():
            continue
        p = R64._pairs(st, t)
        a = np.where(m, p["alpha"], 0.0)
        cp = np.cumprod(1.0 - a, 1)
        Tf = cp[:, -1]
        w = a * np.concatenate([np.ones((256, 1)), cp[:, :-1]], 1)
        C = st["colors"][p["ids"]].astype(np.float64)
        wc = w[:, :, None] * C[None]
        Sc = np.cumsum(wc[:, ::-1], 1)[:, ::-1] - wc
        r = a / (1.0 - a)
        dC = -wc + (Sc + (Tf[:, None] * bg[None, :])[:, None, :]) * r[:, :, None]
        dT = Tf[:, None] * r
        x, y = np.where(p["inside"], p["px"], 0), np.where(p["inside"], p["py"], 0)
        det = (np.abs(dC) > lim_c * ref["color_B"][:, y, x].T[:, None, :]).any(2)
        det |= dT > lim_t * ref["final_T_B"][y, x][:, None]
        det |= m & (np.cumsum(m[:, ::-1], 1)[:, ::-1] == 1)
        seen += int((det & m).sum())
        total += int(m.sum())
    print(f"[{scene}] {total} contributing pairs, detectable fraction {seen / total:.5f}")
    assert total > 0 and seen / total >= (0.98 if scene == "needles" else 0.99)


@pytest.mark.parametrize("scene", SENS_SCENES)
def test_gradient_bounds_see_single_pairs(scene):
    """A backward that drops one contributing pair, or adds one listed pair that did not contribute (one pixel-mask bit
    flipped either way), moves some per-Gaussian gradient checked on the GPU (dL_dmeans2D, dL_dopacity, dL_dcolors,
    dL_dfeature) by more than twice its bound.  200 seeded removals per scene; measured detectable fraction 1.0 on lists,
    term32, term64, empty_run, offscreen and sh3_big, 0.99 ragged, 0.975 opacity and ragged_f32 (opacity: pairs behind the opaque stack; ragged_f32 dense: a Gaussian sums
    hundreds of pairs, so one faint pair falls below the sum's rounding), 0.82 needles (the long needles' terms, as for the
    images).  Additions of a footprint pair behind its pixel's stop (weight <= 1e-4 alpha) are measured and printed only:
    1.0 on term32 / term64, 0.33-0.79 where the stop comes late in a dense pixel."""
    st, masks, ref = _sens_state(scene)
    rng = np.random.default_rng(17)
    res = {}
    for kind in ("remove", "add"):
        cand = []
        for t, m in enumerate(masks):
            p = None
            if kind == "remove":
                pp, jj = np.nonzero(m)
            else:
                # a pair inside the footprint that stayed out because its pixel had stopped
                p = R64._pairs(st, t)
                pp, jj = np.nonzero(~m & p["inside"][:, None] & (p["power"] <= 0) & (p["alpha"] >= R64.ALPHA_MIN))
            cand += [(t, a, b) for a, b in zip(pp, jj)]
        if not cand:
            continue
        pick = rng.choice(len(cand), min(200, len(cand)), replace=False)
        seen = 0
        for i in pick:
            t, px, j = cand[i]
            m = masks[t]
            base, flip = R64.new_out(st), R64.new_out(st)
            R64.blend_tile(st, t, m, base)
            m2 = m.copy()
            m2[px, j] = not m2[px, j]
            R64.blend_tile(st, t, m2, flip)
            hit = False
            for q in GRADS:
                d = np.abs(flip[q] - base[q])
                if d.size and (d > 2.0 * R64.KAPPA[q] * R64.U * ref[q + "_B"]).any():
                    hit = True
                    break
            seen += hit
        res[kind] = (seen / len(pick), len(pick))
    print(f"[{scene}] detectable fraction (removals, additions): {res}")
    assert res["remove"][0] >= {"needles": 0.8, "ragged_f32": 0.97, "opacity": 0.97}.get(scene, 0.99)

"""The float64 heads reference (tests/heads_ref64.py) proves itself without a GPU.

* Against torch float64 autograd of independent restatements -- F.cosine_similarity, F.normalize, sigmoid, clamp_max, the
  feature row normalisation and the reference's _ssim expression (tests/test_ssim_gpu.py) -- every value and gradient agrees
  to 1e-9, on edge inputs: |x| in {0, 1e-30, 1e-12, 5e-9, eps (1 +- 1e-6), 1}, zero targets, constant images, x = g, 1x1
  and 5x7 images, zero quaternions and feature rows, opacity +-100, log-scales around ln 0.05.
* oracle/loss_oracle.py agrees with torch's cosine gradient on the same sub-eps pixels.
* A float32 numpy evaluation of the same expressions lands within the bound (the bound is sound where no GPU checks it).
* Its bounds are tight enough to matter: each mutation in heads_ref64.MUTATIONS moves a checked element past twice its
  bound.
"""
import math

import numpy as np
import pytest

import heads_ref64 as R
from project_ref64 import U

f32 = np.float32
NORMS = [0.0, 1e-30, 1e-12, 5e-9, 1e-8 * (1 - 1e-6), 1e-8 * (1 + 1e-6), 1.0]


def _close(got, want, tol=1e-9, floor=1e-300):
    """max |got - want| <= tol max(|want|, floor)"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = max(float(np.abs(want).max(initial=0.0)), floor)
    assert np.abs(got - want).max(initial=0.0) <= tol * scale, float(np.abs(got - want).max() / scale)


def _t(a):
    import torch
    return torch.from_numpy(np.asarray(a, f32).astype(np.float64)).requires_grad_(True)


def _embed_case(F, seed, N=40):
    """[2,F,N] renders whose pixel norms run through NORMS (the rest random), targets with zero pixels"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((2, F, N))
    for i, n in enumerate(NORMS):
        d = rng.standard_normal(F)
        x[:, :, i] = (d / np.linalg.norm(d) * n)[None]
    y = rng.standard_normal((2, F, N))
    y[:, :, [1, 3, len(NORMS) + 1]] = 0.0          # zero targets (with a sub-eps render, a 1e-30 render and a random one)
    y[:, :, len(NORMS) + 2] *= 1e-12                # a sub-eps target
    return x.astype(f32), y.astype(f32)


@pytest.mark.parametrize("F", [1, 3, 32, 67])
def test_loss_heads_match_torch_autograd(F):
    import torch
    import torch.nn.functional as Fn
    x, y = _embed_case(F, F)
    N = x.shape[-1]
    col = np.random.default_rng(F + 1).uniform(-0.2, 1.2, (2, 3, N)).astype(f32)
    tgt = np.random.default_rng(F + 2).uniform(0, 1, (2, 3, N)).astype(f32)
    tgt[:, :, :3] = 0.0
    col[:, :, 3] = tgt[:, :, 3]
    ref = R.loss_heads(col, tgt, x, y, eps=R.COS_EPS)
    xt, ct = _t(x), _t(col)
    cos = Fn.cosine_similarity(xt, _t(y).detach(), dim=1, eps=R.COS_EPS)
    (1 - cos.mean(1)).sum().backward()
    ((ct - _t(tgt).detach()) ** 2).flatten(1).mean(1).sum().backward()
    _close(ref["cos"].v, cos.detach().numpy())
    _close(ref["S_cos"].v, cos.detach().numpy().sum(1))
    _close(ref["S_rgb"].v, ((col.astype(np.float64) - tgt) ** 2).reshape(2, -1).sum(1))
    for i in range(len(NORMS)):  # pixel by pixel: a whole-plane max would hide the tiny-norm pixels
        _close(ref["cot_feature"].v[:, :, i], xt.grad.numpy()[:, :, i])
    _close(ref["cot_feature"].v, xt.grad.numpy())
    _close(ref["cot_color"].v, ct.grad.numpy())


def test_loss_oracle_matches_torch_below_eps():
    """the numpy oracle's cosine gradient is torch's on both sides of eps, at 0 and at zero targets"""
    import torch
    import torch.nn.functional as Fn
    from oracle import loss_oracle as lo
    for F in (3, 32):
        x, y = _embed_case(F, 10 + F)
        for v in range(2):
            xt = torch.from_numpy(x[v].astype(np.float64)).requires_grad_(True)
            cos = Fn.cosine_similarity(xt, torch.from_numpy(y[v].astype(np.float64)), dim=0, eps=lo.EPS)
            (1 - cos.mean()).backward()
            loss, grad = lo.cosine_head(x[v], y[v])
            assert abs(loss - (1 - float(cos.detach().mean()))) <= 1e-12
            for i in range(len(NORMS) + 3):
                _close(grad[:, i], xt.grad.numpy()[:, i])


def _act_inputs(P, F, seed):
    rng = np.random.default_rng(seed)
    g = dict(means=rng.standard_normal((P, 3)), d_means=rng.standard_normal((P, 3)) * 0.1,
             rot=rng.standard_normal((P, 4)), d_rot=rng.standard_normal((P, 4)) * 0.1,
             scales=math.log(0.05) + rng.uniform(-0.5, 0.5, (P, 3)), d_scales=rng.standard_normal((P, 3)) * 0.01,
             opac=rng.standard_normal((P, 1)) * 3, feature=rng.standard_normal((P, F)))
    g["rot"][0] = 0.0
    g["d_rot"][0] = 0.0                       # a zero quaternion
    g["rot"][1] *= 1e-6                       # a tiny one, far above 1e-12
    g["opac"][2], g["opac"][3] = 100.0, -100.0
    g["feature"][0] = 0.0                     # a zero feature row
    g["feature"][1] *= 1e-6                   # a small one
    g = {k: np.asarray(v, f32) for k, v in g.items()}
    gr = dict(g_means=rng.standard_normal((P, 3)), g_rot=rng.standard_normal((P, 4)), g_scales=rng.standard_normal((P, 3)),
              g_opac=rng.standard_normal((P, 1)), g_feature=rng.standard_normal((P, F)))
    return g, {k: np.asarray(v, f32) for k, v in gr.items()}


def test_activations_match_torch_autograd():
    import torch
    import torch.nn.functional as Fn
    g, gr = _act_inputs(64, 7, 3)
    smax = float(f32(0.05))
    ref = R.activate(**g)
    bwd = R.activate_backward(**g, **gr)
    T = {k: _t(v) for k, v in g.items()}
    out = dict(means=T["means"] + T["d_means"], scales=torch.exp(T["scales"] + T["d_scales"]).clamp_max(smax),
               rot=Fn.normalize(T["rot"] + T["d_rot"], dim=1, eps=R.ROT_EPS), opac=torch.sigmoid(T["opac"]),
               feature=T["feature"] / (T["feature"].norm(dim=1, keepdim=True) + R.FEAT_EPS))
    for k, o in out.items():
        o.backward(torch.from_numpy(gr["g_" + k].astype(np.float64)))
    _close(ref["means"].v, out["means"].detach().numpy())
    _close(ref["scales"].v, out["scales"].detach().numpy())
    _close(np.stack([q.v for q in ref["rot"]], 1), out["rot"].detach().numpy())
    _close(ref["opac"].v, out["opac"].detach().numpy())
    _close(ref["feature"].v, out["feature"].detach().numpy())
    _close(bwd["dL_scales"].v, T["scales"].grad.numpy())
    _close(np.stack([q.v for q in bwd["dL_rot"]], 1), T["rot"].grad.numpy())
    _close(bwd["dL_opac"].v, T["opac"].grad.numpy(), 1e-9)
    _close(bwd["dL_feature"].v, T["feature"].grad.numpy())
    for i in (0, 1):  # the zero and the small rows on their own
        _close(bwd["dL_feature"].v[i], T["feature"].grad.numpy()[i])
        _close(np.array([q.v[i] for q in bwd["dL_rot"]]), T["rot"].grad.numpy()[i])


def _torch_ssim_grad(x, g, scale):
    """the reference's _ssim in float64 (tests/test_ssim_gpu.py) and l1, weighted per view by scale: (S [V,C,H,W], grad)"""
    import torch
    import torch.nn.functional as Fn
    xt, gt = _t(x), _t(g).detach()
    C = x.shape[1]
    gauss = torch.tensor([math.exp(-(i - 5) ** 2 / 4.5) for i in range(11)], dtype=torch.float64)
    gauss = gauss / gauss.sum()
    w = (gauss[:, None] @ gauss[None, :]).expand(C, 1, 11, 11).contiguous()
    mu1, mu2 = Fn.conv2d(xt, w, padding=5, groups=C), Fn.conv2d(gt, w, padding=5, groups=C)
    s1 = Fn.conv2d(xt * xt, w, padding=5, groups=C) - mu1 ** 2
    s2 = Fn.conv2d(gt * gt, w, padding=5, groups=C) - mu2 ** 2
    s12 = Fn.conv2d(xt * gt, w, padding=5, groups=C) - mu1 * mu2
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    smap = ((2 * mu1 * mu2 + c1) * (2 * s12 + c2)) / ((mu1 ** 2 + mu2 ** 2 + c1) * (s1 + s2 + c2))
    sc = torch.from_numpy(scale.astype(np.float64))
    total = (sc[:, 0] * (xt - gt).abs().flatten(1).mean(1) + sc[:, 1] * smap.flatten(1).mean(1)).sum()
    total.backward()
    return smap.detach().numpy(), xt.grad.numpy()


def _ssim_images(V, H, W, kind, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-0.1, 1.1, (V, 3, H, W))
    g = rng.uniform(0, 1, (V, 3, H, W))
    if kind == "constant":
        x[:], g[:] = 0.3, 0.7
    elif kind == "equal":
        g = x.copy()
    elif kind == "outside":
        x = rng.uniform(-2, 3, (V, 3, H, W))
    x, g = x.astype(f32), g.astype(f32)
    if kind == "random":
        x[:, 0, ::2, ::3] = g[:, 0, ::2, ::3]  # sign(0) pixels
    return x, g


@pytest.mark.parametrize("hw,kind", [((1, 1), "random"), ((5, 7), "random"), ((5, 7), "constant"), ((5, 7), "equal"),
                                     ((17, 40), "random"), ((17, 40), "outside"), ((11, 11), "equal")])
def test_ssim_matches_torch_autograd(hw, kind):
    V = 2
    x, g = _ssim_images(V, *hw, kind, sum(hw))
    scale = np.random.default_rng(5).uniform(-2, 2, (V, 2)).astype(f32)
    S, grad = _torch_ssim_grad(x, g, scale)
    fw = R.ssim_forward(x, g)
    _close(fw["S"].v, S)
    _close(fw["sum_S"].v, S.reshape(V, -1).sum(1))
    _close(fw["sum_l1"].v, np.abs(x.astype(np.float64) - g).reshape(V, -1).sum(1))
    # at x = g the SSIM gradient is 0 up to float64 cancellation: scale the tolerance to the size of the loss's 1 / N terms
    _close(R.ssim_backward(x, g, fw, scale).v, grad, floor=1.0 / x[0].size)


# --------------------------------------------------------------------------- the bound against a float32 evaluation
def _conv32(a, axis):
    acc = np.zeros_like(a)
    w = R.GAUSS.astype(f32)
    n = a.shape[axis]
    for k in range(11):
        o = k - 5
        s = np.zeros_like(a)
        src = [slice(None)] * a.ndim
        dst = [slice(None)] * a.ndim
        src[axis] = slice(max(o, 0), n + min(o, 0))
        dst[axis] = slice(max(-o, 0), n - max(o, 0))
        s[tuple(dst)] = a[tuple(src)]
        acc = acc + w[k] * s
    return acc


def _ssim32(x, g):
    m = [_conv32(_conv32(a, -1), -2) for a in (x, g, x * x, g * g, x * g)]
    mux, mug = m[0], m[1]
    sxx, sgg, sxg = m[2] - mux * mux, m[3] - mug * mug, m[4] - mux * mug
    c1, c2 = f32(0.01) * f32(0.01), f32(0.03) * f32(0.03)
    A, B = f32(2) * mux * mug + c1, f32(2) * sxg + c2
    Cc, D = mux * mux + mug * mug + c1, sxx + sgg + c2
    inv = f32(1) / (Cc * D)
    S = A * B * inv
    return dict(S=S, dS_dmu=f32(2) * mug * (B - A) * inv - f32(2) * mux * S * (f32(1) / Cc - f32(1) / D), dS_dxx=-S / D,
                dS_dxg=f32(2) * A * inv)


def test_float32_evaluation_is_within_the_bound():
    x, g = _ssim_images(2, 37, 61, "random", 1)
    fw, got = R.ssim_forward(x, g), _ssim32(x, g)
    for k in ("S", "dS_dmu", "dS_dxx", "dS_dxg"):
        assert R.ratio(got[k], fw[k]).max() <= 1.0, k
    xe, ye = _embed_case(32, 4)
    ref = R.loss_heads(feature=xe, tgt_feature=ye)
    xx, yy, xy = (xe * xe).sum(1), (ye * ye).sum(1), (xe * ye).sum(1)
    nx, ny = np.sqrt(xx), np.sqrt(yy)
    inv_nn = f32(1) / (np.maximum(nx, f32(R.COS_EPS)) * np.maximum(ny, f32(R.COS_EPS)))
    cos = xy * inv_nn
    with np.errstate(divide="ignore", invalid="ignore"):
        k = np.where(nx > f32(R.COS_EPS), cos / xx, np.where(nx > 0, cos / (nx * f32(R.COS_EPS)), f32(0)))
    cot = -(f32(1) / f32(xe.shape[-1])) * (ye * inv_nn[:, None] - k[:, None] * xe)
    assert R.ratio(cot, ref["cot_feature"]).max() <= 1.0
    assert R.ratio(cos, ref["cos"]).max() <= 1.0


# --------------------------------------------------------------------------- mutations
def _moves(ref, mut, kappa):
    """largest |mut - ref| / (kappa u e) over the elements"""
    ref = R._arr(ref)
    return float((np.abs(mut.v - ref.v) / (kappa * U * ref.e + 1e-300)).max())


def _mutated(name):
    """(quantity, reference, mutated reference) on a scene where the mutation bites"""
    if name in ("cos_k0_below_eps", "rgb_one_third"):
        x, y = _embed_case(8, 7)
        col = np.random.default_rng(8).uniform(0, 1, (2, 3, x.shape[-1])).astype(f32)
        tgt = np.random.default_rng(9).uniform(0, 1, (2, 3, x.shape[-1])).astype(f32)
        q = "cot_feature" if name == "cos_k0_below_eps" else "cot_color"
        return q, R.loss_heads(col, tgt, x, y)[q], R.loss_heads(col, tgt, x, y, mutate=(name,))[q]
    if name.startswith("ssim"):
        x, g = _ssim_images(1, 20, 70, "random", 2)
        q = "dS_dxg" if name == "ssim_exg_no_2" else "dS_dmu"
        return q, R.ssim_forward(x, g)[q], R.ssim_forward(x, g, mutate=(name,))[q]
    g, gr = _act_inputs(32, 8, 6)
    if name == "sigmoid_bwd_x":
        return "dL_opac", R.activate_backward(**g, **gr)["dL_opac"], R.activate_backward(**g, **gr, mutate=(name,))["dL_opac"]
    return "feature", R.activate(**g)["feature"], R.activate(**g, mutate=(name,))["feature"]


@pytest.mark.parametrize("name", R.MUTATIONS)
def test_each_mutation_moves_a_checked_element_past_twice_its_bound(name):
    q, ref, mut = _mutated(name)
    assert _moves(ref, mut, R.KAPPA[q]) > 2.0, name


def test_halo_shift_shows_at_the_seam_only():
    """the mutation's footprint: the horizontal pass feeds only its own column, so exactly the seam columns x = 32 k move"""
    x, g = _ssim_images(1, 20, 70, "random", 2)
    ref, mut = R.ssim_forward(x, g)["S"], R.ssim_forward(x, g, mutate=("ssim_halo_shift",))["S"]
    moved = np.abs(mut.v - ref.v).reshape(-1, 70).max(0) > 0
    assert np.flatnonzero(moved).tolist() == [32, 64]

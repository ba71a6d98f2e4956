"""MCMC density control without a GPU: the Philox restatement against Random123's known answers, the float64 relocation
maths against gsplat's double sum and its identities, the integer draw's invariants, the C ABI's declarations, state
size and argument errors, and the Python surface's refusals (gaussian_renderer.mcmc_relocate / mcmc_perturb)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import mcmc_ref64 as R
import util
from manigaussian_b200 import _binding
from manigaussian_b200 import gaussian_renderer as GR


def test_philox_known_answers():
    assert [int(w) for w in R.philox4x32_10(0, 0, 0, 0, 0, 0)] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    f = 0xFFFFFFFF
    assert [int(w) for w in R.philox4x32_10(f, f, f, f, f, f)] == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]


def test_mulhi64_is_the_high_word_of_the_product():
    rng = np.random.default_rng(0)
    a = rng.integers(0, 2 ** 63, 200, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    b = rng.integers(0, 2 ** 63, 200, dtype=np.uint64)
    got = R.mulhi64(a, b)
    assert all(int(g) == (int(x) * int(y)) >> 64 for g, x, y in zip(got, a, b))
    assert int(R.mulhi64(np.uint64(2 ** 64 - 1), np.uint64(2 ** 64 - 1))) == 2 ** 64 - 2


@pytest.mark.parametrize("o", [0.005, 0.01, 0.1, 0.3, 0.5, 0.7, 0.9, 0.99, 0.999])
def test_relocation_maths_matches_gsplats_double_sum(o):
    for n in range(1, 52):
        a, r = R.relocation_maths(np.array([o]), np.array([n]))
        wa, wr = R.gsplat_double_sum(o, n)
        assert abs(a[0] - wa) <= 1e-12 * wa, (n, a[0], wa)
        assert abs(r[0] - wr) <= 1e-9 * wr, (n, r[0], wr)


def test_relocation_maths_identities():
    o = np.linspace(0.005, 0.995, 199)
    a, r = R.relocation_maths(o, np.ones_like(o, dtype=np.int64))
    assert np.allclose(a, o, rtol=1e-15, atol=0) and np.allclose(r, 1.0, rtol=0, atol=1e-15)  # n = 1 changes nothing
    for n in (2, 3, 7, 20, 51):
        a, r = R.relocation_maths(o, np.full(o.shape, n))
        assert np.allclose(1.0 - (1.0 - a) ** n, o, rtol=1e-11, atol=0)  # n copies composite to the source's opacity
        assert (a < o).all() and (r > 0).all() and (r <= 1.0).all()


def test_draw_invariants():
    rng = np.random.default_rng(1)
    P_old, P = 5000, 5600
    x = rng.normal(-2.0, 3.0, P).astype(np.float32)
    t = R.dead_threshold(0.005)
    source, m, relocated = R.draw(x, P_old, P, seed=7, offset=3)
    dest = np.concatenate([x[:P_old] <= t, np.ones(P - P_old, bool)])
    assert relocated == dest.sum() == (source >= 0).sum() == m.sum()
    assert (source[~dest] == -1).all()
    assert (x[source[dest]] > t).all()  # only live Gaussians are sources
    # repeatable, and another offset draws other sources
    assert np.array_equal(R.draw(x, P_old, P, 7, 3)[0], source)
    assert not np.array_equal(R.draw(x, P_old, P, 7, 4)[0], source)
    # nothing alive: nothing drawn
    s0, m0, r0 = R.draw(np.full(10, -10.0, np.float32), 10, 12, 7, 3)
    assert (s0 == -1).all() and r0 == 0 and m0.sum() == 0


def test_normals_look_normal():
    z = R.normals(5, 0, 200_000)
    assert abs(z.mean()) < 0.01 and abs(z.std() - 1.0) < 0.01 and np.isfinite(z).all()


# --------------------------------------------------------------------------- C ABI
def test_header_declares_and_the_library_exports_the_mcmc_calls():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    for sym in ("mgs_mcmc_state_bytes", "mgs_mcmc_relocate", "mgs_mcmc_perturb"):
        assert re.search(r"\b%s\s*\(" % sym, hdr)
        assert sym in _binding.EXPORTED_SYMBOLS
        assert hasattr(_binding.lib(), sym)


_S = 4096  # a non-NULL address: every call below fails before it could be used


def _lists(n, width=3, ptr=_S):
    return n, (ctypes.c_void_p * max(n, 1))(*([ptr] * n)), (ctypes.c_int * max(n, 1))(*([width] * n))


def _relocate(**kw):
    a = dict(state=_S, P_old=10, P=12, min_opacity=0.005, means=_S, quats=_S, log_scales=_S, opacity=_S,
             rows=_lists(2), moments=_lists(4), rng=_S, source=_S, relocated=_S)
    a.update(kw)
    return _binding.lib().mgs_mcmc_relocate(a["state"], a["P_old"], a["P"], a["min_opacity"], a["means"], a["quats"],
                                            a["log_scales"], a["opacity"], *a["rows"], *a["moments"], a["rng"], a["source"],
                                            a["relocated"], 0, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(P_old=-1), "0 <= P_old <= P"),
    (dict(P_old=13), "0 <= P_old <= P"),
    (dict(min_opacity=0.0), "min_opacity"),
    (dict(min_opacity=1.0), "min_opacity"),
    (dict(min_opacity=float("nan")), "min_opacity"),
    (dict(state=None), "required"),
    (dict(rng=None), "required"),
    (dict(relocated=None), "required"),
    (dict(source=None), "required"),
    (dict(means=None), "required with P > 0"),
    (dict(quats=None), "required with P > 0"),
    (dict(log_scales=None), "required with P > 0"),
    (dict(opacity=None), "required with P > 0"),
    (dict(rows=_lists(17)), "rows: the count must be in [0, 16]"),
    (dict(rows=(-1, None, None)), "rows: the count"),
    (dict(moments=_lists(65)), "moments: the count must be in [0, 64]"),
    (dict(rows=(2, None, None)), "rows: the pointer and width arrays are required"),
    (dict(moments=_lists(2, width=0)), "moments: every width must be > 0"),
    (dict(rows=_lists(2, ptr=None)), "rows: every pointer is required"),
])
def test_relocate_argument_errors_return_their_code_without_touching_a_gpu(kw, msg):
    assert _relocate(**kw) == -1
    assert msg in _binding.last_error()


@pytest.mark.parametrize("args,msg", [
    ((-1, _S, _S, _S, _S, _S, _S), "P must be >= 0"),
    ((10, _S, _S, _S, _S, _S, None), "rng is required"),
    ((10, None, _S, _S, _S, _S, _S), "required with P > 0"),
    ((10, _S, None, _S, _S, _S, _S), "required with P > 0"),
    ((10, _S, _S, None, _S, _S, _S), "required with P > 0"),
    ((10, _S, _S, _S, None, _S, _S), "required with P > 0"),
    ((10, _S, _S, _S, _S, None, _S), "required with P > 0"),
    ((10, _S, _S + 4, _S, _S, _S, _S), "16-byte aligned"),
])
def test_perturb_argument_errors_return_their_code_without_touching_a_gpu(args, msg):
    assert _binding.lib().mgs_mcmc_perturb(*args, 0, None) == -1
    assert msg in _binding.last_error()


# --------------------------------------------------------------------------- Python surface
def _params(P=8, opacity_shape=None, **over):
    p = {"pts_xyz": torch.zeros(P, 3), "rotations": torch.zeros(P, 4), "scales": torch.zeros(P, 3),
         "opacity": torch.zeros(opacity_shape or (P,))}
    p.update(over)
    return p


_RNG = torch.zeros(2, dtype=torch.int64)


@pytest.mark.parametrize("case,match", [
    (dict(params=[torch.zeros(8, 3)]), "expected a dict with keys"),
    (dict(params={"pts_xyz": torch.zeros(8, 3)}), "expected a dict with keys"),
    (dict(params=_params(pts_xyz=torch.zeros(8, 3, dtype=torch.float64))), "pts_xyz'\\]: expected float32"),
    (dict(params=_params(pts_xyz=torch.zeros(8, 4))), r"pts_xyz'\]: expected \[P,3\]"),
    (dict(params=_params(rotations=torch.zeros(8, 3))), r"rotations'\]: expected \[8,4\]"),
    (dict(params=_params(scales=torch.zeros(7, 3))), r"scales'\]: expected \[8,3\]"),
    (dict(params=_params(opacity=torch.zeros(8, 2))), r"opacity'\]: expected \[8,1\] or \[8\]"),
    (dict(params=_params(sh=torch.zeros(9, 16, 3))), r"sh'\]: expected \[8, ...\]"),
    (dict(params=_params(sh=torch.zeros(8, 16, 3, dtype=torch.float16))), "sh'\\]: expected float32"),
    (dict(params=_params(sh=torch.zeros(8, 3, 16).transpose(1, 2))), "contiguous"),
    (dict(params=_params(sh=torch.zeros(8, 3, device="meta"))), "expected a tensor on cpu"),
    (dict(params=_params(**{f"f{k}": torch.zeros(8, 2) for k in range(17)})), "at most 16 rows"),
    (dict(n=7), "n must be an int >= P = 8"),
    (dict(n=9.0), "n must be an int"),
    (dict(n=True), "n must be an int"),
    (dict(min_opacity=0.0), r"min_opacity must be a number in \(0, 1\)"),
    (dict(min_opacity=1.5), r"min_opacity must be a number in \(0, 1\)"),
    (dict(rng=torch.zeros(2, dtype=torch.int32)), "rng: expected a contiguous int64 \\[2\\]"),
    (dict(rng=torch.zeros(3, dtype=torch.int64)), "rng: expected a contiguous int64 \\[2\\]"),
    (dict(rng=[0, 0]), "rng: expected a contiguous int64 \\[2\\]"),
    (dict(rng=torch.zeros(2, dtype=torch.int64, device="meta")), "rng: expected a tensor on cpu"),
])
def test_mcmc_relocate_rejects_bad_arguments(case, match):
    kw = dict(params=_params(), rng=_RNG)
    kw.update(case)
    with pytest.raises(ValueError, match=match):
        GR.mcmc_relocate(**kw)


def test_mcmc_relocate_refuses_non_leaf_params_with_an_optimizer():
    leaf = torch.zeros(8, 3, requires_grad=True)
    p = _params(pts_xyz=leaf * 2.0)
    opt = torch.optim.Adam([leaf])
    with pytest.raises(ValueError, match="pts_xyz'\\] is not a leaf"):
        GR.mcmc_relocate(p, optimizer=opt, rng=_RNG)


def test_mcmc_relocate_refuses_too_many_moments():
    p = {k: torch.nn.Parameter(v) for k, v in _params(**{f"f{k}": torch.zeros(8, 2) for k in range(16)}).items()}
    opt = torch.optim.Adam(list(p.values()), amsgrad=True)
    for v in p.values():  # a fourth moment per parameter, as an optimizer of its own might keep
        opt.state[v] = {"step": torch.zeros(()), "exp_avg": torch.zeros_like(v), "exp_avg_sq": torch.zeros_like(v),
                        "max_exp_avg_sq": torch.zeros_like(v), "other": torch.zeros_like(v)}
    with pytest.raises(ValueError, match="at most 64 moment tensors, got 80"):
        GR.mcmc_relocate(p, optimizer=opt, rng=_RNG)


@pytest.mark.parametrize("case,match", [
    (dict(pts_xyz=torch.zeros(8, 2)), r"pts_xyz: expected \[P,3\]"),
    (dict(pts_xyz=torch.zeros(3, 8).t()), "pts_xyz: expected \\[P,3\\]|contiguous"),
    (dict(rotations=torch.zeros(8, 4, dtype=torch.float64)), "rotations: expected float32"),
    (dict(scales=torch.zeros(9, 3)), r"scales: expected \[8,3\]"),
    (dict(opacity=torch.zeros(8, 3)), r"opacity: expected \[8,1\] or \[8\]"),
    (dict(scale=torch.zeros(2)), "scale: expected a float32 tensor of one element"),
    (dict(scale=torch.zeros(1, dtype=torch.float64)), "scale: expected a float32 tensor of one element"),
    (dict(scale=float("inf")), "scale: expected a finite number"),
    (dict(scale="1"), "scale: expected a finite number"),
    (dict(rng=torch.zeros(2)), "rng: expected a contiguous int64"),
])
def test_mcmc_perturb_rejects_bad_arguments(case, match):
    kw = dict(pts_xyz=torch.zeros(8, 3), rotations=torch.zeros(8, 4), scales=torch.zeros(8, 3), opacity=torch.zeros(8),
              scale=1.0, rng=_RNG)
    kw.update(case)
    with pytest.raises(ValueError, match=match):
        GR.mcmc_perturb(**kw)


def test_mcmc_has_no_cpu_path():
    with pytest.raises(RuntimeError, match="no CPU path"):
        GR.mcmc_relocate(_params(), rng=_RNG)
    with pytest.raises(RuntimeError, match="no CPU path"):
        GR.mcmc_perturb(torch.zeros(8, 3), torch.zeros(8, 4), torch.zeros(8, 3), torch.zeros(8), 1.0, _RNG)

"""tests/binning_ref.py, the statement of which tile instances a view keeps and in which order, checked without a GPU.

* No cut: with capacity >= R the reference equals the C oracle's duplicateWithKeys -> SortPairs -> identifyTileRanges
  (oracle/gs_oracle.c, the reference rasterizer's own order) bit for bit, on the oracle's projection of random scenes,
  one with exact duplicate Gaussians so that depths tie.
* Cuts: hand-built cases with known answers -- capacity 0, a cut at a Gaussian boundary, a cut inside the first row of
  a 3x3-tile Gaussian and one inside a later row.
* Sensitivity: each broken convention of binning_ref.MUTATIONS changes the result on at least one of these cases.
"""
import numpy as np
import pytest

import binning_ref as B
import util


def _oracle_case(P, W, H, seed, dup=0, scale0=None):
    """The oracle's projection and binning of a util.make_inputs scene; dup > 0 appends exact copies of the first dup
    Gaussians (same depth bits, larger ids)."""
    from oracle import gs_oracle as O
    inp = util.make_inputs(P=P, W=W, H=H, seed=seed, scale0=scale0)
    cam, g = inp["cam"], inp["g"]
    if dup:
        g = {k: (v if not isinstance(v, np.ndarray) or v.ndim == 0 else np.concatenate([v, v[:dup]], 0)) for k, v in g.items()}
    o = O.forward(g["means3D"], g["opacities"], cam["viewmatrix"], cam["projmatrix"], cam["campos"], W, H, cam["tanfovx"],
                  cam["tanfovy"], inp["bg"], scales=g["scales"], rotations=g["rotations"], shs=g["shs"],
                  sh_degree=g["sh_degree"], stages_only=True)
    want = dict(status=np.array([o["num_rendered"], 0]), point_list=o["point_list"],
                tile_ids=(o["point_list_keys"] >> np.uint64(32)).astype(np.uint32), ranges=o["ranges"])
    return dict(radii=o["radii"], means2D=o["means2D"], depths=o["depths"], W=W, H=H), want


ORACLE_CASES = {
    "small": dict(P=500, W=70, H=50, seed=1),
    "f32_like": dict(P=3000, W=200, H=120, seed=3),
    "big_splats": dict(P=400, W=128, H=96, seed=5, scale0=0.04),
    "duplicates": dict(P=800, W=96, H=64, seed=7, dup=300),
    "one_tile": dict(P=200, W=16, H=16, seed=9),
}


@pytest.mark.parametrize("name", list(ORACLE_CASES))
def test_no_cut_equals_the_oracle_bit_for_bit(name):
    case, want = _oracle_case(**ORACLE_CASES[name])
    R = int(want["status"][0])
    assert R > 0
    if name == "duplicates":
        d = case["depths"].view(np.uint32)[case["radii"] > 0]
        assert len(d) - len(np.unique(d)) >= 100, "the duplicates must tie in depth"
    for cap in (R, R + 1, R + 4097):
        got = B.reference(case["radii"], case["means2D"], case["depths"], case["W"], case["H"], cap)
        assert not B.compare(got, want), (cap, B.compare(got, want))
        assert got["status"][1] == 0


# --------------------------------------------------------------------------- hand-built cuts
def _hand():
    """48 x 48 (3 x 3 tiles).  Gaussian 0: centre (24, 24), radius 20 -> all 9 tiles, depth 1.  Gaussian 1: centre (8, 8),
    radius 1 -> tile 0, depth 0.5 (emitted first).  Gaussian 2: centre (40, 8), radius 2 -> tile 2, depth 2 (last).
    Gaussian 3: culled.  Emission: [1@0, 0@0 0@1 0@2, 0@3 0@4 0@5, 0@6 0@7 0@8, 2@2], R = 11."""
    means2D = np.array([[24, 24], [8, 8], [40, 8], [5, 5]], np.float32)
    radii = np.array([20, 1, 2, 0], np.int32)
    depths = np.array([1.0, 0.5, 2.0, np.inf], np.float32)
    return dict(radii=radii, means2D=means2D, depths=depths, W=48, H=48)


def _state(pairs, status):
    """dict of the expected state from the kept (tile, gid) pairs in tile order."""
    tiles = np.array([t for t, _ in pairs], np.int64)
    ranges = np.zeros((9, 2), np.int64)
    for t in np.unique(tiles):
        idx = np.nonzero(tiles == t)[0]
        ranges[t] = (idx[0], idx[-1] + 1)
    return dict(status=np.array(status), point_list=np.array([g for _, g in pairs], np.int64), tile_ids=tiles, ranges=ranges)


HAND = {
    0: _state([], (11, 1)),
    1: _state([(0, 1)], (11, 1)),                                          # at the boundary after Gaussian 1
    3: _state([(0, 1), (0, 0), (1, 0)], (11, 1)),                          # inside Gaussian 0's first row
    6: _state([(0, 1), (0, 0), (1, 0), (2, 0), (3, 0), (4, 0)], (11, 1)),  # inside its second row
    10: _state([(0, 1), (0, 0), (1, 0), (2, 0), (3, 0), (4, 0), (5, 0), (6, 0), (7, 0), (8, 0)], (11, 1)),  # boundary
    11: _state([(0, 1), (0, 0), (1, 0), (2, 0), (2, 2), (3, 0), (4, 0), (5, 0), (6, 0), (7, 0), (8, 0)], (11, 0)),
}


@pytest.mark.parametrize("cap", list(HAND))
def test_hand_built_cuts(cap):
    c = _hand()
    got = B.reference(c["radii"], c["means2D"], c["depths"], c["W"], c["H"], cap)
    assert not B.compare(got, HAND[cap]), B.compare(got, HAND[cap])
    assert list(got["offset"][:3]) == [1, 0, 10] and list(got["count"]) == [9, 1, 1, 0]


def test_tile_rect_is_float32():
    """The rectangle's bounds are float32 expressions, each operation rounded: px = 17 - 2^-19 with r = 16 gives
    px + r = 33 exactly in float32 (a tie, to even), so x1 = (33 + 16 - 1) / 16 = 3, where float64 gives 47.99.. / 16 -> 2.
    Far-off means clamp to the grid."""
    px = np.float32(17.0 - 2.0 ** -19)
    assert float(px) == 17.0 - 2.0 ** -19
    x0, _, x1, _ = B.tile_rect(np.array([[px, 8.0]], np.float32), np.array([16]), 4, 1)
    assert (int(x0[0]), int(x1[0])) == (0, 3)
    assert int((float(px) + 16 + 16 - 1) // 16) == 2
    x0, y0, x1, y1 = B.tile_rect(np.array([[-1e9, 3e9]], np.float32), np.array([5]), 4, 3)
    assert (int(x0[0]), int(x1[0]), int(y0[0]), int(y1[0])) == (0, 0, 3, 3)


# --------------------------------------------------------------------------- sensitivity
def _all_cases():
    c = _hand()
    for cap in HAND:
        yield f"hand cap {cap}", c, cap
    for name in ("small", "duplicates"):
        case, want = _oracle_case(**ORACLE_CASES[name])
        R = int(want["status"][0])
        for cap in (R, R // 2 + 1):
            yield f"{name} cap {cap}", case, cap


@pytest.mark.parametrize("mutation", B.MUTATIONS)
def test_each_mutation_changes_a_case(mutation):
    changed = []
    for name, c, cap in _all_cases():
        ref = B.reference(c["radii"], c["means2D"], c["depths"], c["W"], c["H"], cap)
        mut = B.reference(c["radii"], c["means2D"], c["depths"], c["W"], c["H"], cap, mutate={mutation})
        if B.compare(mut, ref):
            changed.append(name)
    print(mutation, "changes:", changed)
    assert changed, f"{mutation} changes no case"

"""Per-block work lists of the binning stage (binning.cu block_lists_kernel) and the forward's per-block replay bounds.

Every 8x4 pixel block's list must be exactly the tile-list positions whose block bit is set, in list order; the forward's
block_nwalk must end at the block's last contributor, and the pixel mask stored there must name that pixel."""
import numpy as np
import pytest

import util


@pytest.mark.gpu
@pytest.mark.parametrize("W,H,F", [(80, 56, 32), (64, 64, 3)])
def test_block_lists_match_block_bits(W, H, F):
    import torch
    from manigaussian_b200 import rasterizer as R
    inp = util.make_inputs(P=4096, W=W, H=H, F=F, seed=11)
    cam, g = inp["cam"], inp["g"]
    t = util._t
    args = (t(inp["bg"]), t(g["means3D"]), t(g["colors_precomp"]), t(g["feature"]), t(g["opacities"]), t(g["scales"]),
            t(g["rotations"]), 1.0, t(g["cov3D_precomp"]), t(cam["viewmatrix"]), t(cam["projmatrix"]),
            cam["tanfovx"], cam["tanfovy"], H, W, t(g["shs"]), g["sh_degree"], t(cam["campos"]), False, False, True)
    num_rendered, _, _, _, geomB, binB, imgB = R.rasterize_gaussians_raw(*args)[:7]
    torch.cuda.synchronize()
    Rn = num_rendered
    assert Rn > 0
    gx, gy = (W + 15) // 16, (H + 15) // 16
    T = gx * gy
    S = (Rn + 11) & ~3  # row stride of pixel_masks and block_lists

    def arr(which, name, state, a0, a1, dtype, count):
        off = R.state_array(which, name, state, a0, a1) - state.data_ptr()
        nbytes = count * torch.empty((), dtype=dtype).element_size()
        return state[off:off + nbytes].view(dtype).cpu().numpy()

    recs = arr("binning", "records", binB, Rn, 0, torch.int32, 8 * Rn).view(np.uint32).reshape(Rn, 8)
    bits = arr("binning", "block_bits", binB, Rn, 0, torch.uint8, Rn)
    lists = arr("binning", "block_lists", binB, Rn, 0, torch.int32, 8 * S).view(np.uint32).reshape(8, S)
    masks = arr("binning", "pixel_masks", binB, Rn, 0, torch.int32, 8 * S).view(np.uint32).reshape(8, S)
    ranges = arr("image", "ranges", imgB, W, H, torch.int32, 2 * T).view(np.uint32).reshape(T, 2)
    count = arr("image", "block_count", imgB, W, H, torch.int32, 8 * T).view(np.uint32).reshape(T, 8)
    nwalk = arr("image", "block_nwalk", imgB, W, H, torch.int32, 8 * T).view(np.uint32).reshape(T, 8)
    n_contrib = arr("image", "n_contrib", imgB, W, H, torch.int32, W * H).view(np.uint32).reshape(H, W)

    assert np.array_equal(bits, recs[:, 6].astype(np.uint8)), "block_bits must be the records' block masks"
    assert check_block_lists(W, H, ranges, bits, lists, masks, count, nwalk, n_contrib) > 0


def check_block_lists(W, H, ranges, bits, lists, masks, count, nwalk, n_contrib):
    """The block-list invariants of one view's binning state (numpy arrays as read back from its states): every 8x4 block's
    list is exactly the positions of its tile's list whose block bit is set, in order; block_nwalk ends at the block's last
    contributor, and the mask stored there names each pixel's last contributor.  Returns the number of blocks walked."""
    gx = (W + 15) // 16
    walked = 0
    for tile in range(ranges.shape[0]):
        x0, x1 = (int(v) for v in ranges[tile])
        tb = bits[x0:x1]
        tx, ty = tile % gx, tile // gx
        for s in range(8):
            want = np.nonzero((tb >> s) & 1)[0].astype(np.uint32)
            assert count[tile, s] == len(want), (tile, s)
            got = lists[s, x0:x0 + len(want)]
            assert np.array_equal(got, want), (tile, s)
            bx0, by0 = tx * 16 + (s & 1) * 8, ty * 16 + (s >> 1) * 4
            if bx0 >= W or by0 >= H:
                continue  # no pixel of the block is inside the image: neither blend runs it
            nc = n_contrib[by0:by0 + 4, bx0:bx0 + 8]
            m = int(nc.max())
            k = int(nwalk[tile, s])
            if m == 0:
                assert k == 0, (tile, s)
                continue
            walked += 1
            assert 0 < k <= len(want) and got[k - 1] == m - 1, (tile, s, k, m)
            # every pixel's last contributor is an entry of the walked prefix whose mask names that pixel
            for yy in range(nc.shape[0]):
                for xx in range(nc.shape[1]):
                    c = int(nc[yy, xx])
                    if c == 0:
                        continue
                    e = np.nonzero(got[:k] == c - 1)[0]
                    assert len(e) == 1, (tile, s, xx, yy)
                    assert (masks[s, x0 + e[0]] >> (xx * 4 + yy)) & 1, (tile, s, xx, yy)
    return walked

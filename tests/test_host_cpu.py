"""Host-side logic of the layers around the rasterizer (rows f1-f3) that needs no GPU: argument checking, the reference's
call signatures, error codes of the pre-op entry points, and the refusal to run on CPU tensors (no fallback)."""
import inspect

import numpy as np
import pytest
import torch

import util  # noqa: F401  (sys.path)
from manigaussian_b200 import _binding, cameras, gaussian_params, gaussian_renderer


def test_render_keeps_the_reference_signature():
    """agents/manigaussian_bc/gaussian_renderer/__init__.py:17: render(data, idx, pts_xyz, rotations, scales, opacity,
    bg_color, pts_rgb=None, features_color=None, features_language=None); ours only appends optional arguments."""
    params = list(inspect.signature(gaussian_renderer.render).parameters)
    assert params[:10] == ["data", "idx", "pts_xyz", "rotations", "scales", "opacity", "bg_color", "pts_rgb", "features_color",
                           "features_language"]
    sig = inspect.signature(gaussian_renderer.render)
    assert all(sig.parameters[p].default is None for p in ("pts_rgb", "features_color", "features_language"))


def test_no_cpu_fallback_in_the_new_layers():
    P = 8
    z = lambda *s: torch.zeros(*s)
    with pytest.raises(RuntimeError, match="CUDA"):
        gaussian_params.activate_gaussians(z(P, 3), z(P, 4), z(P, 3), z(P, 1))
    with pytest.raises(RuntimeError, match="CUDA"):
        gaussian_renderer.normalize_features(torch.ones(P, 4))
    cb = cameras.build_cameras(np.tile(np.array([[100., 0, 32], [0, 100., 32], [0, 0, 1]]), (2, 1, 1)),
                               np.tile(np.eye(4), (2, 1, 1)), 64, 64)
    with pytest.raises(RuntimeError, match="CUDA"):
        gaussian_renderer.render_views(cb, z(P, 3), z(P, 4), z(P, 3), z(P, 1), pts_rgb=z(P, 3))


def test_argument_checks():
    P = 4
    z = lambda *s: torch.zeros(*s)
    with pytest.raises(ValueError):
        gaussian_params.activate_gaussians(z(P, 3), z(P, 4), z(P, 3), z(P), opacity_activation="tanh")
    cb = cameras.build_cameras(np.array([[100., 0, 32], [0, 100., 32], [0, 0, 1]]), np.eye(4), 64, 64)
    with pytest.raises(ValueError):  # neither SH nor precomputed colours (the reference's exception text is kept)
        gaussian_renderer.render_views(cb, z(P, 3), z(P, 4), z(P, 3), z(P, 1))
    with pytest.raises(ValueError):
        gaussian_renderer.render_views(cb, z(P, 3), z(P, 4), z(P, 3), z(P, 1), pts_rgb=z(P, 3), view_ids=[])


def test_pre_op_entry_points_reject_bad_arguments_without_a_gpu():
    L = _binding.lib()
    assert L.mgs_activate(-1, 0, *([None] * 8), 0, 0.05, 0, 0, 0, *([None] * 6)) < 0
    assert L.mgs_activate(4, 0, *([None] * 8), 7, 0.05, 0, 0, 0, *([None] * 6)) < 0 and "mode" in _binding.last_error()
    assert L.mgs_activate(0, 0, *([None] * 8), 1, 0.05, 1, 1, 1, *([None] * 6)) == 0          # empty cloud: nothing to do
    assert L.mgs_activate_backward(0, 0, *([None] * 8), 1, 0.05, 1, 1, 1, *([None] * 14)) == 0
    # an output requested for an input that is NULL
    assert L.mgs_activate(4, 0, *([None] * 8), 0, 0.05, 0, 0, 0, 4096, None, None, None, None, None) < 0


def test_camera_batch_is_host_resident():
    K = np.array([[120., 0, 40], [0, 110., 30], [0, 0, 1]])
    cb = cameras.build_cameras(np.stack([K, K]), np.stack([np.eye(4), np.eye(4)]), 80, 60)
    nv = cb.as_novel_view()
    s = gaussian_renderer._camera_scalars(nv, 1)
    assert s == (cb.tanfovx[1], cb.tanfovy[1], 60, 80)            # no tensor reads: host scalars
    assert cb.world_view_transform.shape == (2, 4, 4) and cb.camera_center.shape == (2, 3)
    assert cameras.focal2fov(120.0, 80) == pytest.approx(2 * np.arctan(80 / 240.0))
    # identity pose: world->view is the identity, the camera sits at the origin
    np.testing.assert_allclose(cb.host["world_view_transform"][0], np.eye(4), atol=1e-7)
    np.testing.assert_allclose(cb.host["camera_center"][0], 0, atol=1e-7)


def test_packed_gradient_buffer_layout():
    """One flat message for the all-reduce; every field starts on a 16-byte boundary (128-bit reductions target it) and the
    optional precomputed-colour field only exists when asked for."""
    from manigaussian_b200.parallel import FIELDS, PackedGradients, shard_views
    P, F, M = 1001, 32, 4   # odd P: field sizes are not multiples of four floats
    pk = PackedGradients(P, F, M, "cpu")
    base = pk.flat.data_ptr()
    for k, v in pk.views.items():
        assert (v.data_ptr() - base) % 16 == 0, k
        assert v.shape == (P, pk.widths[k]) and v.is_contiguous()
    assert "dL_dcolors" not in pk.views and set(pk.views) <= set(FIELDS)
    assert pk.bytes_per_gaussian == 4 * (3 + 3 + 4 + 1 + 3 * M + F)  # the per-view screen-space gradients are not in the message
    assert "dL_dmeans2D" not in pk.views and "dL_dmeans2D" in PackedGradients(P, F, M, "cpu", means2D=True).views
    assert "dL_dcolors" in PackedGradients(P, 0, 0, "cpu", colors=True).views
    # fields do not overlap
    spans = sorted((v.data_ptr(), v.data_ptr() + v.numel() * 4) for v in pk.views.values())
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
    assert sorted(shard_views(8, 0, 4) + shard_views(8, 1, 4) + shard_views(8, 2, 4) + shard_views(8, 3, 4)) == list(range(8))


def test_binning_capacity_estimator():
    """Host logic of the no-sync forward (rasterizer.py): capacities live in geometric buckets, an observed count grows the
    estimate at once, shrinks it only when the state is more than twice too large, and an overflow is reported and answered
    with a larger margin.  The counts arrive through pinned status slots guarded by events -- faked here."""
    import warnings
    import numpy as np
    from manigaussian_b200 import rasterizer as R

    prev = 0
    for n in [1, 4095, 4097, 10_000, 99_999, 1_000_000, 1_441_792, 5_000_000]:
        c = R._round_capacity(n)
        assert c >= max(n, 4096) and c - max(n, 4096) <= max(1023, 0.125 * n) and c >= prev
        assert R._round_capacity(c) == c  # a bucket boundary is a fixed point: stable sizes keep one cached allocation
        prev = c

    class Ev:
        def __init__(self, done):
            self.done = done

        def query(self):
            return self.done

        def synchronize(self):
            self.done = True

    saved_cap, saved_pending = dict(R._CAPACITY), list(R._PENDING_STATUS)
    try:
        R._CAPACITY.clear()
        R._PENDING_STATUS[:] = []
        key = (0, 1000, 64, 64, 0)
        R._CAPACITY[key] = R._round_capacity(20_000)
        # an unfinished forward is left alone
        R._PENDING_STATUS.append((key, np.array([50_000, 0], np.int32), Ev(False), R._CAPACITY[key]))
        R._poll_status()
        assert R._CAPACITY[key] == R._round_capacity(20_000) and len(R._PENDING_STATUS) == 1
        # finished: grows at once to count * 1.25 + 4096
        R._PENDING_STATUS[0][2].done = True
        R._poll_status()
        assert R._CAPACITY[key] == R._round_capacity(50_000 * 1.25 + 4096) and not R._PENDING_STATUS
        big = R._CAPACITY[key]
        # a somewhat smaller count keeps the allocation; less than half releases it
        R._PENDING_STATUS.append((key, np.array([40_000, 0], np.int32), Ev(True), big))
        R._poll_status()
        assert R._CAPACITY[key] == big
        R._PENDING_STATUS.append((key, np.array([10_000, 0], np.int32), Ev(True), big))
        R._poll_status()
        assert R._CAPACITY[key] == R._round_capacity(10_000 * 1.25 + 4096) < big // 2
        # overflow: warned, and the next capacity carries a 1.5x margin
        cur = R._CAPACITY[key]
        R._PENDING_STATUS.append((key, np.array([60_000, 1], np.int32), Ev(True), cur))
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            R._poll_status()
        assert any("tile instances" in str(x.message) for x in w)
        assert R._CAPACITY[key] == R._round_capacity(60_000 * 1.5 + 4096)
        # block=True waits for the event instead of skipping it
        R._PENDING_STATUS.append((key, np.array([200_000, 0], np.int32), Ev(False), R._CAPACITY[key]))
        R._poll_status(block=True)
        assert R._CAPACITY[key] == R._round_capacity(200_000 * 1.25 + 4096)
    finally:
        R._CAPACITY.clear()
        R._CAPACITY.update(saved_cap)
        R._PENDING_STATUS[:] = saved_pending


def test_allocator_and_library_errors_reach_the_caller():
    """An exception inside the C library's allocation callback (ctypes would print and swallow it) is stashed on the allocator
    and re-raised by the call that triggered it; the allocators are released on every error path."""
    import pytest
    from manigaussian_b200 import rasterizer as R
    from manigaussian_b200 import _binding as B

    class Boom(R._Alloc):
        def alloc(self, nbytes):
            raise MemoryError("no room for %d bytes" % nbytes)

    a, b = Boom("cpu"), R._Alloc("cpu")
    assert a.key in R._Alloc._live and b.key in R._Alloc._live
    assert R._alloc_trampoline(a.key, 1234) == 0 and isinstance(a.error, MemoryError)
    assert R._alloc_trampoline(b.key, 64) != 0 and b.tensor is not None and b.tensor.numel() >= 64
    assert R._alloc_trampoline(987654321, 64) == 0  # unknown user handle: NULL, the library reports MGS_ERR_ALLOC
    with pytest.raises(MemoryError):
        R._checked((a, b), -3, "unit")
    assert a.key not in R._Alloc._live and b.key not in R._Alloc._live
    # a library error code without a stashed exception raises the binding's error and releases too
    c = R._Alloc("cpu")
    with pytest.raises(Exception):
        R._checked((c,), B.lib().mgs_forward_views(0, None, None, 0, 0, 0, 0, None, None, None, None, None, None, 1.0, None, None, 0, 0, None), "unit")
    assert c.key not in R._Alloc._live
    d = R._Alloc("cpu")
    assert R._checked((d,), 7, "unit") == 7 and d.key in R._Alloc._live
    d.release()

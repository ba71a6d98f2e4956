"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol include/mgs_rasterizer.h
declares, the Python mirror keeps the reference's surface, and the product path refuses to run without CUDA."""
import ctypes
import os
import re

import pytest
import torch

import util  # noqa: F401  (sys.path)
from manigaussian_b200 import _binding


def test_library_exports_every_declared_symbol_of_abi_300():
    hdr = open(os.path.join(util.ROOT, "include", "mgs_rasterizer.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(mgs_[a-z_]+)\s*\(", hdr)) - {"mgs_alloc_fn"}
    assert declared, "no declarations parsed"
    L = _binding.lib()
    for sym in sorted(declared):
        assert hasattr(L, sym), f"{sym} declared in include/mgs_rasterizer.h but not exported"
    assert declared == set(_binding.EXPORTED_SYMBOLS)
    assert L.mgs_abi_version() == 300


def test_state_size_queries_are_monotone_and_aligned():
    L = _binding.lib()
    prev = 0
    for P in (0, 1, 1000, 16384, 500000):
        b = L.mgs_geometry_state_bytes(P)
        assert b >= prev and b >= 79 * P
        prev = b
    assert L.mgs_image_state_bytes(256, 256) >= 256 * 256 * 8 + 256 * 8
    assert L.mgs_binning_state_bytes(1000) >= 1000 * (4 + 4 + 4 + 4 + 32)
    assert L.mgs_backward_scratch_bytes(10) >= 10 * 48


def test_invalid_arguments_return_error_codes_without_touching_a_gpu():
    L = _binding.lib()
    cb = _binding.ALLOC_FN(lambda u, n: 0)
    rc = L.mgs_forward(cb, None, cb, None, cb, None, 10, 1, 4, 33, None, 64, 64, None, None, None, None, None, None, 1.0, None,
                       None, None, None, None, 0.3, 0.3, 0, None, None, None, None, 0, None)
    assert rc < 0 and _binding.last_error()
    assert L.mgs_mark_visible(-1, None, None, None, None, None) == -1
    out = ctypes.c_void_p()
    assert L.mgs_state_array(b"geometry", b"nope", ctypes.c_void_p(4096), 10, 0, ctypes.byref(out)) < 0
    assert L.mgs_state_array(b"scratch", b"nope", ctypes.c_void_p(4096), 10, 0, ctypes.byref(out)) < 0
    # the blend-stage records: gb [P][12] at the start of the scratch, gn [P][4] behind it (no device access)
    base = 1 << 20
    assert L.mgs_state_array(b"scratch", b"gb", ctypes.c_void_p(base), 10, 0, ctypes.byref(out)) == 0 and out.value == base
    assert L.mgs_state_array(b"scratch", b"gn", ctypes.c_void_p(base), 10, 0, ctypes.byref(out)) == 0
    assert out.value >= base + 10 * 12 * 4 and out.value % 16 == 0
    assert out.value - base + 10 * 4 * 4 <= L.mgs_backward_scratch_bytes_normal(10)


def test_python_surface_matches_reference():
    import diff_gaussian_rasterization as d
    from manigaussian_b200 import GaussianRasterizationSettings, GaussianRasterizer
    assert d.GaussianRasterizer is GaussianRasterizer
    # reference NamedTuple field order (DGR/diff_gaussian_rasterization/__init__.py:166-179)
    assert GaussianRasterizationSettings._fields == (
        "image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix", "projmatrix", "sh_degree",
        "campos", "prefiltered", "debug", "include_feature")
    for fn in ("rasterize_gaussians", "rasterize_gaussians_backward", "mark_visible"):
        assert callable(getattr(d._C, fn))
    st = GaussianRasterizationSettings(8, 8, 0.3, 0.3, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 1, torch.zeros(3), False,
                                       False, False)
    r = GaussianRasterizer(raster_settings=st)
    m = torch.zeros(4, 3)
    with pytest.raises(Exception, match="SHs or precomputed colors"):
        r(means3D=m, means2D=m, opacities=torch.zeros(4, 1), scales=m, rotations=torch.zeros(4, 4))
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(means3D=m, means2D=m, opacities=torch.zeros(4, 1), shs=torch.zeros(4, 4, 3))


def test_no_cpu_fallback():
    from manigaussian_b200 import GaussianRasterizationSettings, GaussianRasterizer
    st = GaussianRasterizationSettings(8, 8, 0.3, 0.3, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 1, torch.zeros(3), False,
                                       False, False)
    m = torch.rand(4, 3)
    with pytest.raises(RuntimeError, match="no CPU path"):
        GaussianRasterizer(st)(means3D=m, means2D=m, opacities=torch.ones(4, 1), shs=torch.zeros(4, 4, 3), scales=m,
                               rotations=torch.ones(4, 4))


def test_product_package_never_imports_the_oracle():
    import subprocess
    import sys
    code = ("import sys; import manigaussian_b200, diff_gaussian_rasterization; "
            "bad=[m for m in sys.modules if m.startswith('oracle') or 'gs_oracle' in m]; print(bad); sys.exit(1 if bad else 0)")
    r = subprocess.run([sys.executable, "-c", code], cwd=util.ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    for root, _, files in os.walk(os.path.join(util.ROOT, "manigaussian_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(root, f)).read()
                assert "gs_oracle" not in src and "import oracle" not in src and "from oracle" not in src, f

"""Every ctypes mirror in manigaussian_b200/_binding.py has the layout the C compiler gives its struct in
include/mgs_rasterizer.h: a small C probe, compiled with the host compiler nvcc uses, prints sizeof and each field's offsetof,
and both must equal ctypes.sizeof and the mirror's field offsets.  A mirror out of step with the header would hand the
library a wrong pointer, which only shows on the GPU; here it fails on the CPU."""
import ctypes
import os
import shutil
import subprocess

import pytest

import util
from manigaussian_b200 import _binding

MIRRORS = {
    "mgs_view": _binding.View, "mgs_view_alpha": _binding.ViewAlpha, "mgs_view_depth_mask": _binding.ViewDepthMask,
    "mgs_view_ssim": _binding.ViewSsim, "mgs_view_camera_grad": _binding.ViewCameraGrad,
    "mgs_view_intrinsics": _binding.ViewIntrinsics, "mgs_view_median": _binding.ViewMedian, "mgs_view_normal": _binding.ViewNormal,
    "mgs_view_flow": _binding.ViewFlow, "mgs_cloud_flow": _binding.CloudFlow, "mgs_view_fisheye": _binding.ViewFisheye,
    "mgs_view_distortion": _binding.ViewDistortion, "mgs_view_lift": _binding.ViewLift, "mgs_cloud": _binding.Cloud,
    "mgs_render_options": _binding.RenderOptions,
}


@pytest.fixture(scope="module")
def c_layout(tmp_path_factory):
    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "no host C compiler (nvcc needs one too)"
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "mgs_rasterizer.h"', "int main(void) {"]
    for name, mirror in MIRRORS.items():
        lines.append('printf("%s %%zu\\n", sizeof(%s));' % (name, name))
        for field, _ in mirror._fields_:
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (name, field, name, field))
    lines += ["return 0;", "}"]
    d = tmp_path_factory.mktemp("abi_layout")
    src, exe = d / "probe.c", d / "probe"
    src.write_text("\n".join(lines) + "\n")
    subprocess.run([cc, "-std=c99", "-I", os.path.join(util.ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    return {k: int(v) for k, v in (line.split() for line in out.splitlines())}


@pytest.mark.parametrize("name", sorted(MIRRORS))
def test_mirror_matches_the_header(c_layout, name):
    mirror = MIRRORS[name]
    assert ctypes.sizeof(mirror) == c_layout[name], name
    for field, _ in mirror._fields_:
        assert getattr(mirror, field).offset == c_layout[f"{name}.{field}"], (name, field)

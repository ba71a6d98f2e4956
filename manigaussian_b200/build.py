"""Build the sm_90a CUDA library behind the C ABI (include/mgs_rasterizer.h), in-tree.

    python -m manigaussian_b200.build [--force] [--verbose]

Output: manigaussian_b200/lib/libmgs_rasterizer.so (git-ignored).
nvcc cross-compiles for sm_90a without a GPU.  No torch headers are involved: the library is plain
CUDA C++ with a C ABI, loaded from Python with ctypes.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
OBJDIR = os.path.join(LIBDIR, "obj" + (("_" + os.environ["MGS_VARIANT"]) if os.environ.get("MGS_VARIANT") else ""))
# experiment hooks: MGS_VARIANT names an alternative library built with MGS_NVCC_DEFINES (e.g. "-DMGS_FWD_NSUB=4"); the
# default build ignores both
VARIANT = os.environ.get("MGS_VARIANT", "")
EXTRA = os.environ.get("MGS_NVCC_DEFINES", "").split() if VARIANT else []
LIB = os.path.join(LIBDIR, "libmgs_rasterizer%s.so" % (("_" + VARIANT) if VARIANT else ""))
SOURCES = ["project.cu", "project_bwd.cu", "binning.cu", "blend_fwd.cu", "blend_bwd.cu", "loss_heads.cu", "ssim.cu", "activate.cu", "normals.cu", "planar.cu", "flow.cu", "visibility.cu",
           "lift.cu", "field.cu", "knn.cu", "neighbour_reg.cu", "deform.cu", "rays.cu", "fps.cu", "tsdf.cu", "marching_cubes.cu", "mcmc.cu", "densify.cu", "api.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
          "-Xptxas", "-v", "-I", os.path.join(PKG, "..", "include")]


def _deps():
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))]
    files.append(os.path.join(PKG, "..", "include", "mgs_rasterizer.h"))
    files.append(os.path.abspath(__file__))
    return files


def _stamp():
    h = hashlib.sha256()
    for f in _deps():
        with open(f, "rb") as fh:
            h.update(os.path.basename(f).encode())  # not the absolute path: the GPU box unpacks the snapshot elsewhere
            h.update(fh.read())
    h.update(" ".join(EXTRA).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    if os.environ.get("MGS_NO_BUILD") and os.path.exists(LIB):
        return LIB  # profilers that follow child processes (ncu) must not see a compiler being spawned
    os.makedirs(OBJDIR, exist_ok=True)
    stamp_file = os.path.join(LIBDIR, "build%s.stamp" % (("_" + VARIANT) if VARIANT else ""))
    stamp = _stamp()
    if not force and os.path.exists(LIB) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return LIB
    if not os.path.exists(NVCC):
        # a library built from other sources (or for another architecture) must not be loaded in place of this one
        raise RuntimeError(f"nvcc not found at {NVCC}, and {LIB} is missing or was built from other sources")

    def compile_one(src):
        obj = os.path.join(OBJDIR, src.replace(".cu", ".o"))
        cmd = [NVCC] + ARCH + CFLAGS + EXTRA + ["-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, obj, r

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        results = list(ex.map(compile_one, SOURCES))
    log = []
    for src, obj, r in results:
        log.append(f"== {src}\n{r.stdout}{r.stderr}")
        if r.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {src}")
    with open(os.path.join(LIBDIR, "ptxas%s.log" % (("_" + VARIANT) if VARIANT else "")), "w") as fh:
        fh.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    cmd = [NVCC] + ARCH + ["-shared", "-Xcompiler", "-fPIC", "-o", LIB] + [o for _, o, _ in results]
    subprocess.check_call(cmd)
    with open(stamp_file, "w") as fh:
        fh.write(stamp)
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(p)

"""Drop-in module name for simple-knn: `from simple_knn._C import distCUDA2`, as every 3DGS code base imports it, resolves to
this repository's k-nearest-neighbour kernel (manigaussian_b200.gaussian_renderer.knn) when this repository's root is on
sys.path (or the package is installed)."""
from ._C import distCUDA2  # noqa: F401

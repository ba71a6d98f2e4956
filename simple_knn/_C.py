"""Stands in for simple-knn's extension module `_C`."""
from manigaussian_b200.gaussian_renderer import knn


def distCUDA2(points):
    """Per point of `points` [P,3] (float32, CUDA, P >= 4), the mean squared distance to its three nearest other points:
    [P] float32, the value 3DGS turns into initial scales with log(sqrt(clamp_min(dist2, 1e-7))).  The three are the exact
    nearest by fp32 squared distance, ties to the lower index (a duplicate point counts at distance 0); simple-knn's own
    box search may pick differently where it approximates.  Raises ValueError below 4 points, RuntimeError on CPU tensors."""
    import torch
    if not torch.is_tensor(points) or points.dim() != 2 or points.shape[1] != 3:
        raise ValueError(f"distCUDA2: expected points [P,3], got {tuple(points.shape) if torch.is_tensor(points) else type(points)}")
    if points.shape[0] < 4:
        raise ValueError(f"distCUDA2: needs at least 4 points (three neighbours each), got {points.shape[0]}")
    return knn(points, 3)["dist2"].mean(dim=1)

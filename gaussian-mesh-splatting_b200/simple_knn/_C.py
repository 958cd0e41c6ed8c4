"""simple_knn._C.distCUDA2: points [P,3] (CUDA, float32) -> mean squared distance to the three nearest other points [P]."""
from gms_b200.knn import mean_dist2 as distCUDA2

__all__ = ["distCUDA2"]

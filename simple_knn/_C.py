"""`distCUDA2(points)` — same name, argument and result as /root/reference/simple-knn/spatial.cu:15-26: points [P,3] CUDA
float tensor -> float32 [P] mean squared distance to the 3 nearest other points.  Runs this library's own sm_90a kernels
(dreamgaussian_b200/csrc/dgr_knn.cuh) on the current stream; there is no CPU path."""
from dreamgaussian_b200.knn import distCUDA2  # noqa: F401

"""`pytorch3d.loss.chamfer_distance` with pytorch3d's defaults, backed by lidiff_b200.metrics.chamfer_distance (exact fp64 nearest
neighbours on the GPU); non-default arguments raise NotImplementedError."""
from lidiff_b200.metrics import chamfer_distance  # noqa: F401

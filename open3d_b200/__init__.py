"""open3d_b200 — H100-native (sm_90a) implementation of the two dense-geometry
hot paths of Open3D's tensor pipelines: point-to-plane ICP
(``t.pipelines.registration``) and VoxelBlockGrid TSDF integration
(``t.pipelines.slam`` / ``t.geometry.VoxelBlockGrid``).

The compute lives in ``libo3db200.so`` (hand-written CUDA behind the C ABI of
``include/open3d_b200.h``); this package mirrors the reference's Python surface
for that path (same names, argument meaning and error behaviour as
``open3d.t.pipelines.registration`` / ``open3d.t.pipelines.slam`` /
``open3d.t.geometry.VoxelBlockGrid``) with torch CUDA tensors standing in for
``open3d.core.Tensor``.  There is no CPU fallback.
"""
from . import _lib  # noqa: F401  (fails loudly if the shared library is missing)
from . import core, t, utility  # noqa: F401

__version__ = "0.1.0"

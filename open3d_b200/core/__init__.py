"""Boundary helpers standing in for ``open3d.core`` on this path: torch CUDA
tensors carry device memory (cf. core/Tensor.h:1244-1254 DLPack interop), and
``HashMap`` exposes the int32x3 block map of the voxel grid
(core/hashmap/HashMap.cpp:117-216)."""
from __future__ import annotations

import numpy as np
import torch


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)   # what torch.cuda.current_stream() wraps; ~10x cheaper
_has_cuda = None


def current_stream_ptr() -> int:
    global _has_cuda
    if _has_cuda is None:
        _has_cuda = bool(torch.cuda.is_available())
    if not _has_cuda:
        return 0   # the C ABI call that follows fails with O3DB_ERR_CUDA (no CPU fallback)
    if _raw_stream is not None:
        return int(_raw_stream(torch.cuda.current_device()))
    return int(torch.cuda.current_stream().cuda_stream)


def as_device_f32_points(x, name="points") -> torch.Tensor:
    """[N,3] float32 contiguous CUDA tensor (kernel/Registration.cpp:56-59 calls .Contiguous())."""
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(x))
    if not isinstance(x, torch.Tensor):
        raise RuntimeError(f"{name}: expected a torch.Tensor or numpy array")
    if x.dtype != torch.float32:
        # Registration.cpp:119-130 accepts Float32/Float64; this build implements Float32
        raise RuntimeError(f"{name}: only Float32 point clouds are supported by open3d_b200 (got {x.dtype})")
    if x.dim() != 2 or x.shape[1] != 3:
        raise RuntimeError(f"{name}: expected shape [N, 3], got {tuple(x.shape)}")
    if not x.is_cuda and torch.cuda.is_available():
        x = x.cuda()
    # Without a CUDA device the tensor stays on the host so that argument validation can
    # still be exercised; every compute entry point of the C ABI then fails with
    # O3DB_ERR_CUDA (there is no CPU fallback).
    return x.contiguous()


def as_host_f64_4x4(T, name="transformation") -> np.ndarray:
    """Transformation tensors are always 4x4 Float64 on CPU:0 (Registration.h:69-73)."""
    if isinstance(T, torch.Tensor):
        T = T.detach().cpu().numpy()
    T = np.ascontiguousarray(np.asarray(T, dtype=np.float64))
    if T.shape != (4, 4):
        raise RuntimeError(f"{name}: expected shape [4, 4], got {T.shape}")
    return T


from . import nns  # noqa: E402,F401  (uses the helpers above)

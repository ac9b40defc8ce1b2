"""ctypes front-end of the CPU oracle of TransformationEstimationSymmetric and its ICP loop (symmetric_oracle.c).

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle``: importable from tests/ and profiles/, never from
``open3d_b200``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libsymmetric_oracle.so")
_lib = None

_vp = C.c_void_p
_d = C.c_double
_i = C.c_int
_i64 = C.c_int64

ROBUST = {"L2Loss": 0, "L1Loss": 1, "HuberLoss": 2, "CauchyLoss": 3, "GMLoss": 4, "TukeyLoss": 5, "GeneralizedLoss": 6}


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        oracle.lib()   # ../liboracle.so, which this library links (search, transforms, 6x6 solve, robust weights)
        src = os.path.join(_HERE, "symmetric_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-C", _HERE, "libsymmetric_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        for name, res, args in (
                ("orc_sym_sums_f32", None, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _i, _d, _d, _i, _vp]),
                ("orc_sym_means_f32", _i64, [_vp, _vp, _vp, _i64, _vp, _vp]),
                ("orc_pose_to_symmetric_transformation", None, [_vp, _vp, _vp, _vp]),
                ("orc_sym_transformation_f32", _i, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _i, _d, _d, _i, _vp]),
                ("orc_rmse_sym_f32", _d, [_vp, _vp, _vp, _vp, _vp, _i64, _i64]),
                ("orc_icp_sym_f32", _i, [_vp, _vp, _i64, _vp, _vp, _i64, _d, _vp, _i, _d, _d, _i, _d, _d, _i, _vp, _vp,
                                         _vp])):
            getattr(L, name).restype = res
            getattr(L, name).argtypes = args
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32).reshape(-1, 3)


def _corr(c, n):
    c = np.ascontiguousarray(c, np.int64).reshape(-1)
    assert c.shape[0] == n
    return c


def _kernel(kernel):
    """(method, scale, shape) from None, a tuple, or an object with type / scaling_parameter / shape_parameter."""
    if kernel is None:
        return 0, 1.0, 1.0
    if isinstance(kernel, tuple):
        return int(kernel[0]), float(kernel[1]), float(kernel[2])
    return int(kernel.type), float(kernel.scaling_parameter), float(kernel.shape_parameter)


def means(src, tgt, corr):
    """The matched pairs' means, rounded to f32 -> (ms, mt, count)."""
    s, t = _f32(src), _f32(tgt)
    c = _corr(corr, s.shape[0])
    ms, mt = np.zeros(3, np.float32), np.zeros(3, np.float32)
    n = lib().orc_sym_means_f32(s.ctypes.data, t.ctypes.data, c.ctypes.data, s.shape[0], ms.ctypes.data, mt.ctypes.data)
    return ms, mt, int(n)


def sums(src, tgt, src_n, tgt_n, corr, ms, mt, kernel=None, accumulate_f64=False) -> np.ndarray:
    """ComputePoseSymmetricKernelCPU's 29 sums about the given means (f32 accumulators unless accumulate_f64)."""
    s, t, sn, tn = _f32(src), _f32(tgt), _f32(src_n), _f32(tgt_n)
    c = _corr(corr, s.shape[0])
    ms, mt = np.ascontiguousarray(ms, np.float32), np.ascontiguousarray(mt, np.float32)
    out = np.zeros(29, np.float64)
    lib().orc_sym_sums_f32(s.ctypes.data, t.ctypes.data, sn.ctypes.data, tn.ctypes.data, c.ctypes.data, s.shape[0],
                           ms.ctypes.data, mt.ctypes.data, *_kernel(kernel), int(bool(accumulate_f64)), out.ctypes.data)
    return out


def pose_to_transformation(pose, ms, mt) -> np.ndarray:
    """PoseToSymmetricTransformation in f64 (atan, cos, sin and Rodrigues' formula)."""
    p = np.ascontiguousarray(pose, np.float64)
    a, b = np.ascontiguousarray(ms, np.float64), np.ascontiguousarray(mt, np.float64)
    T = np.zeros((4, 4), np.float64)
    lib().orc_pose_to_symmetric_transformation(p.ctypes.data, a.ctypes.data, b.ctypes.data, T.ctypes.data)
    return T


def compute_transformation(src, tgt, src_n, tgt_n, corr, kernel=None, accumulate_f64=False) -> np.ndarray:
    """ComputeTransformationSymmetric -> 4x4 Float64; raises as the reference does."""
    s, t, sn, tn = _f32(src), _f32(tgt), _f32(src_n), _f32(tgt_n)
    c = _corr(corr, s.shape[0])
    T = np.zeros((4, 4), np.float64)
    rc = lib().orc_sym_transformation_f32(s.ctypes.data, t.ctypes.data, sn.ctypes.data, tn.ctypes.data, c.ctypes.data,
                                          s.shape[0], t.shape[0], *_kernel(kernel), int(bool(accumulate_f64)),
                                          T.ctypes.data)
    if rc == -2:
        raise RuntimeError("SymmetricICP correspondences must be -1 or a target point index")
    if rc == 1:
        raise RuntimeError("Singular 6x6 linear system detected, tracking failed.")
    return T


def rmse(src, tgt, src_n, tgt_n, corr) -> float:
    """TransformationEstimationSymmetric::ComputeRMSE."""
    s, t, sn, tn = _f32(src), _f32(tgt), _f32(src_n), _f32(tgt_n)
    c = _corr(corr, s.shape[0])
    v = lib().orc_rmse_sym_f32(s.ctypes.data, t.ctypes.data, sn.ctypes.data, tn.ctypes.data, c.ctypes.data, s.shape[0],
                               t.shape[0])
    if v < 0:
        raise RuntimeError("SymmetricICP correspondences must be -1 or a target point index")
    return float(v)


def icp(source, source_normals, target, target_normals, max_corr_dist, init=None, max_iteration=30,
        relative_fitness=1e-6, relative_rmse=1e-6, kernel=None, accumulate_f64=True) -> oracle.IcpResult:
    """The reference's single-scale loop with the symmetric estimator (points and normals transformed every
    iteration); arguments and result as ``oracle.icp_p2plane``."""
    src, sn, tgt, tn = _f32(source), _f32(source_normals), _f32(target), _f32(target_normals)
    T0 = np.ascontiguousarray(np.eye(4) if init is None else init, np.float64).reshape(16)
    res = oracle._IcpResult()
    per = np.full((max(max_iteration, 1), 2), np.nan, np.float64)
    corr = np.empty(src.shape[0], np.int64)
    rc = lib().orc_icp_sym_f32(src.ctypes.data, sn.ctypes.data, src.shape[0], tgt.ctypes.data, tn.ctypes.data,
                               tgt.shape[0], float(max_corr_dist), T0.ctypes.data, int(max_iteration),
                               float(relative_fitness), float(relative_rmse), *_kernel(kernel),
                               int(bool(accumulate_f64)), C.byref(res), per.ctypes.data, corr.ctypes.data)
    if rc < 0:
        raise MemoryError("orc_icp_sym_f32")
    executed = int(np.sum(~np.isnan(per[:, 0])))
    return oracle.IcpResult(np.array(res.transformation, np.float64).reshape(4, 4), res.fitness, res.inlier_rmse,
                            bool(res.converged), res.num_iterations, per[:executed].copy(), corr, rc)

"""ctypes front-end of the CPU oracle of TransformationEstimationPointToPoint and its ICP loop (p2p_oracle.c).

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
_LIB_PATH = os.path.join(_HERE, "libp2p_oracle.so")
_lib = None

_vp = C.c_void_p


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        oracle.lib()   # ../liboracle.so, which this library links (search, transform)
        src = os.path.join(_HERE, "p2p_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-C", _HERE, "libp2p_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        for name, res, args in (("orc_p2p_sxy_f32", C.c_int64, [_vp, _vp, _vp, C.c_int64, _vp, _vp, _vp]),
                                ("orc_p2p_sxy_f64", C.c_int64, [_vp, _vp, _vp, C.c_int64, _vp, _vp, _vp]),
                                ("orc_rmse_p2p_f32", C.c_double, [_vp, _vp, _vp, C.c_int64]),
                                ("orc_rmse_p2p_f64", C.c_double, [_vp, _vp, _vp, C.c_int64]),
                                ("orc_p2p_kabsch_f64", C.c_int, [_vp, _vp, _vp, _vp]),
                                ("orc_icp_p2p_f32", C.c_int, [_vp, C.c_int64, _vp, C.c_int64, C.c_double, _vp, C.c_int,
                                                              C.c_double, C.c_double, C.c_int, _vp, _vp, _vp])):
            getattr(L, name).restype = res
            getattr(L, name).argtypes = args
        _lib = L
    return _lib


def _inputs(source, target, corr, dtype):
    s = np.ascontiguousarray(source, dtype).reshape(-1, 3)
    t = np.ascontiguousarray(target, dtype).reshape(-1, 3)
    c = np.ascontiguousarray(corr, np.int64).reshape(-1)
    assert c.shape[0] == s.shape[0]
    return s, t, c


def sxy(source, target, corr, dtype=np.float32):
    """Get3x3SxyLinearSystem<dtype> -> (Sxy [3,3] target rows x source columns, target mean, source mean, count);
    a count of 0 is upstream's "No valid correspondence present."."""
    s, t, c = _inputs(source, target, corr, dtype)
    S, mt, ms = np.zeros((3, 3), dtype), np.zeros(3, dtype), np.zeros(3, dtype)
    fn = lib().orc_p2p_sxy_f32 if dtype == np.float32 else lib().orc_p2p_sxy_f64
    count = fn(s.ctypes.data, t.ctypes.data, c.ctypes.data, s.shape[0], S.ctypes.data, mt.ctypes.data, ms.ctypes.data)
    return S, mt, ms, int(count)


def rmse(source, target, corr, dtype=np.float32) -> float:
    """TransformationEstimationPointToPoint::ComputeRMSE."""
    s, t, c = _inputs(source, target, corr, dtype)
    fn = lib().orc_rmse_p2p_f32 if dtype == np.float32 else lib().orc_rmse_p2p_f64
    return float(fn(s.ctypes.data, t.ctypes.data, c.ctypes.data, s.shape[0]))


def kabsch(S, mean_t, mean_s) -> np.ndarray:
    """ComputeRtPointToPointCPU's SVD step + RtToTransformation in f64 -> 4x4; raises for rank < 2."""
    S = np.ascontiguousarray(S, np.float64).reshape(3, 3)
    mt, ms = np.ascontiguousarray(mean_t, np.float64), np.ascontiguousarray(mean_s, np.float64)
    T = np.zeros((4, 4), np.float64)
    if not lib().orc_p2p_kabsch_f64(S.ctypes.data, mt.ctypes.data, ms.ctypes.data, T.ctypes.data):
        raise RuntimeError("Sxy has rank < 2: the rotation is not unique")
    return T


def compute_transformation(source, target, corr, dtype=np.float32) -> np.ndarray:
    """TransformationEstimationPointToPoint::ComputeTransformation -> 4x4 Float64."""
    S, mt, ms, count = sxy(source, target, corr, dtype)
    if count == 0:
        raise RuntimeError("No valid correspondence present.")
    return kabsch(S, mt, ms)


def icp(source, target, max_corr_dist, init=None, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6,
        accumulate_f64=True) -> oracle.IcpResult:
    """The reference's single-scale loop with the point-to-point estimator; arguments and result as
    ``oracle.icp_p2plane``."""
    src = np.ascontiguousarray(source, np.float32).reshape(-1, 3)
    tgt = np.ascontiguousarray(target, np.float32).reshape(-1, 3)
    T0 = np.ascontiguousarray(np.eye(4) if init is None else init, np.float64).reshape(16)
    res = oracle._IcpResult()
    per = np.full((max(max_iteration, 1), 2), np.nan, np.float64)
    corr = np.empty(src.shape[0], np.int64)
    rc = lib().orc_icp_p2p_f32(src.ctypes.data, src.shape[0], tgt.ctypes.data, tgt.shape[0], float(max_corr_dist),
                               T0.ctypes.data, int(max_iteration), float(relative_fitness), float(relative_rmse),
                               int(bool(accumulate_f64)), C.byref(res), per.ctypes.data, corr.ctypes.data)
    if rc < 0:
        raise MemoryError("orc_icp_p2p_f32")
    executed = int(np.sum(~np.isnan(per[:, 0])))
    return oracle.IcpResult(np.array(res.transformation, np.float64).reshape(4, 4), res.fitness, res.inlier_rmse,
                            bool(res.converged), res.num_iterations, per[:executed].copy(), corr, rc)

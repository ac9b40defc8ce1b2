"""ctypes front-end of the CPU oracle of TransformationEstimationForDopplerICP and its ICP loop (doppler_oracle.c).

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
_LIB_PATH = os.path.join(_HERE, "libdoppler_oracle.so")
_lib = None

_vp = C.c_void_p
_d = C.c_double
_i = C.c_int
_i64 = C.c_int64


class Params(C.Structure):
    """orc_dop_params"""
    _fields_ = [("R", C.c_float * 9), ("r", C.c_float * 3), ("period", _d), ("lambda_doppler", _d), ("threshold", _d),
                ("reject", _i), ("min_reject", _i64), ("min_geo", _i64), ("min_dop", _i64), ("method_g", _i),
                ("scale_g", _d), ("shape_g", _d), ("method_d", _i), ("scale_d", _d), ("shape_d", _d)]


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        oracle.lib()
        src = os.path.join(_HERE, "doppler_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-C", _HERE, "libdoppler_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        P = C.POINTER(Params)
        for name, res, args in (
                ("orc_dop_transformation_to_pose", None, [_vp, _vp]),
                ("orc_dop_state", None, [_vp, _d, _vp, _vp]),
                ("orc_dop_precompute", None, [_vp, _vp, _vp, _vp, _vp]),
                ("orc_dop_velocity", None, [P, _vp, _vp]),
                ("orc_dop_sums_f32", None, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, P, _vp, _i64, _i, _vp]),
                ("orc_dop_transformation_f32", _i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, P, _vp, _i64, _i, _vp]),
                ("orc_icp_dop_f32", _i, [_vp, _vp, _vp, _i64, _vp, _vp, _i64, _d, _vp, _i, _d, _d, P, _i, _vp, _vp,
                                         _vp])):
            getattr(L, name).restype = res
            getattr(L, name).argtypes = args
        _lib = L
    return _lib


def _kernel(k):
    if k is None:
        return 0, 1.0, 1.0
    if isinstance(k, tuple):
        return int(k[0]), float(k[1]), float(k[2])
    return int(k.type), float(k.scaling_parameter), float(k.shape_parameter)


def params(period=0.1, lambda_doppler=0.01, reject_dynamic_outliers=False, doppler_outlier_threshold=2.0,
           outlier_rejection_min_iteration=2, geometric_robust_loss_min_iteration=0,
           doppler_robust_loss_min_iteration=2, geometric_kernel=None, doppler_kernel=None,
           transform_vehicle_to_sensor=None) -> Params:
    """The estimator's fields (the C++ constructor's defaults) -> orc_dop_params, with R_S_to_V the f64 (LAPACK)
    inverse of the calibration's rotation block cast to f32, and the constructor's lambda fallback."""
    if lambda_doppler < 0 or lambda_doppler > 1.0:
        lambda_doppler = 0.01
    C4 = np.eye(4) if transform_vehicle_to_sensor is None else np.asarray(transform_vehicle_to_sensor, np.float64)
    p = Params()
    p.R[:] = [float(v) for v in np.linalg.inv(C4[:3, :3]).astype(np.float32).reshape(9)]
    p.r[:] = [float(v) for v in C4[:3, 3].astype(np.float32)]
    p.period, p.lambda_doppler, p.threshold = float(period), float(lambda_doppler), float(doppler_outlier_threshold)
    p.reject = int(bool(reject_dynamic_outliers))
    p.min_reject = int(outlier_rejection_min_iteration)
    p.min_geo = int(geometric_robust_loss_min_iteration)
    p.min_dop = int(doppler_robust_loss_min_iteration)
    p.method_g, p.scale_g, p.shape_g = _kernel(geometric_kernel)
    p.method_d, p.scale_d, p.shape_d = _kernel(doppler_kernel)
    return p


def from_estimator(est) -> Params:
    """params() of an open3d_b200 TransformationEstimationForDopplerICP."""
    return params(est.period, est.lambda_doppler, est.reject_dynamic_outliers, est.doppler_outlier_threshold,
                  est.outlier_rejection_min_iteration, est.geometric_robust_loss_min_iteration,
                  est.doppler_robust_loss_min_iteration, est.geometric_kernel, est.doppler_kernel,
                  est.transform_vehicle_to_sensor)


def _f32(a, cols=3):
    return np.ascontiguousarray(a, np.float32).reshape(-1, cols)


def _T(T):
    return np.ascontiguousarray(np.eye(4) if T is None else T, np.float64).reshape(16)


def state(T, period):
    """(w_v_in_V, v_v_in_V) of T, f32."""
    w, v = np.zeros(3, np.float32), np.zeros(3, np.float32)
    lib().orc_dop_state(_T(T).ctypes.data, float(period), w.ctypes.data, v.ctypes.data)
    return w, v


def transformation_to_pose(T):
    out = np.zeros(6, np.float64)
    lib().orc_dop_transformation_to_pose(_T(T).ctypes.data, out.ctypes.data)
    return out


def velocity(p: Params, T) -> np.ndarray:
    """v_s_in_S for the accumulated transformation T."""
    out = np.zeros(3, np.float32)
    lib().orc_dop_velocity(C.byref(p), _T(T).ctypes.data, out.ctypes.data)
    return out


def sums(src, dops, dirs, tgt, nrm, corr, p: Params, T=None, iteration=0, accumulate_f64=False) -> np.ndarray:
    """The 29 sums of iteration `iteration` at T (f32 accumulators unless accumulate_f64)."""
    s, dr, t, n = _f32(src), _f32(dirs), _f32(tgt), _f32(nrm)
    d = np.ascontiguousarray(dops, np.float32).reshape(-1)
    c = np.ascontiguousarray(corr, np.int64).reshape(-1)
    assert d.shape[0] == c.shape[0] == s.shape[0] == dr.shape[0]
    out = np.zeros(29, np.float64)
    lib().orc_dop_sums_f32(s.ctypes.data, d.ctypes.data, dr.ctypes.data, t.ctypes.data, n.ctypes.data, c.ctypes.data,
                           s.shape[0], C.byref(p), _T(T).ctypes.data, int(iteration), int(bool(accumulate_f64)),
                           out.ctypes.data)
    return out


def compute_transformation(src, dops, dirs, tgt, nrm, corr, p: Params, T=None, iteration=0,
                           accumulate_f64=False) -> np.ndarray:
    s, dr, t, n = _f32(src), _f32(dirs), _f32(tgt), _f32(nrm)
    d = np.ascontiguousarray(dops, np.float32).reshape(-1)
    c = np.ascontiguousarray(corr, np.int64).reshape(-1)
    U = np.zeros(16, np.float64)
    rc = lib().orc_dop_transformation_f32(s.ctypes.data, d.ctypes.data, dr.ctypes.data, t.ctypes.data, n.ctypes.data,
                                          c.ctypes.data, s.shape[0], C.byref(p), _T(T).ctypes.data, int(iteration),
                                          int(bool(accumulate_f64)), U.ctypes.data)
    if rc:
        raise RuntimeError("Singular 6x6 linear system detected, tracking failed.")
    return U.reshape(4, 4)


def icp(source, dopplers, directions, target, target_normals, max_corr_dist, p: Params, init=None, max_iteration=30,
        relative_fitness=1e-6, relative_rmse=1e-6, accumulate_f64=True) -> oracle.IcpResult:
    """The reference's single-scale loop with the Doppler estimator; arguments and result as ``oracle.icp_p2plane``."""
    src, dr, tgt, tn = _f32(source), _f32(directions), _f32(target), _f32(target_normals)
    d = np.ascontiguousarray(dopplers, np.float32).reshape(-1)
    res = oracle._IcpResult()
    per = np.full((max(max_iteration, 1), 2), np.nan, np.float64)
    corr = np.empty(src.shape[0], np.int64)
    rc = lib().orc_icp_dop_f32(src.ctypes.data, d.ctypes.data, dr.ctypes.data, src.shape[0], tgt.ctypes.data,
                               tn.ctypes.data, tgt.shape[0], float(max_corr_dist), _T(init).ctypes.data,
                               int(max_iteration), float(relative_fitness), float(relative_rmse), C.byref(p),
                               int(bool(accumulate_f64)), C.byref(res), per.ctypes.data, corr.ctypes.data)
    if rc < 0:
        raise MemoryError("orc_icp_dop_f32")
    executed = int(np.sum(~np.isnan(per[:, 0])))
    return oracle.IcpResult(np.array(res.transformation, np.float64).reshape(4, 4), res.fitness, res.inlier_rmse,
                            bool(res.converged), res.num_iterations, per[:executed].copy(), corr, rc)

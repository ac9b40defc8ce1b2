"""ctypes front-end of the CPU oracle of PointCloud::SmoothLaplacian, SmoothTaubin, SmoothMLS and SmoothBilateral
(smooth_oracle.c), with the neighbour lists of oracle/knn's brute force and oracle.hybrid_search(bruteforce=True).

device_math=False evaluates exp / acos / cos as libm's f32 functions, as the reference's object code does;
device_math=True evaluates them in f64 and rounds to f32, as the device does.

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle``: importable from tests/ and profiles/, never from
``open3d_b200``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle
from oracle import knn as oknn

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libsmooth_oracle.so")
_lib = None

_vp = C.c_void_p


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its sources."""
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "smooth_oracle.c"), os.path.join(_HERE, "..", "normals", "normals_oracle.c")]
        if not os.path.exists(_LIB_PATH) or max(map(os.path.getmtime, srcs)) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libsmooth_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        for name, args in (
                ("orc_laplacian_pass_f32", [_vp, _vp, C.c_int64, _vp, C.c_int, C.c_double, _vp]),
                ("orc_mls_f32", [_vp, C.c_int64, _vp, _vp, _vp, C.c_int, C.c_double, _vp, _vp, C.c_int]),
                ("orc_bilateral_f32", [_vp, _vp, C.c_int64, _vp, _vp, _vp, C.c_int, C.c_double, C.c_double, _vp,
                                       C.c_int])):
            getattr(L, name).restype = None
            getattr(L, name).argtypes = args
        _lib = L
    return _lib


def _f32(a, cols=3):
    return np.ascontiguousarray(a, np.float32).reshape(-1, cols)


def _ptr(a):
    return None if a is None else a.ctypes.data


def laplacian_pass(points, idx, factor, rows=None):
    """One ApplyLaplacianPass over the neighbour lists idx [len(rows), k'] -> the moved rows [len(rows), 3]
    (rows=None: every row)."""
    p = _f32(points)
    idx = np.ascontiguousarray(idx, np.int32)
    r = None if rows is None else np.ascontiguousarray(rows, np.int64)
    out = np.empty((idx.shape[0], 3), np.float32)
    lib().orc_laplacian_pass_f32(p.ctypes.data, _ptr(r), idx.shape[0], idx.ctypes.data, idx.shape[1], float(factor),
                                 out.ctypes.data)
    return out


def smooth_laplacian(points, iterations, factors, max_nn, fixed_neighborhoods=False):
    """SmoothLaplacian (factors = (lambda,)) or SmoothTaubin (factors = (lambda, mu)) -> [n, 3]; the k' =
    min(n, max_nn + 1) nearest neighbours are searched by brute force before every pass, or once."""
    cur = _f32(points).copy()
    n = cur.shape[0]
    if n == 0 or iterations == 0 or max_nn <= 0:
        return cur
    kp = min(n, max_nn + 1)
    idx = oknn.knn(cur, cur, kp)[0] if fixed_neighborhoods else None
    for _ in range(iterations):
        for f in factors:
            cur = laplacian_pass(cur, idx if fixed_neighborhoods else oknn.knn(cur, cur, kp)[0], f)
    return cur


def mls_neighbours(points, radius, max_nn):
    """SmoothMLS's search -> (idx, d2 or None, cnt or None, stride)."""
    p = _f32(points)
    if radius > 0:
        idx, d2, cnt = oracle.hybrid_search(p, p, radius, max_nn, bruteforce=True)
        return idx, d2, cnt, max_nn
    idx = oknn.knn(p, p, min(p.shape[0], max_nn))[0]
    return idx, None, None, idx.shape[1]


def smooth_mls(points, radius, max_nn, normals=None, device_math=True, lists=None):
    """SmoothMLS(radius, max_nn) -> (positions [n,3], normals [n,3] or None); radius > 0 with max_nn > 0 (hybrid) or
    radius <= 0 with max_nn > 0 (KNN).  lists: mls_neighbours' result, to reuse one search."""
    p = _f32(points)
    out = p.copy()
    nrm = None if normals is None else _f32(normals).copy()
    if p.shape[0] == 0 or (radius <= 0 and max_nn <= 0):
        return out, nrm
    idx, d2, cnt, stride = mls_neighbours(p, radius, max_nn) if lists is None else lists
    lib().orc_mls_f32(p.ctypes.data, p.shape[0], idx.ctypes.data, _ptr(d2), _ptr(cnt), int(stride), float(radius),
                      _ptr(nrm), out.ctypes.data, int(bool(device_math)))
    return out, nrm


def smooth_bilateral(points, normals, radius, max_nn, sigma_s, sigma_r, device_math=True, lists=None):
    """SmoothBilateral(radius, max_nn, sigma_s, sigma_r) on a cloud with normals -> positions [n, 3].  lists: the
    hybrid search's (idx, d2, cnt), to reuse one search."""
    p = _f32(points)
    nrm = _f32(normals)
    out = p.copy()
    if p.shape[0] == 0:
        return out
    idx, d2, cnt = oracle.hybrid_search(p, p, radius, max_nn, bruteforce=True) if lists is None else lists
    lib().orc_bilateral_f32(p.ctypes.data, nrm.ctypes.data, p.shape[0], idx.ctypes.data, d2.ctypes.data,
                            cnt.ctypes.data, int(max_nn), float(sigma_s), float(sigma_r), out.ctypes.data,
                            int(bool(device_math)))
    return out

"""ctypes front-end of the CPU oracle of ComputeFPFHFeature and CorrespondencesFromFeatures (fpfh_oracle.c).

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle``: importable from tests/ and profiles/, never from
``open3d_b200``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libfpfh_oracle.so")
_lib = None

_vp = C.c_void_p


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "fpfh_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libfpfh_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        for name, args in (("orc_fpfh_lists_f32", [_vp, C.c_int64, _vp, C.c_int64, C.c_int, C.c_float, _vp, _vp, _vp]),
                           ("orc_pair_feature_f32", [_vp, _vp, _vp, _vp, _vp]),
                           ("orc_fpfh_f32", [_vp, _vp, C.c_int64, _vp, _vp, _vp, C.c_int, _vp, C.c_int64, _vp]),
                           ("orc_feature_nn_f32", [_vp, C.c_int64, _vp, C.c_int64, C.c_int, _vp])):
            getattr(L, name).restype = None
            getattr(L, name).argtypes = args
        _lib = L
    return _lib


def _f32(a, cols):
    return np.ascontiguousarray(a, np.float32).reshape(-1, cols)


def thr_of(radius):
    """The cap (float)r * (float)r of the hybrid search; +inf for KNN only (radius None)."""
    if radius is None:
        return np.float32(np.inf)
    r = np.float32(radius)
    return np.float32(r * r)


def lists(points, max_nn, radius=None, rows=None):
    """Brute-force neighbour lists of the points `rows` (default all) -> (idx [m, kp] int32, d2 [m, kp] f32,
    cnt [m] int32), kp = min(max_nn, n): the kp nearest with dist^2 <= (float)r^2, ascending by (dist^2, index)."""
    p = _f32(points, 3)
    n = p.shape[0]
    kp = min(int(max_nn), n)
    q = None if rows is None else np.ascontiguousarray(rows, np.int32)
    m = n if q is None else q.shape[0]
    idx = np.empty((m, kp), np.int32)
    d2 = np.empty((m, kp), np.float32)
    cnt = np.empty(m, np.int32)
    if m and kp:
        lib().orc_fpfh_lists_f32(p.ctypes.data, n, None if q is None else q.ctypes.data, m, int(max_nn),
                                 float(thr_of(radius)), idx.ctypes.data, d2.ctypes.data, cnt.ctypes.data)
    return idx, d2, cnt


def fpfh_from_lists(points, normals, idx, d2, cnt, indices=None):
    """FPFH [rows, 33] f32 over the lists of every point; indices selects the distinct rows, ascending."""
    p, nrm = _f32(points, 3), _f32(normals, 3)
    idx = np.ascontiguousarray(idx, np.int32)
    d2 = np.ascontiguousarray(d2, np.float32)
    cnt = np.ascontiguousarray(cnt, np.int32)
    n = p.shape[0]
    sel = None if indices is None else np.unique(np.asarray(indices, np.int64).reshape(-1))
    ns = n if sel is None else sel.shape[0]
    out = np.zeros((ns, 33), np.float32)
    if n and ns:
        lib().orc_fpfh_f32(p.ctypes.data, nrm.ctypes.data, n, idx.ctypes.data, d2.ctypes.data, cnt.ctypes.data,
                           idx.shape[1], None if sel is None else sel.ctypes.data, ns, out.ctypes.data)
    return out


def compute_fpfh_feature(points, normals, max_nn=100, radius=None, indices=None):
    """ComputeFPFHFeature with brute-force lists -> f32 [rows, 33]."""
    idx, d2, cnt = lists(points, max_nn, radius)
    return fpfh_from_lists(points, normals, idx, d2, cnt, indices)


def pair_feature(p1, n1, p2, n2):
    a = [np.ascontiguousarray(x, np.float32).reshape(3) for x in (p1, n1, p2, n2)]
    f = np.zeros(4, np.float32)
    lib().orc_pair_feature_f32(*(x.ctypes.data for x in a), f.ctypes.data)
    return f


def feature_nn(query, target):
    """The nearest target row of each query row (f32 fmaf sum in index order, ties to the lowest index)."""
    q = np.ascontiguousarray(query, np.float32)
    t = np.ascontiguousarray(target, np.float32)
    nn = np.zeros(q.shape[0], np.int64)
    if q.shape[0]:
        lib().orc_feature_nn_f32(q.ctypes.data, q.shape[0], t.ctypes.data, t.shape[0], q.shape[1], nn.ctypes.data)
    return nn


def correspondences_from_features(source, target, mutual_filter=False, mutual_consistency_ratio=0.1):
    """-> (corres int64 [K, 2], fell_back bool)."""
    ij = feature_nn(source, target)
    n = ij.shape[0]
    full = np.stack([np.arange(n, dtype=np.int64), ij], 1)
    if not mutual_filter:
        return full, False
    ji = feature_nn(target, source)
    keep = ji[ij] == np.arange(n)
    if np.float32(keep.sum()) > np.float32(mutual_consistency_ratio) * np.float32(n):
        return full[keep], False
    return full, True

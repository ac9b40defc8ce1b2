"""ctypes front-end of the CPU oracle of RANSAC registration, RegistrationRANSACBasedOnCorrespondence
(ransac_oracle.c), and of the reference's own RegistrationRANSACBasedOnCorrespondence and UniformIntGenerator<int>
compiled into oracle/_ref/libo3dref_ransac.so (oracle/ref_shim_ransac) where the reference sources were readable at
build time.

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle``: importable from tests/ and profiles/, never from
``open3d_b200``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import NamedTuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libransac_oracle.so")
REF_PATH = os.path.join(os.path.dirname(_HERE), "_ref", "libo3dref_ransac.so")
TILE = 128    # the library's tile of the validation sums (kRanTile in open3d_b200/csrc/ransac.cu)
WAVE = 64     # passing hypotheses per validation wave (kRanWave)
BATCH = 8192  # hypotheses drawn per batch (kRanBatch)
_lib = None
_ref = None


class Checkers(C.Structure):
    _fields_ = [("use_edge_length", C.c_int), ("use_distance", C.c_int), ("use_normal", C.c_int),
                ("edge_length_similarity", C.c_double), ("distance_threshold", C.c_double),
                ("cos_normal_angle_threshold", C.c_double)]


class Result(NamedTuple):
    transformation: np.ndarray   # [4, 4] float64
    correspondence_set: np.ndarray   # [n] int64, -1 for none
    drawn: int
    validated: int
    best_index: int
    fitness: float
    rmse: float


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "ransac_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libransac_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        vp = C.c_void_p
        L.orc_ransac.restype = C.c_int
        L.orc_ransac.argtypes = [vp, vp, C.c_int64, vp, vp, C.c_int64, vp, C.c_int64, vp, C.c_int64, C.c_double,
                                 C.c_int, C.c_int, C.c_double, C.POINTER(Checkers), C.c_int64, vp, vp, vp, vp]
        L.orc_ransac_kabsch.argtypes = [vp, vp]
        L.orc_ransac_estimate.argtypes = [vp, vp, vp, C.c_int, vp]
        _lib = L
    return _lib


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, np.float32).reshape(-1, 3)


def checkers(edge=None, distance=None, normal_angle=None):
    """The checker struct: edge length similarity, distance threshold, normal angle (radians; cos taken here)."""
    import math
    return Checkers(int(edge is not None), int(distance is not None), int(normal_angle is not None),
                    float(edge or 0.0), float(distance or 0.0),
                    math.cos(normal_angle) if normal_angle is not None else 0.0)


def ransac(src, tgt, corres, draws, max_dist, ransac_n=3, max_iteration=100000, confidence=0.999, ck=None,
           src_normals=None, tgt_normals=None, tile=TILE):
    """The oracle on the given draws (ints in [0, K)); tile=None sums over the whole source in one sequence."""
    s, t = _f32(src), _f32(tgt)
    sn, tn = _f32(src_normals), _f32(tgt_normals)
    c = np.ascontiguousarray(corres, np.int64).reshape(-1, 2)
    d = np.ascontiguousarray(draws, np.int32).reshape(-1)
    n = s.shape[0]
    T = np.zeros(16, np.float64)
    out = np.empty(max(n, 1), np.int64)
    stats = np.zeros(3, np.int64)
    fr = np.zeros(2, np.float64)
    ck = ck if ck is not None else Checkers()
    rc = lib().orc_ransac(s.ctypes.data, None if sn is None else sn.ctypes.data, n, t.ctypes.data,
                          None if tn is None else tn.ctypes.data, t.shape[0], c.ctypes.data, c.shape[0],
                          d.ctypes.data, d.shape[0], float(max_dist), int(ransac_n), int(max_iteration),
                          float(confidence), C.byref(ck), max(n, 1) if tile is None else int(tile), T.ctypes.data,
                          out.ctypes.data, stats.ctypes.data, fr.ctypes.data)
    if rc == -1:
        raise ValueError("orc_ransac: the run needs more draws than were given")
    if rc:
        raise MemoryError("orc_ransac: out of memory")
    return Result(T.reshape(4, 4), out[:n].copy(), int(stats[0]), int(stats[1]), int(stats[2]), float(fr[0]),
                  float(fr[1]))


def estimate(src, tgt, pairs):
    """The point-to-point estimate of one sample [rn, 2] -> [4, 4]."""
    s, t = _f32(src), _f32(tgt)
    p = np.ascontiguousarray(pairs, np.int64).reshape(-1, 2)
    T = np.zeros(16, np.float64)
    lib().orc_ransac_estimate(s.ctypes.data, t.ctypes.data, p.ctypes.data, p.shape[0], T.ctypes.data)
    T[15] = 1.0
    return T.reshape(4, 4)


def ref() -> C.CDLL | None:
    """The compiled reference, or None where it was not built."""
    global _ref
    if _ref is None and os.path.exists(REF_PATH):
        R = C.CDLL(REF_PATH)
        vp = C.c_void_p
        R.ref_ransac_last_error.restype = C.c_char_p
        R.ref_ransac_seed.argtypes = [C.c_int]
        R.ref_uniform_ints.restype = C.c_int
        R.ref_uniform_ints.argtypes = [C.c_int, C.c_int, C.c_int64, vp]
        R.ref_ransac.restype = C.c_int
        R.ref_ransac.argtypes = [vp, vp, C.c_int64, vp, vp, C.c_int64, vp, C.c_int64, C.c_double, C.c_int, C.c_int,
                                 C.c_double, C.c_int, C.c_double, C.c_int, C.c_double, C.c_int, C.c_double, vp, vp,
                                 C.POINTER(C.c_int64), vp, vp]
        _ref = R
    return _ref


def ref_seed(seed):
    ref().ref_ransac_seed(int(seed))


def ref_uniform_ints(low, high, count):
    out = np.zeros(max(int(count), 1), np.int32)
    if ref().ref_uniform_ints(int(low), int(high), int(count), out.ctypes.data):
        raise RuntimeError(ref().ref_ransac_last_error().decode())
    return out[:int(count)]


class RefResult(NamedTuple):
    transformation: np.ndarray
    correspondence_set: np.ndarray   # [n] int64, -1 for none, from upstream's pair list
    validations: int                 # from upstream's summary line (-1 when it returned before the loop)
    warnings: int
    fitness: float
    rmse: float


def ref_ransac(src, tgt, corres, max_dist, ransac_n=3, max_iteration=100000, confidence=0.999, edge=None,
               distance=None, normal_angle=None, src_normals=None, tgt_normals=None):
    """The reference's RegistrationRANSACBasedOnCorrespondence on its own engine; raises RuntimeError with its
    message."""
    s, t = _f32(src), _f32(tgt)
    sn, tn = _f32(src_normals), _f32(tgt_normals)
    c = np.ascontiguousarray(corres, np.int64).reshape(-1, 2)
    n = s.shape[0]
    T = np.zeros(16, np.float64)
    pairs = np.zeros((max(n, 1), 2), np.int64)
    k = C.c_int64()
    fr = np.zeros(2, np.float64)
    st = np.zeros(2, np.int64)
    rc = ref().ref_ransac(s.ctypes.data, None if sn is None else sn.ctypes.data, n, t.ctypes.data,
                          None if tn is None else tn.ctypes.data, t.shape[0], c.ctypes.data, c.shape[0],
                          float(max_dist), int(ransac_n), int(max_iteration), float(confidence), int(edge is not None),
                          float(edge or 0.0), int(distance is not None), float(distance or 0.0),
                          int(normal_angle is not None), float(normal_angle or 0.0), T.ctypes.data, pairs.ctypes.data,
                          C.byref(k), fr.ctypes.data, st.ctypes.data)
    if rc:
        raise RuntimeError(ref().ref_ransac_last_error().decode())
    cs = np.full(n, -1, np.int64)
    cs[pairs[:k.value, 0]] = pairs[:k.value, 1]
    return RefResult(T.reshape(4, 4), cs, int(st[0]), int(st[1]), float(fr[0]), float(fr[1]))

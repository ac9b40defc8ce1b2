"""ctypes front-end of the CPU oracle of RANSAC plane segmentation, PointCloud::SegmentPlane (segment_oracle.c), and
of the reference's own SegmentPlane and RandomSampler compiled into oracle/_ref/libo3dref_segment.so
(oracle/ref_shim_segment) where the reference sources were readable at build time.

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
_LIB_PATH = os.path.join(_HERE, "libsegment_oracle.so")
REF_PATH = os.path.join(os.path.dirname(_HERE), "_ref", "libo3dref_segment.so")
TILE = 1024   # the library's tile of the score and refit sums (kSegTile in open3d_b200/csrc/segment.cu)
_lib = None
_ref = None


class Result(NamedTuple):
    plane: np.ndarray      # [4] float64
    inliers: np.ndarray    # [K] int64, ascending
    best_index: int        # -1 for none (None from the reference, which does not report it)
    evaluated: int
    fitness: float
    rmse: float


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "segment_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libsegment_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        L.orc_segment_plane.restype = C.c_int
        L.orc_segment_plane.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double,
                                        C.c_int64, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p,
                                        C.c_void_p]
        _lib = L
    return _lib


def ref() -> C.CDLL | None:
    """The compiled reference, or None where it was not built."""
    global _ref
    if _ref is None and os.path.exists(REF_PATH):
        R = C.CDLL(REF_PATH)
        R.ref_segment_last_error.restype = C.c_char_p
        R.ref_random_seed.argtypes = [C.c_int]
        R.ref_random_sample.argtypes = [C.c_int64, C.c_int, C.c_int, C.c_void_p]
        R.ref_segment_plane.restype = C.c_int
        R.ref_segment_plane.argtypes = [C.c_void_p, C.c_int64, C.c_double, C.c_int, C.c_int, C.c_double, C.c_void_p,
                                        C.c_void_p, C.POINTER(C.c_int64), C.c_void_p, C.POINTER(C.c_int64)]
        _ref = R
    return _ref


def _f32(points):
    return np.ascontiguousarray(points, np.float32).reshape(-1, 3)


def segment_plane(points, samples, distance_threshold, probability=0.999, tile=TILE):
    """The oracle on the given samples [num_iterations, ransac_n]; tile=None sums over the whole cloud in one
    sequence, upstream's order."""
    p = _f32(points)
    s = np.ascontiguousarray(samples, np.int64)
    H, rn = s.shape
    n = p.shape[0]
    plane = np.zeros(4, np.float64)
    inl = np.empty(max(n, 1), np.int64)
    k = C.c_int64()
    stats = np.zeros(2, np.int64)
    fr = np.zeros(2, np.float64)
    rc = lib().orc_segment_plane(p.ctypes.data, n, s.ctypes.data, H, rn, float(distance_threshold),
                                 float(probability), max(n, 1) if tile is None else int(tile), plane.ctypes.data,
                                 inl.ctypes.data, C.byref(k), stats.ctypes.data, fr.ctypes.data)
    if rc == -2:
        raise MemoryError("orc_segment_plane: out of memory")
    if rc:
        raise ValueError(f"orc_segment_plane: bad arguments (n={n}, ransac_n={rn}, probability={probability})")
    return Result(plane, inl[:k.value].copy(), int(stats[0]), int(stats[1]), float(fr[0]), float(fr[1]))


def ref_seed(seed):
    ref().ref_random_seed(int(seed))


def ref_samples(n, ransac_n, num_iterations):
    """[num_iterations, ransac_n] int64: what the reference's SegmentPlane draws from its engine."""
    out = np.zeros((max(num_iterations, 0), ransac_n), np.int64)
    ref().ref_random_sample(int(n), int(ransac_n), max(int(num_iterations), 0), out.ctypes.data)
    return out


def ref_segment_plane(points, distance_threshold=0.01, ransac_n=3, num_iterations=100, probability=0.999):
    """The reference's SegmentPlane on its own engine; raises RuntimeError with its message."""
    p = _f32(points)
    n = p.shape[0]
    plane = np.zeros(4, np.float64)
    inl = np.empty(max(n, 1), np.int64)
    k = C.c_int64()
    dbg = np.zeros(2, np.float64)
    ev = C.c_int64()
    rc = ref().ref_segment_plane(p.ctypes.data, n, float(distance_threshold), int(ransac_n), int(num_iterations),
                                 float(probability), plane.ctypes.data, inl.ctypes.data, C.byref(k), dbg.ctypes.data,
                                 C.byref(ev))
    if rc:
        raise RuntimeError(ref().ref_segment_last_error().decode())
    return Result(plane, inl[:k.value].copy(), None, ev.value, float(dbg[0]), float(dbg[1]))

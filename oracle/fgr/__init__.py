"""ctypes front-end of the CPU oracle of Fast Global Registration, FastGlobalRegistrationBasedOnCorrespondence and
FastGlobalRegistrationBasedOnFeatureMatching (fgr_oracle.c), and of the reference's own functions compiled into
oracle/_ref/libo3dref_fgr.so (oracle/ref_shim_fgr) where the reference sources were readable at build time.

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
_LIB_PATH = os.path.join(_HERE, "libfgr_oracle.so")
REF_PATH = os.path.join(os.path.dirname(_HERE), "_ref", "libo3dref_fgr.so")
TILE = 128      # the library's tile of the evaluation sums (kFgrTile in open3d_b200/csrc/fgr.cu)
BATCH = 16384   # tuple trials drawn per batch (kFgrBatch)
_lib = None
_ref = None


class Option(C.Structure):
    _fields_ = [("division_factor", C.c_double), ("use_absolute_scale", C.c_int), ("decrease_mu", C.c_int),
                ("maximum_correspondence_distance", C.c_double), ("iteration_number", C.c_int),
                ("tuple_scale", C.c_double), ("maximum_tuple_count", C.c_int), ("tuple_test", C.c_int)]


def option(division_factor=1.4, use_absolute_scale=False, decrease_mu=False, maximum_correspondence_distance=0.025,
           iteration_number=64, tuple_scale=0.95, maximum_tuple_count=1000, tuple_test=True):
    """The option struct, with the defaults of upstream's Python binding."""
    return Option(float(division_factor), int(bool(use_absolute_scale)), int(bool(decrease_mu)),
                  float(maximum_correspondence_distance), int(iteration_number), float(tuple_scale),
                  int(maximum_tuple_count), int(bool(tuple_test)))


class Result(NamedTuple):
    transformation: np.ndarray       # [4, 4] float64
    correspondence_set: np.ndarray   # [n] int64, -1 for none
    tuples: int
    trials: int                      # tuple trials consumed: the engine advanced by 3 x trials
    pairs: np.ndarray                # [P, 2] int64: the pairs the optimisation ran on
    warned: bool                     # the "not enough correspondences" warning
    fitness: float
    rmse: float


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "fgr_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libfgr_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        vp = C.c_void_p
        L.orc_fgr.restype = C.c_int
        L.orc_fgr.argtypes = [vp, C.c_int64, vp, C.c_int64, vp, C.c_int64, C.c_int, vp, C.c_int64, C.POINTER(Option),
                              C.c_int64, vp, vp, vp, vp, vp]
        L.orc_fgr_ldlt_solve6.argtypes = [vp, vp]
        L.orc_fgr_vec6_to_mat4.argtypes = [vp, vp]
        L.orc_fgr_inverse4.argtypes = [vp, vp]
        L.orc_fgr_sincos.restype = C.c_double
        L.orc_fgr_sincos.argtypes = [C.c_double, C.c_int]
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32).reshape(-1, 3)


def mutual_pairs(source_feature, target_feature, source_is_query=True):
    """InitialMatching's mutual nearest rows (f32 distances, ties to the lowest row, oracle.fpfh.feature_nn), in
    ascending query row: (source, target) pairs, or (target, source) pairs when the target's rows are the queries."""
    from oracle import fpfh
    fs = np.ascontiguousarray(source_feature, np.float32)
    ft = np.ascontiguousarray(target_feature, np.float32)
    q, t = (fs, ft) if source_is_query else (ft, fs)
    if len(q) == 0 or len(t) == 0:
        return np.zeros((0, 2), np.int64)
    ij, ji = fpfh.feature_nn(q, t), fpfh.feature_nn(t, q)
    keep = np.nonzero(ji[ij] == np.arange(len(q)))[0]
    return np.stack([keep, ij[keep]], 1).astype(np.int64)


def fgr(src, tgt, corres, draws, opt=None, swapped=False, tile=TILE):
    """The oracle on the given draws (ints in [0, K)); corres are (target, source) pairs when swapped; tile=None sums
    over the whole source in one sequence.  Raises RuntimeError for an invalid scale."""
    s, t = _f32(src), _f32(tgt)
    c = np.ascontiguousarray(corres, np.int64).reshape(-1, 2)
    d = np.ascontiguousarray(draws, np.int32).reshape(-1)
    opt = option() if opt is None else opt
    n, K = s.shape[0], c.shape[0]
    T = np.zeros(16, np.float64)
    out = np.empty(max(n, 1), np.int64)
    stats = np.zeros(4, np.int64)
    fr = np.zeros(3, np.float64)
    # the optimiser's pairs: the K given, or 3 per passing trial, at most min(maximum_tuple_count, 100 K) trials
    tuples = max(1, min(opt.maximum_tuple_count, 100 * K))
    pairs = np.zeros((max(K, 3 * tuples, 1), 2), np.int64)
    rc = lib().orc_fgr(s.ctypes.data, n, t.ctypes.data, t.shape[0], c.ctypes.data, K, int(bool(swapped)),
                       d.ctypes.data, d.shape[0], C.byref(opt), max(n, 1) if tile is None else int(tile), T.ctypes.data,
                       out.ctypes.data, stats.ctypes.data, fr.ctypes.data, pairs.ctypes.data)
    if rc == -1:
        raise ValueError("orc_fgr: the run needs more draws than were given")
    if rc == -3:
        raise RuntimeError(f"Invalid scale_global: {fr[2]}, it must be > 0.")
    if rc:
        raise MemoryError("orc_fgr: out of memory")
    return Result(T.reshape(4, 4), out[:n].copy(), int(stats[0]), int(stats[1]), pairs[:stats[2]].copy(),
                  bool(stats[3]), float(fr[0]), float(fr[1]))


def fgr_features(src, tgt, source_feature, target_feature, draws, opt=None, tile=TILE):
    """The feature call: the mutual pairs with the smaller cloud's rows as the queries when the tuple test runs (the
    source's when the sizes are equal or the test is off), then fgr."""
    opt = option() if opt is None else opt
    swapped = bool(opt.tuple_test) and len(src) < len(tgt)
    c = mutual_pairs(source_feature, target_feature, not swapped)
    return fgr(src, tgt, c, draws, opt, swapped, tile), len(c)


def ldlt_solve(A, b):
    """The stated LDLT solve of the 6x6 A x = b."""
    a = np.ascontiguousarray(A, np.float64).copy()
    x = np.ascontiguousarray(b, np.float64).copy()
    lib().orc_fgr_ldlt_solve6(a.ctypes.data, x.ctypes.data)
    return x


def vec6_to_mat4(x):
    v = np.ascontiguousarray(x, np.float64)
    D = np.zeros(16, np.float64)
    lib().orc_fgr_vec6_to_mat4(v.ctypes.data, D.ctypes.data)
    return D.reshape(4, 4)


def inverse4(M):
    a = np.ascontiguousarray(M, np.float64)
    out = np.zeros(16, np.float64)
    lib().orc_fgr_inverse4(a.ctypes.data, out.ctypes.data)
    return out.reshape(4, 4)


def ref() -> C.CDLL | None:
    """The compiled reference, or None where it was not built."""
    global _ref
    if _ref is None and os.path.exists(REF_PATH):
        R = C.CDLL(REF_PATH)
        vp = C.c_void_p
        R.ref_fgr_last_error.restype = C.c_char_p
        R.ref_fgr_seed.argtypes = [C.c_int]
        R.ref_fgr_uniform_ints.restype = C.c_int
        R.ref_fgr_uniform_ints.argtypes = [C.c_int, C.c_int, C.c_int64, vp]
        R.ref_fgr_ldlt_solve6.argtypes = [vp, vp, vp]
        R.ref_fgr_inverse4.argtypes = [vp, vp]
        R.ref_fgr_vec6_to_mat4.argtypes = [vp, vp]
        R.ref_fgr_sincos.restype = C.c_double
        R.ref_fgr_sincos.argtypes = [C.c_double, C.c_int]
        R.ref_fgr.restype = C.c_int
        R.ref_fgr.argtypes = [vp, C.c_int64, vp, C.c_int64, vp, C.c_int64, vp, vp, C.c_int, C.POINTER(Option), vp, vp,
                              C.POINTER(C.c_int64), vp, vp]
        _ref = R
    return _ref


def ref_ldlt_solve(A, b):
    """The shim's Eigen stub: A.ldlt().solve(b) for a 6x6 A."""
    a = np.ascontiguousarray(A, np.float64)
    v = np.ascontiguousarray(b, np.float64)
    x = np.zeros(6, np.float64)
    ref().ref_fgr_ldlt_solve6(a.ctypes.data, v.ctypes.data, x.ctypes.data)
    return x


def ref_inverse4(M):
    a = np.ascontiguousarray(M, np.float64)
    out = np.zeros(16, np.float64)
    ref().ref_fgr_inverse4(a.ctypes.data, out.ctypes.data)
    return out.reshape(4, 4)


def ref_vec6_to_mat4(x):
    v = np.ascontiguousarray(x, np.float64)
    out = np.zeros(16, np.float64)
    ref().ref_fgr_vec6_to_mat4(v.ctypes.data, out.ctypes.data)
    return out.reshape(4, 4)


def sincos(x, want_cos):
    return lib().orc_fgr_sincos(float(x), int(want_cos))


def ref_sincos(x, want_cos):
    return ref().ref_fgr_sincos(float(x), int(want_cos))


def ref_seed(seed):
    ref().ref_fgr_seed(int(seed))


def ref_uniform_ints(low, high, count):
    out = np.zeros(max(int(count), 1), np.int32)
    if ref().ref_fgr_uniform_ints(int(low), int(high), int(count), out.ctypes.data):
        raise RuntimeError(ref().ref_fgr_last_error().decode())
    return out[:int(count)]


class RefResult(NamedTuple):
    transformation: np.ndarray
    correspondence_set: np.ndarray   # [n] int64, -1 for none, from upstream's pair list
    cross: int                       # from upstream's "Initial matchings" line (-1 without it)
    tuples: int                      # from upstream's tuple summary line (-1 without it)
    trials: int                      # the trials consumed, from the same line
    warnings: int
    fitness: float
    rmse: float


def ref_fgr(src, tgt, opt=None, corres=None, source_feature=None, target_feature=None):
    """The reference's FastGlobalRegistrationBasedOnCorrespondence (corres given) or ...BasedOnFeatureMatching, on its
    own engine; raises RuntimeError with its message."""
    s, t = _f32(src), _f32(tgt)
    opt = option() if opt is None else opt
    n = s.shape[0]
    T = np.zeros(16, np.float64)
    pairs = np.zeros((max(n, 1), 2), np.int64)
    k = C.c_int64()
    fr = np.zeros(2, np.float64)
    st = np.zeros(5, np.int64)
    if corres is not None:
        c = np.ascontiguousarray(corres, np.int64).reshape(-1, 2)
        args = (c.ctypes.data, c.shape[0], None, None, 0)
    else:
        fs = np.ascontiguousarray(source_feature, np.float32)
        ft = np.ascontiguousarray(target_feature, np.float32)
        args = (None, 0, fs.ctypes.data, ft.ctypes.data, fs.shape[1])
    rc = ref().ref_fgr(s.ctypes.data, n, t.ctypes.data, t.shape[0], *args, C.byref(opt), T.ctypes.data,
                       pairs.ctypes.data, C.byref(k), fr.ctypes.data, st.ctypes.data)
    if rc:
        raise RuntimeError(ref().ref_fgr_last_error().decode())
    cs = np.full(n, -1, np.int64)
    cs[pairs[:k.value, 0]] = pairs[:k.value, 1]
    return RefResult(T.reshape(4, 4), cs, int(st[0]), int(st[1]), int(st[2]), int(st[3]), float(fr[0]), float(fr[1]))

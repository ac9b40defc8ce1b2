"""The FPFH oracle (oracle/fpfh) against the reference's own ComputePairFeature and ComputeFPFHFeatureCPU, compiled from
its headers into oracle/_ref/libo3dref_fpfh.so (oracle/ref_shim_fpfh), on the same neighbour lists.  Every comparison
is bit for bit.  Also the oracle's brute-force lists against the KNN oracle, its indices path against its full rows,
and its feature 1-NN and mutual filter against numpy.  CPU only."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import fpfh as of
from tests import fpfh_cases as fc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libo3dref_fpfh.so")
_vp = C.c_void_p
CASES = fc.cases()


@pytest.fixture(scope="module")
def ref():
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref/libo3dref_fpfh.so not built (needs the reference sources)")
    L = C.CDLL(REF)
    L.ref_pair_feature_f32.restype = None
    L.ref_pair_feature_f32.argtypes = [_vp] * 5
    L.ref_compute_fpfh_feature_f32.restype = None
    L.ref_compute_fpfh_feature_f32.argtypes = [_vp, _vp, C.c_int64, _vp, _vp, C.c_int64, _vp, _vp]
    return L


def _ref_fpfh(L, pts, nrm, idx, d2, cnt):
    pts, nrm = np.ascontiguousarray(pts, np.float32), np.ascontiguousarray(nrm, np.float32)
    out = np.zeros((len(pts), 33), np.float32)
    L.ref_compute_fpfh_feature_f32(pts.ctypes.data, nrm.ctypes.data, len(pts), idx.ctypes.data, d2.ctypes.data,
                                   idx.shape[1], cnt.ctypes.data, out.ctypes.data)
    return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_reference(ref, name):
    pts, nrm, radius, max_nn = CASES[name]
    idx, d2, cnt = of.lists(pts, max_nn, radius)
    want = _ref_fpfh(ref, pts, nrm, idx, d2, cnt)
    got = of.fpfh_from_lists(pts, nrm, idx, d2, cnt)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    # the indices path: each selected row is the full call's row
    sel = np.random.default_rng(1).integers(0, len(pts), 300)
    assert np.array_equal(of.fpfh_from_lists(pts, nrm, idx, d2, cnt, sel).view(np.int32),
                          want[np.unique(sel)].view(np.int32))


# radius 0.1 gives lists of 22..84 points, 0.15 of 47..128 (cut at max_nn 80 / 100 / 128)
@pytest.mark.parametrize("max_nn", [4, 30, 80, 100, 128])
@pytest.mark.parametrize("radius", [None, 0.04, 0.1, 0.15])
def test_oracle_equals_reference_max_nn(ref, max_nn, radius):
    pts, nrm = fc.scan(3000, 36)
    idx, d2, cnt = of.lists(pts, max_nn, radius)
    want = _ref_fpfh(ref, pts, nrm, idx, d2, cnt)
    assert np.array_equal(of.fpfh_from_lists(pts, nrm, idx, d2, cnt).view(np.int32), want.view(np.int32))
    if radius is None:
        assert (cnt == min(max_nn, len(pts))).all()


def test_pair_feature_equals_reference(ref):
    rng = np.random.default_rng(2)
    for _ in range(20000):
        p1, p2 = rng.normal(size=(2, 3)).astype(np.float32)
        n1, n2 = rng.normal(size=(2, 3)).astype(np.float32)
        if rng.random() < 0.2:
            n2 = n1.copy()
        if rng.random() < 0.1:
            p2 = p1.copy()
        want = np.zeros(4, np.float32)
        a = [np.ascontiguousarray(x) for x in (p1, n1, p2, n2)]
        ref.ref_pair_feature_f32(*(x.ctypes.data for x in a), want.ctypes.data)
        assert np.array_equal(of.pair_feature(p1, n1, p2, n2).view(np.int32), want.view(np.int32))


def test_lists_equal_knn_oracle():
    from oracle import knn as ok
    pts, _ = fc.scan(3000, 37)
    idx, d2, cnt = of.lists(pts, 30)
    kidx, kd2 = ok.knn(pts, pts, 30)
    assert np.array_equal(idx, kidx) and np.array_equal(d2.view(np.int32), kd2.view(np.int32))
    hidx, hd2, hcnt = of.lists(pts, 30, 0.03)
    thr = of.thr_of(0.03)
    for i in range(len(pts)):
        c = int((kd2[i] <= thr).sum())
        assert hcnt[i] == c and np.array_equal(hidx[i, :c], kidx[i, :c]) and (hidx[i, c:] == -1).all()


def test_feature_nn_and_mutual_filter():
    rng = np.random.default_rng(3)
    s = rng.integers(0, 4, (500, 33)).astype(np.float32)   # many exact ties
    t = rng.integers(0, 4, (400, 33)).astype(np.float32)
    d = ((s[:, None, :].astype(np.float64) - t[None]) ** 2).sum(-1)
    assert np.array_equal(of.feature_nn(s, t), d.argmin(1))   # integer data: exact sums; argmin takes the lowest
    corres, fell = of.correspondences_from_features(s, t, True, 0.0)
    ji = d.argmin(0)
    keep = ji[d.argmin(1)] == np.arange(500)
    assert not fell and np.array_equal(corres[:, 0], np.flatnonzero(keep))
    _, fell = of.correspondences_from_features(s, t, True, 1.0)
    assert fell

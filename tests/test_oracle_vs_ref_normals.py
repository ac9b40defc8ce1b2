"""The normal-estimation oracle (oracle/normals) against the reference's own code, compiled from its headers into
oracle/_ref/libo3dref_normals.so (oracle/ref_shim_normals): the covariance of each point, the fast 3x3 eigen solve,
both orientation rules of EstimateNormalsFromCovariances and the two OrientNormals* functions.  Every comparison is
bit for bit.  The oracle's normals are also checked against the analytic normals of planes and a sphere.  CPU only."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle
from oracle import normals as on
from tests import normals_cases as nc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libo3dref_normals.so")

_vp = C.c_void_p


@pytest.fixture(scope="module")
def ref():
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref/libo3dref_normals.so not built (needs the reference sources)")
    L = C.CDLL(REF)
    for name, args in (("ref_covariance_point_f32", [_vp, _vp, C.c_int32, _vp]),
                       ("ref_normal_from_covariance_f32", [_vp, _vp]),
                       ("ref_normals_from_covariances_f32", [_vp, C.c_int64, C.c_int, _vp]),
                       ("ref_orient_normals_to_align_with_direction_f32", [_vp, C.c_int64, _vp]),
                       ("ref_orient_normals_towards_camera_location_f32", [_vp, _vp, C.c_int64, _vp])):
        getattr(L, name).restype = None
        getattr(L, name).argtypes = args
    return L


def _ref_covariances(ref, pts, idx, cnt):
    out = np.zeros((len(pts), 9), np.float32)
    for i in range(len(pts)):
        ref.ref_covariance_point_f32(pts.ctypes.data, idx[i].ctypes.data, int(cnt[i]), out[i].ctypes.data)
    return out


def _ref_normals(ref, cov, prior=None):
    out = np.zeros((len(cov), 3), np.float32) if prior is None else prior.copy()
    ref.ref_normals_from_covariances_f32(cov.ctypes.data, len(cov), int(prior is not None), out.ctypes.data)
    return out


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _random_signs(normals, seed):
    rng = np.random.default_rng(seed)
    prior = normals * rng.choice([-1.0, 1.0], (len(normals), 1)).astype(np.float32)
    prior[::7] = 0.0   # some prior normals are zero: the dot is zero, nothing flips
    return np.ascontiguousarray(prior, np.float32)


@pytest.mark.parametrize("name", sorted(nc.cases()))
def test_covariances_and_normals_bit_exact(ref, name):
    pts, radius, max_nn = nc.cases()[name]
    normals, cov, cnt = on.estimate_normals(pts, radius, max_nn)
    idx, _, cnt2 = oracle.hybrid_search(pts, pts, radius, max_nn)
    assert np.array_equal(cnt, cnt2)
    want_cov = _ref_covariances(ref, pts, idx, cnt)
    assert np.array_equal(_bits(cov), _bits(want_cov))
    want = _ref_normals(ref, want_cov)
    assert np.array_equal(_bits(normals), _bits(want))
    # with prior normals of random sign (and some zero): the flip rule, and zero normals staying zero
    prior = _random_signs(want, 11)
    got, _, _ = on.estimate_normals(pts, radius, max_nn, prior_normals=prior)
    assert np.array_equal(_bits(got), _bits(_ref_normals(ref, want_cov, prior)))


@pytest.mark.parametrize("max_nn", [3, 8, 30, 32])
def test_max_nn_values(ref, max_nn):
    pts = nc.scan(6000, seed=9)
    normals, cov, cnt = on.estimate_normals(pts, 0.06, max_nn)
    idx, _, _ = oracle.hybrid_search(pts, pts, 0.06, max_nn)
    want_cov = _ref_covariances(ref, pts, idx, cnt)
    assert np.array_equal(_bits(cov), _bits(want_cov))
    assert np.array_equal(_bits(normals), _bits(_ref_normals(ref, want_cov)))
    assert cnt.max() == max_nn


def test_branches_are_exercised(ref):
    """The cases reach every fallback: identity covariances (< 3 neighbours), zero covariances, the diagonal branch
    with each of its three outcomes, and a rank-1 covariance."""
    cases = nc.cases()
    _, _, cnt = on.estimate_normals(*cases["sparse"])
    assert set(np.unique(cnt)) == {1, 2, 3}
    _, _, cnt = on.estimate_normals(*cases["sparse_knn32"])
    assert set(np.unique(cnt)) == {1, 2, 3, 4}
    n, cov, _ = on.estimate_normals(*cases["duplicates"])
    zero = ~cov.any(axis=1)
    assert zero.sum() > 50
    assert (n[zero] == [0, 0, 1]).all()                         # no prior: a zero normal becomes (0,0,1)
    prior = _random_signs(np.ones_like(n), 3)
    got, _, _ = on.estimate_normals(*cases["duplicates"], prior_normals=prior)
    assert not got[zero].any()                                  # with a prior it stays zero
    pts, an = nc.axis_planes()
    n, cov, _ = on.estimate_normals(pts, 0.5, 30)
    assert not cov[:, [1, 2, 5]].any()                          # exactly diagonal
    assert np.array_equal(n, an.astype(np.float32))             # (1,0,0), (0,1,0), (0,0,1)
    n, cov, _ = on.estimate_normals(*cases["line"])
    ev = np.linalg.eigvalsh(cov.reshape(-1, 3, 3).astype(np.float64))
    assert (ev[:, 1] < 1e-6 * ev[:, 2]).mean() > 0.9            # rank 1 up to rounding
    assert np.isfinite(n).all()


def test_covariance_point_with_0_to_3_neighbours(ref):
    pts = np.array([[0.1, 0.2, 0.3], [0.4, -0.1, 0.0], [0.2, 0.2, 0.9], [1.0, 0.5, 0.25]], np.float32)
    idx = np.array([2, 0, 3, 1], np.int32)
    for count in range(5):
        want = np.zeros(9, np.float32)
        ref.ref_covariance_point_f32(pts.ctypes.data, idx.ctypes.data, count, want.ctypes.data)
        got = on.covariance_point(pts, idx, count)
        assert np.array_equal(_bits(got), _bits(want)), count
        if count < 3:
            assert np.array_equal(got, np.eye(3, dtype=np.float32).ravel())


def test_fast_eigen_on_hand_made_covariances(ref):
    rng = np.random.default_rng(12)
    covs = [np.zeros(9), np.eye(3).ravel(), np.diag([1.0, 2.0, 3.0]).ravel(), np.diag([3.0, 1.0, 2.0]).ravel(),
            np.diag([2.0, 3.0, 1.0]).ravel(), np.diag([1.0, 1.0, 1.0]).ravel(), np.diag([0.0, 0.0, 5.0]).ravel()]
    for _ in range(3000):
        Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        lam = np.sort(rng.choice([0.0, 1e-9, 1e-4, 1.0, 2.0], 3) * rng.uniform(0.5, 2.0, 3))
        covs.append((Q @ np.diag(lam) @ Q.T).ravel())
    covs = np.ascontiguousarray(np.array(covs), np.float32)
    covs[:, 3], covs[:, 6], covs[:, 7] = covs[:, 1], covs[:, 2], covs[:, 5]   # symmetric, as the kernel stores it
    for c in covs:
        want = np.zeros(3, np.float32)
        ref.ref_normal_from_covariance_f32(c.ctypes.data, want.ctypes.data)
        assert np.array_equal(_bits(on.normal_from_covariance(c)), _bits(want)), c
    assert np.array_equal(_bits(on.normals_from_covariances(covs)), _bits(_ref_normals(ref, covs)))
    prior = _random_signs(rng.normal(size=(len(covs), 3)).astype(np.float32), 4)
    assert np.array_equal(_bits(on.normals_from_covariances(covs, prior)), _bits(_ref_normals(ref, covs, prior)))


def _orient_inputs(seed):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-1, 1, (3000, 3)).astype(np.float32)
    nrm = rng.normal(size=(3000, 3)).astype(np.float32)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    nrm[::9] = 0.0                                   # zero normals take the fallbacks
    pts[::18] = [0.25, -0.5, 0.75]                   # some of them sit on the camera: (0,0,1)
    return pts, np.ascontiguousarray(nrm, np.float32)


@pytest.mark.parametrize("direction", [(0.0, 0.0, 1.0), (0.3, -0.7, 0.2), (0.0, 0.0, 0.0)])
def test_orient_to_align_with_direction_bit_exact(ref, direction):
    _, nrm = _orient_inputs(1)
    d = np.array(direction, np.float32)
    want = nrm.copy()
    ref.ref_orient_normals_to_align_with_direction_f32(want.ctypes.data, len(want), d.ctypes.data)
    got = on.orient_normals_to_align_with_direction(nrm, d)
    assert np.array_equal(_bits(got), _bits(want))
    assert np.array_equal(got[::9], np.tile(d, (len(got[::9]), 1)))


@pytest.mark.parametrize("camera", [(0.25, -0.5, 0.75), (0.0, 0.0, 0.0), (10.0, 3.0, -2.0)])
def test_orient_towards_camera_location_bit_exact(ref, camera):
    pts, nrm = _orient_inputs(2)
    c = np.array(camera, np.float32)
    want = nrm.copy()
    ref.ref_orient_normals_towards_camera_location_f32(pts.ctypes.data, want.ctypes.data, len(want), c.ctypes.data)
    got = on.orient_normals_towards_camera_location(pts, nrm, c)
    assert np.array_equal(_bits(got), _bits(want))
    if camera == (0.25, -0.5, 0.75):
        assert (got[::18] == [0, 0, 1]).all()


def _angle_up_to_sign(a, b):
    a = a / np.linalg.norm(a, axis=1, keepdims=True)
    return np.arccos(np.clip(np.abs((a * b).sum(1)), 0.0, 1.0))


def test_oracle_normals_match_analytic_normals():
    """A sanity check of the checker itself: on planes and on the symmetric patch centres of a sphere the oracle's
    normals are the surface's normals up to sign, within 1e-4 rad."""
    pts, an = nc.axis_planes()
    n, _, _ = on.estimate_normals(pts, 0.5, 30)
    assert _angle_up_to_sign(n.astype(np.float64), an).max() < 1e-4
    pts, an = nc.tilted_plane()
    n, _, cnt = on.estimate_normals(pts, 0.05, 32)
    ok = cnt >= 3
    assert ok.mean() > 0.99 and _angle_up_to_sign(n[ok].astype(np.float64), an[ok]).max() < 1e-4
    pts, an, centres = nc.sphere()
    n, _, cnt = on.estimate_normals(pts, 0.06, 30)
    assert (cnt[centres] == 25).all()
    assert _angle_up_to_sign(n[centres].astype(np.float64), an[centres]).max() < 1e-4

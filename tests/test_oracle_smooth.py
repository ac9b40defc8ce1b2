"""The smoothing oracle (oracle/smooth) against the reference's own SmoothLaplacianCPU, SmoothTaubinCPU, SmoothMLSCPU
and SmoothBilateralCPU, compiled whole from its headers into oracle/_ref/libo3dref_smooth.so (oracle/ref_shim_smooth),
whose neighbour searches are the oracle's brute force.  In libm mode every comparison is bit for bit.  The oracle also
reproduces the reference's known answers (tests/golden/smooth_kats.json).  CPU only."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import oracle
from oracle import knn as ok
from oracle import normals as on
from oracle import smooth as osm
from tests import knn_cases as kc
from tests import normals_cases as nc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libo3dref_smooth.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "smooth_kats.json")
ROWS = 2000   # points of each fixture: the reference's search is the O(n^2) brute force

_vp, _i64, _dbl, _i = C.c_void_p, C.c_int64, C.c_double, C.c_int


@pytest.fixture(scope="module")
def ref():
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref/libo3dref_smooth.so not built (needs the reference sources)")
    L = C.CDLL(REF)
    for name, args in (("ref_smooth_set_search", [_vp, _vp]),
                       ("ref_smooth_laplacian_f32", [_vp, _i64, _i64, _dbl, _i, _i, _vp]),
                       ("ref_smooth_taubin_f32", [_vp, _i64, _i64, _dbl, _dbl, _i, _i, _vp]),
                       ("ref_smooth_mls_f32", [_vp, _i64, _dbl, _i, _vp, _vp]),
                       ("ref_smooth_bilateral_f32", [_vp, _vp, _i64, _dbl, _i, _dbl, _dbl, _vp])):
        getattr(L, name).restype = None if name == "ref_smooth_set_search" else C.c_int
        getattr(L, name).argtypes = args
    L.ref_smooth_set_search(C.cast(ok.lib().orc_knn_f32, _vp), C.cast(oracle.lib().orc_hybrid_search_bruteforce_f32, _vp))
    return L


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _knn_fixtures():
    return {name: np.ascontiguousarray(data[:ROWS]) for name, (data, _) in kc.cases().items()}


def _normals_fixtures():
    return {name: (np.ascontiguousarray(p[:ROWS]), r, m) for name, (p, r, m) in nc.cases().items()}


@pytest.mark.parametrize("name", list(kc.cases()))
def test_laplacian_and_taubin_match_reference(ref, name):
    p = _knn_fixtures()[name]
    n = len(p)
    for max_nn in (1, 7, 20, 31):
        for fixed in (0, 1):
            out = np.empty_like(p)
            assert ref.ref_smooth_laplacian_f32(p.ctypes.data, n, 3, 0.5, max_nn, fixed, out.ctypes.data) == 0
            want = osm.smooth_laplacian(p, 3, (0.5,), max_nn, fixed)
            np.testing.assert_array_equal(_bits(want), _bits(out), err_msg=f"laplacian {name} {max_nn} {fixed}")
            assert ref.ref_smooth_taubin_f32(p.ctypes.data, n, 3, 0.5, -0.53, max_nn, fixed, out.ctypes.data) == 0
            want = osm.smooth_laplacian(p, 3, (0.5, -0.53), max_nn, fixed)
            np.testing.assert_array_equal(_bits(want), _bits(out), err_msg=f"taubin {name} {max_nn} {fixed}")


@pytest.mark.parametrize("name", list(nc.cases()))
def test_mls_and_bilateral_match_reference(ref, name):
    p, radius, _ = _normals_fixtures()[name]
    n = len(p)
    prior = on.estimate_normals(p, radius, 30)[0]
    for max_nn in (1, 7, 20, 32):
        for r in (radius, 0.0):   # the hybrid branch and the KNN branch
            nrm = prior.copy()
            out = np.empty_like(p)
            assert ref.ref_smooth_mls_f32(p.ctypes.data, n, r, max_nn, nrm.ctypes.data, out.ctypes.data) == 0
            want, wn = osm.smooth_mls(p, r, max_nn, prior, device_math=False)
            np.testing.assert_array_equal(_bits(want), _bits(out), err_msg=f"mls {name} {r} {max_nn}")
            np.testing.assert_array_equal(_bits(wn), _bits(nrm), err_msg=f"mls normals {name} {r} {max_nn}")
        out = np.empty_like(p)
        assert ref.ref_smooth_mls_f32(p.ctypes.data, n, radius, max_nn, None, out.ctypes.data) == 0
        np.testing.assert_array_equal(_bits(osm.smooth_mls(p, radius, max_nn, device_math=False)[0]), _bits(out))
        for sigma_s, sigma_r in ((radius, radius), (0.5 * radius, 2 * radius)):
            assert ref.ref_smooth_bilateral_f32(p.ctypes.data, prior.ctypes.data, n, radius, max_nn, sigma_s, sigma_r,
                                                out.ctypes.data) == 0
            want = osm.smooth_bilateral(p, prior, radius, max_nn, sigma_s, sigma_r, device_math=False)
            np.testing.assert_array_equal(_bits(want), _bits(out), err_msg=f"bilateral {name} {max_nn} {sigma_s}")


def test_reference_boundaries(ref):
    p = np.array([[0, 0, 0], [1, 0, 0]], np.float32)
    out = np.empty_like(p)
    for it, max_nn in ((0, 20), (3, 0), (3, -1)):
        assert ref.ref_smooth_laplacian_f32(p.ctypes.data, 2, it, 0.5, max_nn, 0, out.ctypes.data) == 0
        np.testing.assert_array_equal(out, p)
    assert ref.ref_smooth_mls_f32(p.ctypes.data, 2, 0.0, 0, None, out.ctypes.data) == 0
    np.testing.assert_array_equal(out, p)
    # radius-only MLS needs the fixed-radius search, which the shim (like the product) does not have
    assert ref.ref_smooth_mls_f32(p.ctypes.data, 2, 1.0, 0, None, out.ctypes.data) == -1


@pytest.mark.parametrize("device_math", [False, True])
def test_kats(device_math):
    kats = json.load(open(GOLDEN))
    for case in kats["cases"]:
        p = np.asarray(case["points"], np.float32)
        a = case["args"]
        if case["call"] in ("smooth_laplacian", "smooth_taubin"):
            factors = (a.get("lambda_", 0.5),) if case["call"] == "smooth_laplacian" else (a.get("lambda_", 0.5),
                                                                                           a.get("mu", -0.53))
            got = osm.smooth_laplacian(p, a["iterations"], factors, a.get("max_nn", 20),
                                       a.get("use_fixed_neighborhoods", False))
        elif case["call"] == "smooth_mls":
            got = osm.smooth_mls(p, a["radius"], a["max_nn"], device_math=device_math)[0]
        else:
            got = osm.smooth_bilateral(p, np.asarray(case["normals"], np.float32), a["radius"], a["max_nn"],
                                       a["sigma_s"], a["sigma_r"], device_math=device_math)
        np.testing.assert_allclose(got, case["want"], rtol=0, atol=case["atol"], err_msg=case["name"])


def test_device_math_differs_from_libm_only_in_the_last_bits():
    """The two modes differ only through exp / acos / cos: the fraction of bit-identical rows is high and the rest are
    within a few ulp of the coordinates."""
    p, radius, max_nn = nc.cases()["scan"]
    prior = on.estimate_normals(p, radius, max_nn)[0]
    lists = oracle.hybrid_search(p, p, radius, max_nn, bruteforce=True)
    a = osm.smooth_bilateral(p, prior, radius, max_nn, radius, radius, device_math=False, lists=lists)
    b = osm.smooth_bilateral(p, prior, radius, max_nn, radius, radius, device_math=True, lists=lists)
    same = np.all(_bits(a) == _bits(b), axis=1).mean()
    print(f"\nbilateral, scan: {same:.6f} of the rows bit-identical between libm and device math")
    assert same > 0.9
    np.testing.assert_allclose(a, b, rtol=4e-7, atol=0)

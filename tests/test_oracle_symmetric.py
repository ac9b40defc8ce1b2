"""The symmetric-ICP CPU oracle (oracle/symmetric) against the reference's compiled ComputePoseSymmetricCPU
(oracle/_ref/libo3dref_symmetric.so, built from oracle/ref_shim_symmetric), its inline known answers
(cpp/tests/t/pipelines/registration/TransformationEstimation.cpp, parsed into tests/golden/symmetric_kats.json by
tests/golden/make_symmetric_kats.py) and scipy's rotations.  Runs without a GPU."""
import ctypes as C
import json
import os

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle import symmetric as sym

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libo3dref_symmetric.so")
KERNELS = [(0, 1.0, 1.0), (1, 1.0, 1.0), (2, 0.05, 1.0), (3, 0.05, 1.0), (4, 0.05, 1.0), (5, 0.1, 1.0),
           (6, 0.05, 0.5)]


def load_symmetric_kats():
    with open(os.path.join(ROOT, "tests", "golden", "symmetric_kats.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def skats():
    return load_symmetric_kats()


def unit(a):
    a = np.asarray(a, np.float32)
    return (a / np.linalg.norm(a, axis=1, keepdims=True).astype(np.float32)).astype(np.float32)


def random_pair(n, m, seed, holes=0.2):
    rng = np.random.default_rng(seed)
    src = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    tgt = rng.uniform(-1, 1, (m, 3)).astype(np.float32)
    corr = rng.integers(0, m, n).astype(np.int64)
    corr[rng.random(n) < holes] = -1
    return src, tgt, unit(rng.normal(size=(n, 3))), unit(rng.normal(size=(m, 3))), corr


def transform_f32(T, p, normals=False):
    T32 = np.asarray(T, np.float32)
    out = p.astype(np.float32) @ T32[:3, :3].T
    return out if normals else (out + T32[:3, 3]).astype(np.float32)


def expected_motion(kat):
    axis = np.array(kat["axis"], np.float64)
    T = np.eye(4)
    T[:3, :3] = Rotation.from_rotvec(kat["angle"] * axis / np.linalg.norm(axis)).as_matrix()
    T[:3, 3] = kat["translation"]
    return T


@pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref not built (needs the reference source tree)")
@pytest.mark.parametrize("kernel", KERNELS)
def test_sums_equal_the_reference_kernel_bit_for_bit(kernel):
    L = C.CDLL(REF)
    L.ref_pose_symmetric_sums_f32.argtypes = [C.c_void_p] * 5 + [C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                                                                  C.c_int, C.c_double, C.c_double, C.c_void_p]
    src, tgt, sn, tn, corr = random_pair(3000, 2000, seed=kernel[0])
    ms, mt, count = sym.means(src, tgt, corr)
    assert count > 0
    want = np.zeros(29)
    L.ref_pose_symmetric_sums_f32(src.ctypes.data, tgt.ctypes.data, sn.ctypes.data, tn.ctypes.data, corr.ctypes.data,
                                  len(src), len(tgt), ms.ctypes.data, mt.ctypes.data, *kernel, want.ctypes.data)
    got = sym.sums(src, tgt, sn, tn, corr, ms, mt, kernel)
    assert got.tobytes() == want.tobytes()


def test_rmse_kats(skats):
    k = skats["rmse"]
    s, ns = np.array([k["source_point"]], np.float32), np.array([k["source_normal"]], np.float32)
    t, nt = np.array([k["target_point"]], np.float32), np.array([k["target_normal"]], np.float32)
    c = np.array([0])
    got = [sym.rmse(s, t, ns, nt, c), sym.rmse(s, t, ns, -nt, c)]
    t = np.zeros((1, 3), np.float32)
    got += [sym.rmse(s, t, ns, ns, c), sym.rmse(s, t, ns, -ns, c)]
    np.testing.assert_allclose(got, k["expected"], atol=k["tol_f32"])
    assert sym.rmse(s, t, ns, ns, np.array([-1])) == 0.0


def _kat_clouds(k):
    src = np.array(k["source_points"], np.float32)
    sn = unit(k["source_normals"])
    T = expected_motion(k)
    return src, sn, transform_f32(T, src), transform_f32(T, sn, normals=True), T


def test_transformation_kats(skats):
    k = skats["transformation"]
    src, sn, tgt, tn, T = _kat_clouds(k)
    corr = np.arange(len(src))
    np.testing.assert_allclose(sym.compute_transformation(src, tgt, sn, tn, corr), T, atol=k["tol_f32"])
    tn_alt = (tn * np.array(k["alternating_signs"], np.float32)[:, None]).astype(np.float32)
    np.testing.assert_allclose(sym.compute_transformation(src, tgt, sn, tn_alt, corr), T, atol=k["tol_f32"])
    assert np.array_equal(sym.compute_transformation(src, tgt, sn, tn, np.full(len(src), -1)), np.eye(4))
    for bad in (-2, len(tgt)):
        c = corr.copy()
        c[0] = bad
        with pytest.raises(RuntimeError):
            sym.compute_transformation(src, tgt, sn, tn, c)
        with pytest.raises(RuntimeError):
            sym.rmse(src, tgt, sn, tn, c)


def test_cauchy_kat(skats):
    k = skats["transformation"]
    src = np.array(k["robust_source_points"], np.float32)
    sn = unit(k["robust_source_normals"])
    T = expected_motion(k)
    tgt = (transform_f32(T, src) + np.array(k["robust_noise"], np.float32)).astype(np.float32)
    tn = transform_f32(T, sn, normals=True)
    rk = k["robust_kernel"]
    kernel = (sym.ROBUST[rk["method"]], rk["scaling_parameter"], rk["shape_parameter"])
    got = sym.compute_transformation(src, tgt, sn, tn, np.arange(len(src)), kernel)
    np.testing.assert_allclose(got, np.array(k["robust_expected"]), atol=k["tol_f32"])


@pytest.mark.parametrize("seed", range(4))
def test_pose_conversion_matches_scipy(seed):
    rng = np.random.default_rng(seed)
    pose = rng.normal(scale=0.3, size=6)
    ms, mt = rng.normal(size=3), rng.normal(size=3)
    g = pose[:3]
    theta = np.arctan(np.linalg.norm(g))
    H = Rotation.from_rotvec(theta * g / np.linalg.norm(g)).as_matrix()
    R = H @ H
    want = np.eye(4)
    want[:3, :3] = R
    want[:3, 3] = mt + H @ (pose[3:] * np.cos(theta)) - R @ ms
    np.testing.assert_allclose(sym.pose_to_transformation(pose, ms, mt), want, atol=1e-14)
    assert np.array_equal(sym.pose_to_transformation(np.zeros(6), ms, mt)[:3, :3], np.eye(3))

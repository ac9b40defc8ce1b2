"""The CPU oracle of Doppler ICP (oracle/doppler) against the reference's own CPU kernel
(oracle/_ref/libo3dref_doppler.so, built from oracle/ref_shim_doppler): the 29 sums bit for bit in f32 for every robust
pair the dual dispatch accepts, with and without outlier rejection, under a non-identity calibration, on both sides of
every switch iteration.  Also the estimator's constructor rules and the velocity precompute against an f64 derivation.
Needs no GPU."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from oracle import doppler as dop
from tests.doppler_cases import CALIB, make_doppler_pair

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libo3dref_doppler.so")
KERNELS = [(0, 1.0, 1.0), (5, 0.4, 1.0)]   # L2 and Tukey: what DISPATCH_DUAL_ROBUST_KERNEL_FUNCTION accepts


def _ref():
    L = C.CDLL(REF)
    vp, d, i, i64 = C.c_void_p, C.c_double, C.c_int, C.c_int64
    L.ref_pose_doppler_sums_f32.restype = i
    L.ref_pose_doppler_sums_f32.argtypes = [vp] * 6 + [i64, i64] + [vp] * 4 + [d, i, d, i, d, d, i, d, d, d, vp]
    L.ref_precompute_doppler_f32.restype = None
    L.ref_precompute_doppler_f32.argtypes = [vp] * 5
    return L


def _motion():
    T = np.eye(4)
    a, b, g = 0.03, -0.02, 0.05
    Rx = np.array([[1, 0, 0], [0, math.cos(a), -math.sin(a)], [0, math.sin(a), math.cos(a)]])
    Ry = np.array([[math.cos(b), 0, math.sin(b)], [0, 1, 0], [-math.sin(b), 0, math.cos(b)]])
    Rz = np.array([[math.cos(g), -math.sin(g), 0], [math.sin(g), math.cos(g), 0], [0, 0, 1]])
    T[:3, :3] = Rz @ Ry @ Rx
    T[:3, 3] = [0.21, -0.07, 0.04]
    return T


@pytest.fixture(scope="module")
def case():
    src, d, dirs, tgt, nrm, _, _ = make_doppler_pair(6000, seed=3, dynamic=0.1)
    rng = np.random.default_rng(9)
    corr = rng.integers(0, len(tgt), len(src)).astype(np.int64)
    corr[rng.random(len(src)) < 0.1] = -1
    return src, d, dirs, tgt, nrm, corr


def _ref_sums(L, case, p, T, it):
    """The reference kernel with the switches of kernel/Registration.cpp:222-235 applied for iteration `it`."""
    src, d, dirs, tgt, nrm, corr = case
    w, v = dop.state(T, p.period)
    R = np.array(p.R[:], np.float32)
    r = np.array(p.r[:], np.float32)
    mg = p.method_g if it >= p.min_geo else 0
    md = p.method_d if it >= p.min_dop else 0
    reject = int(bool(p.reject) and it >= p.min_reject)
    out = np.zeros(29, np.float64)
    arrs = [np.ascontiguousarray(a) for a in (src, d, dirs, tgt, nrm, corr)]
    rc = L.ref_pose_doppler_sums_f32(*[a.ctypes.data for a in arrs], len(src), len(tgt), R.ctypes.data, r.ctypes.data,
                                     w.ctypes.data, v.ctypes.data, p.period, reject, p.threshold, mg, p.scale_g,
                                     p.shape_g, md, p.scale_d, p.shape_d, p.lambda_doppler, out.ctypes.data)
    assert rc == 0
    return out


@pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref not built (needs the reference source tree)")
@pytest.mark.parametrize("kg", KERNELS)
@pytest.mark.parametrize("kd", KERNELS)
@pytest.mark.parametrize("reject", [False, True])
@pytest.mark.parametrize("calib", ["identity", "mounted"])
def test_sums_equal_the_reference_kernel_bit_for_bit(case, kg, kd, reject, calib):
    L = _ref()
    p = dop.params(period=0.1, lambda_doppler=0.3, reject_dynamic_outliers=reject, doppler_outlier_threshold=2.0,
                   outlier_rejection_min_iteration=2, geometric_robust_loss_min_iteration=1,
                   doppler_robust_loss_min_iteration=3, geometric_kernel=kg, doppler_kernel=kd,
                   transform_vehicle_to_sensor=None if calib == "identity" else CALIB)
    T = _motion()
    for it in range(5):   # 0..4: both sides of 1 (geometric), 2 (rejection) and 3 (Doppler)
        got = dop.sums(*case, p, T, it)
        want = _ref_sums(L, case, p, T, it)
        assert got.tobytes() == want.tobytes(), (it, np.flatnonzero(got != want))


@pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref not built (needs the reference source tree)")
def test_rejection_changes_the_sums_and_the_other_kernels_are_refused(case):
    L = _ref()
    T = _motion()
    on = dop.params(reject_dynamic_outliers=True, transform_vehicle_to_sensor=CALIB)
    off = dop.params(reject_dynamic_outliers=False, transform_vehicle_to_sensor=CALIB)
    a, b = dop.sums(*case, on, T, 2), dop.sums(*case, off, T, 2)
    assert a[28] == b[28] and a[27] < b[27]   # rejected points still count, with zero residual
    huber = dop.params(doppler_kernel=(2, 0.5, 1.0), doppler_robust_loss_min_iteration=0)
    src, d, dirs, tgt, nrm, corr = case
    arrs = [np.ascontiguousarray(x) for x in (src, d, dirs, tgt, nrm, corr)]
    w, v = dop.state(T, 0.1)
    R, r = np.array(huber.R[:], np.float32), np.array(huber.r[:], np.float32)
    out = np.zeros(29)
    assert L.ref_pose_doppler_sums_f32(*[x.ctypes.data for x in arrs], len(src), len(tgt), R.ctypes.data,
                                       r.ctypes.data, w.ctypes.data, v.ctypes.data, 0.1, 0, 2.0, 0, 1.0, 1.0, 2, 0.5,
                                       1.0, 0.01, out.ctypes.data) == 1


@pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref not built (needs the reference source tree)")
def test_precompute_equals_the_reference_bit_for_bit():
    L = _ref()
    p = dop.params(period=0.05, transform_vehicle_to_sensor=CALIB)
    rng = np.random.default_rng(4)
    R, r = np.array(p.R[:], np.float32), np.array(p.r[:], np.float32)
    for _ in range(200):
        w, v = rng.normal(0, 3, 3).astype(np.float32), rng.normal(0, 20, 3).astype(np.float32)
        a, b = np.zeros(3, np.float32), np.zeros(3, np.float32)
        dop.lib().orc_dop_precompute(R.ctypes.data, r.ctypes.data, w.ctypes.data, v.ctypes.data, a.ctypes.data)
        L.ref_precompute_doppler_f32(R.ctypes.data, r.ctypes.data, w.ctypes.data, v.ctypes.data, b.ctypes.data)
        assert a.tobytes() == b.tobytes()


def test_velocity_against_an_f64_derivation():
    """v_s_in_S = R_S_to_V (v + w x r) with w, v = -pose / period, in f64 from the same T: equal within f32 rounding."""
    rng = np.random.default_rng(1)
    p = dop.params(period=0.1, transform_vehicle_to_sensor=CALIB)
    Rinv = np.linalg.inv(CALIB[:3, :3])
    for k in range(50):
        T = _motion()
        T[:3, 3] = rng.normal(0, 1, 3)
        got = dop.velocity(p, T)
        pose = dop.transformation_to_pose(T)
        # TransformationToPose is the ZYX Euler decomposition of the rotation block
        assert abs(pose[0] - math.atan2(T[2, 1], T[2, 2])) < 1e-15 and np.array_equal(pose[3:], T[:3, 3])
        w, v = -pose[:3] / 0.1, -pose[3:] / 0.1
        want = Rinv @ (v + np.cross(w, CALIB[:3, 3]))
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-5 * max(1.0, np.abs(want).max()))


def test_constructor_rules():
    import open3d_b200 as o3d
    reg = o3d.t.pipelines.registration
    e = reg.TransformationEstimationForDopplerICP()
    assert (e.period, e.lambda_doppler, e.reject_dynamic_outliers, e.doppler_outlier_threshold,
            e.outlier_rejection_min_iteration, e.geometric_robust_loss_min_iteration,
            e.doppler_robust_loss_min_iteration) == (0.1, 0.01, False, 2.0, 2, 0, 2)
    assert e.geometric_kernel.type == reg.RobustKernelMethod.L2Loss and e.doppler_kernel.type == reg.RobustKernelMethod.L2Loss
    assert np.array_equal(e.transform_vehicle_to_sensor, np.eye(4))
    assert repr(e) == "TransformationEstimationForDopplerICP with lambda_doppler: 0.010000"
    for bad in (1.5, -0.1):
        assert reg.TransformationEstimationForDopplerICP(lambda_doppler=bad).lambda_doppler == 0.01
    assert reg.TransformationEstimationForDopplerICP(lambda_doppler=1.0).lambda_doppler == 1.0
    for small in (0.0, 9.99e-4, -5e-4):
        with pytest.raises(RuntimeError, match="Time period too small."):
            reg.TransformationEstimationForDopplerICP(period=small)
    assert reg.TransformationEstimationForDopplerICP(period=-0.1).period == -0.1
    with pytest.raises(RuntimeError, match="expected to have \\[4, 4\\]"):
        reg.TransformationEstimationForDopplerICP(transform_vehicle_to_sensor=np.eye(3))
    e.period, e.reject_dynamic_outliers = 0.2, True   # every field is writable
    assert e._params().period == 0.2 and e._params().reject_dynamic_outliers == 1

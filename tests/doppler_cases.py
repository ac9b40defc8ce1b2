"""Seeded synthetic FMCW scans for Doppler ICP (there is no Doppler dataset offline; upstream's test reads
DemoDopplerICPSequence).

A scene from tests/synth.py is seen by a sensor mounted on the vehicle with a known calibration
(transform_vehicle_to_sensor).  Each source point's direction is its unit ray from the sensor, in the vehicle frame, as
upstream's ComputeDirectionVectors gives it; its Doppler value is the radial velocity the reference's model predicts
for the true source->target motion over `period`, -(R_S_to_V d) . v_s_in_S, plus Gaussian noise.  A seeded subset of
dynamic points gets Doppler values 4-8 m/s off."""
import numpy as np

from oracle import doppler as dop
from tests.synth import axis_angle, make_icp_pair

CALIB = np.eye(4)
CALIB[:3, :3] = axis_angle([0.2, 0.1, 1.0], 12.0)
CALIB[:3, 3] = [0.6, -0.2, 1.3]


def _directions(points, calib):
    d = points.astype(np.float64) - calib[:3, 3]
    return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def _dopplers(dirs, T_gt, calib, period, noise, dynamic, rng):
    """The reference's predicted Doppler at the true motion, in f32 through the oracle, plus noise and dynamic points."""
    p = dop.params(period=period, transform_vehicle_to_sensor=calib)
    v = dop.velocity(p, T_gt)
    R = np.array(p.R[:], np.float32).reshape(3, 3)
    pred = -((dirs @ R.T).astype(np.float32) @ v).astype(np.float32)
    d = pred + rng.normal(0, noise, len(dirs)).astype(np.float32)
    moving = rng.random(len(dirs)) < dynamic
    d[moving] += (rng.choice([-1.0, 1.0], moving.sum()) * rng.uniform(4, 8, moving.sum())).astype(np.float32)
    return d.astype(np.float32), moving


def make_doppler_pair(n_points, seed=1, calib=CALIB, period=0.1, noise=0.02, dynamic=0.0):
    """make_icp_pair's clouds plus directions and Doppler values for its true motion.  Returns (source, dopplers [N],
    directions [N,3], target, target_normals, T_gt, moving mask)."""
    src, tgt, nrm, T_gt = make_icp_pair(n_points, seed=seed)
    rng = np.random.default_rng(seed + 77)
    dirs = _directions(src, calib)
    d, moving = _dopplers(dirs, T_gt, calib, period, noise, dynamic, rng)
    return src, d, dirs, tgt, nrm, T_gt, moving


def make_corridor(n_points, seed=1, shift=(0.3, 0.02, -0.01), calib=CALIB, period=0.1, noise=0.02, dynamic=0.0):
    """A straight corridor along x (floor z = 0, walls y = +-2, 30 m long): its geometry leaves translation along x
    free.  The source is an independent sampling moved by -shift, so T_gt translates by +shift."""
    rng = np.random.default_rng(seed)

    def sample(k, r):
        which = r.integers(0, 3, k)
        x = r.uniform(0, 30, k)
        u = r.uniform(-2, 2, k)
        h = r.uniform(0, 2.5, k)
        p = np.stack([x, u, np.zeros(k)], 1)
        nrm = np.tile([0.0, 0.0, 1.0], (k, 1))
        for side, s in ((1, 2.0), (2, -2.0)):
            m = which == side
            p[m] = np.stack([x[m], np.full(m.sum(), s), h[m]], 1)
            nrm[m] = [0.0, -np.sign(s), 0.0]
        return p, nrm

    tgt, nrm = sample(n_points, rng)
    base, _ = sample(n_points, np.random.default_rng(seed + 1000))
    T_gt = np.eye(4)
    T_gt[:3, 3] = shift
    src = (base - np.asarray(shift)).astype(np.float32)
    dirs = _directions(src, calib)
    d, moving = _dopplers(dirs, T_gt, calib, period, noise, dynamic, np.random.default_rng(seed + 77))
    return src, d, dirs, tgt.astype(np.float32), nrm.astype(np.float32), T_gt, moving

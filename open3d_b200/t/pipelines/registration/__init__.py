"""Mirror of ``open3d.t.pipelines.registration`` for the point-to-point, point-to-plane, symmetric, coloured and Doppler
ICP paths (cpp/pybind/t/pipelines/registration/registration.cpp:96-140, 469-530;
cpp/open3d/t/pipelines/registration/{Registration,TransformationEstimation}.cpp).

The iteration loop itself runs device-resident inside libo3db200.so
(``o3db_icp_*``); this module only validates arguments the way
``AssertInputMultiScaleICP`` does (Registration.cpp:119-219) and marshals
results into the reference's result type.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field
from enum import IntEnum

import numpy as np
import torch

from ... import geometry as _geometry
from ...._lib import (ERR_SINGULAR, DopplerParams, IcpOptions, IcpResult, O3DBError, RobustKernel as _CRobust, check, dptr,
                      lib)
from ....core import as_device_f32_points, as_host_f64_4x4, current_stream_ptr

PointCloud = _geometry.PointCloud


class RobustKernelMethod(IntEnum):
    """t/pipelines/registration/RobustKernel.h:15-23"""
    L2Loss = 0
    L1Loss = 1
    HuberLoss = 2
    CauchyLoss = 3
    GMLoss = 4
    TukeyLoss = 5
    GeneralizedLoss = 6


@dataclass
class RobustKernel:
    """robust_kernel.RobustKernel(type, scaling_parameter, shape_parameter) (RobustKernel.h:33-58)"""
    type: RobustKernelMethod = RobustKernelMethod.L2Loss
    scaling_parameter: float = 1.0
    shape_parameter: float = 1.0

    def _c(self):
        return _CRobust(int(self.type), float(self.scaling_parameter), float(self.shape_parameter))


class robust_kernel:  # namespace shim: open3d.t.pipelines.registration.robust_kernel.*
    RobustKernel = RobustKernel
    RobustKernelMethod = RobustKernelMethod


@dataclass
class ICPConvergenceCriteria:
    """Registration.h:43-48"""
    relative_fitness: float = 1e-6
    relative_rmse: float = 1e-6
    max_iteration: int = 30


@dataclass
class RegistrationResult:
    """Registration.h:65-98.  transformation: 4x4 Float64 on CPU (numpy);
    correspondence_set: [N] int64 on the compute device, -1 = no correspondence."""
    transformation: np.ndarray = field(default_factory=lambda: np.eye(4))
    correspondence_set: torch.Tensor | None = None
    inlier_rmse: float = 0.0
    fitness: float = 0.0
    converged: bool = False
    num_iterations: int = 0

    def __repr__(self):
        n = 0 if self.correspondence_set is None else int(self.correspondence_set.shape[0])
        return (f"RegistrationResult[converged={self.converged}, num_iteration={self.num_iterations:d}, "
                f"fitness_={self.fitness:e}, inlier_rmse={self.inlier_rmse:e}, correspondences={n:d}].")


class TransformationEstimation:
    """TransformationEstimation.h:53-95 (abstract)."""

    def compute_rmse(self, source, target, correspondences):
        raise NotImplementedError

    def compute_transformation(self, source, target, correspondences, current_transform=None, iteration=0):
        raise NotImplementedError


def _corr_arg(corr, n):
    if isinstance(corr, np.ndarray):
        corr = torch.from_numpy(corr)
    if corr.dtype != torch.int64:
        raise RuntimeError("correspondences must be Int64")          # AssertValidCorrespondences
    corr = corr.reshape(-1)
    if corr.shape[0] != n:
        raise RuntimeError("Correspondences must be of same length as source point-cloud positions.")
    return corr.cuda().contiguous()


class TransformationEstimationPointToPoint(TransformationEstimation):
    """TransformationEstimation.h:101-150 / TransformationEstimation.cpp:101-159: the estimator ``icp`` and
    ``multi_scale_icp`` use when none is given.  Positions only; no robust kernel."""

    kernel = RobustKernel()   # (the C options struct carries one; this estimator ignores it)

    @staticmethod
    def _check(source, target):
        if not target.has_point_positions() or not source.has_point_positions():
            raise RuntimeError("Source and/or Target pointcloud is empty.")

    def compute_rmse(self, source, target, correspondences):
        """TransformationEstimation.cpp:101-130 (tensor ops upstream; torch ops on the device here)."""
        self._check(source, target)
        s, t = source.point["positions"], target.point["positions"]
        corr = _corr_arg(correspondences, s.shape[0])
        valid = corr != -1
        idx = corr[valid]
        e = (s[valid] - t[idx]) ** 2
        return float(torch.sqrt(e.sum().to(torch.float64) / idx.shape[0]))

    def compute_rt(self, source, target, correspondences):
        """kernel::ComputeRtPointToPoint (kernel/Registration.cpp:365-404) through o3db_compute_rt_point_to_point:
        R [3,3] and t [3], Float64 on the host, and the number of valid correspondences."""
        self._check(source, target)
        s, t = source.point["positions"], target.point["positions"]
        corr = _corr_arg(correspondences, s.shape[0])
        R, tr, count = np.zeros((3, 3), np.float64), np.zeros(3, np.float64), C.c_int(0)
        check(lib.o3db_compute_rt_point_to_point(s.data_ptr(), t.data_ptr(), corr.data_ptr(), s.shape[0], dptr(R),
                                                 dptr(tr), C.byref(count), current_stream_ptr()))
        return R, tr, int(count.value)

    def compute_transformation(self, source, target, correspondences, current_transform=None, iteration=0):
        """TransformationEstimation.cpp:132-159 -> 4x4 Float64 on CPU (RtToTransformation)."""
        R, tr, _ = self.compute_rt(source, target, correspondences)
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, tr
        return T


class TransformationEstimationPointToPlane(TransformationEstimation):
    """TransformationEstimation.h:155-212 / TransformationEstimation.cpp:161-227."""

    def __init__(self, kernel: RobustKernel | None = None):
        self.kernel = kernel if kernel is not None else RobustKernel()

    def _check(self, source, target):
        if not target.has_point_positions() or not source.has_point_positions():
            raise RuntimeError("Source and/or Target pointcloud is empty.")
        if not target.has_point_normals():
            raise RuntimeError("Target pointcloud missing normals attribute.")

    def compute_rmse(self, source, target, correspondences):
        """TransformationEstimation.cpp:161-194 (host-side glue around tensor ops upstream;
        evaluated here with torch ops on the device — not part of the timed hot path)."""
        self._check(source, target)
        s, t, n = source.point["positions"], target.point["positions"], target.point["normals"]
        corr = _corr_arg(correspondences, s.shape[0])
        valid = corr != -1
        idx = corr[valid]
        e = ((s[valid] - t[idx]) * n[idx]) ** 2
        return float(torch.sqrt(e.sum(dtype=torch.float64) / idx.shape[0]))

    def compute_pose(self, source, target, correspondences):
        """kernel::ComputePosePointToPlane (kernel/Registration.cpp:35-78): pose [6] f64,
        residual, inlier_count — through the C ABI seam o3db_compute_pose_point_to_plane."""
        self._check(source, target)
        s, t, n = source.point["positions"], target.point["positions"], target.point["normals"]
        corr = _corr_arg(correspondences, s.shape[0])
        pose = torch.zeros(6, dtype=torch.float64, device=s.device)
        sums = torch.zeros(29, dtype=torch.float64, device=s.device)
        residual, count = C.c_float(0), C.c_int(0)
        k = self.kernel._c()
        check(lib.o3db_compute_pose_point_to_plane(s.data_ptr(), t.data_ptr(), n.data_ptr(), corr.data_ptr(),
                                                   s.shape[0], C.byref(k), sums.data_ptr(), pose.data_ptr(),
                                                   C.byref(residual), C.byref(count), current_stream_ptr()))
        return pose, float(residual.value), int(count.value), sums

    def compute_transformation(self, source, target, correspondences, current_transform=None, iteration=0):
        """TransformationEstimation.cpp:196-227 -> 4x4 Float64 on CPU."""
        pose, _, _, _ = self.compute_pose(source, target, correspondences)
        p = np.ascontiguousarray(pose.cpu().numpy())
        T = np.zeros((4, 4), np.float64)
        lib.o3db_pose_to_transformation(dptr(p), dptr(T))
        return T


class TransformationEstimationForColoredICP(TransformationEstimation):
    """TransformationEstimation.h:318-395 / TransformationEstimation.cpp:294-432.  The target needs the
    "color_gradients" attribute (``PointCloud.estimate_color_gradients``; ``icp`` / ``multi_scale_icp``
    compute it on the finest pyramid level when it is missing, Registration.cpp:243-263)."""

    def __init__(self, lambda_geometric: float = 0.968, kernel: RobustKernel | None = None):
        if lambda_geometric < 0 or lambda_geometric > 1.0:
            lambda_geometric = 0.968                                  # TransformationEstimation.h:337-340
        self.lambda_geometric = lambda_geometric
        self.kernel = kernel if kernel is not None else RobustKernel()

    @staticmethod
    def _check(source, target, need_gradients=True):
        if not target.has_point_positions() or not source.has_point_positions():
            raise RuntimeError("Source and/or Target pointcloud is empty.")
        if not target.has_point_colors() or not source.has_point_colors():
            raise RuntimeError("Source and/or Target pointcloud missing colors attribute.")
        if not target.has_point_normals():
            raise RuntimeError("Target pointcloud missing normals attribute.")
        if need_gradients and "color_gradients" not in target.point:
            raise RuntimeError("Target pointcloud missing color_gradients attribute.")

    def compute_rmse(self, source, target, correspondences):
        """TransformationEstimation.cpp:294-380 — returns, as upstream, the summed squared joint
        residual (not a root mean), evaluated with torch ops on the device (host-side glue upstream)."""
        self._check(source, target)
        corr = _corr_arg(correspondences, source.point["positions"].shape[0])
        valid = corr != -1
        idx = corr[valid]
        vs, cs = source.point["positions"][valid], source.point["colors"][valid]
        vt, nt = target.point["positions"][idx], target.point["normals"][idx]
        ct, dit = target.point["colors"][idx], target.point["color_gradients"][idx]
        d = ((vs - vt) * nt).sum(1, keepdim=True)
        vs_proj = vs - d * nt
        i_s, i_t = cs.mean(1, keepdim=True), ct.mean(1, keepdim=True)
        is_proj = (dit * (vs_proj - vt)).sum(1, keepdim=True) + i_t
        rg = d * float(np.sqrt(self.lambda_geometric))
        rp = (i_s - is_proj) * float(np.sqrt(1.0 - self.lambda_geometric))
        return float((rg * rg + rp * rp).sum().to(torch.float64))

    def compute_pose(self, source, target, correspondences, target_color_gradients=None):
        """kernel::ComputePoseColoredICP (kernel/Registration.cpp:80-131) through the C ABI seam
        o3db_compute_pose_colored_icp."""
        self._check(source, target, need_gradients=target_color_gradients is None)
        s, sc = source.point["positions"], source.point["colors"]
        t, n, tc = target.point["positions"], target.point["normals"], target.point["colors"]
        g = as_device_f32_points(target.point["color_gradients"] if target_color_gradients is None
                                 else target_color_gradients, "color_gradients")
        corr = _corr_arg(correspondences, s.shape[0])
        pose = torch.zeros(6, dtype=torch.float64, device=s.device)
        sums = torch.zeros(29, dtype=torch.float64, device=s.device)
        residual, count = C.c_float(0), C.c_int(0)
        k = self.kernel._c()
        check(lib.o3db_compute_pose_colored_icp(s.data_ptr(), sc.data_ptr(), t.data_ptr(), n.data_ptr(),
                                                tc.data_ptr(), g.data_ptr(), corr.data_ptr(), s.shape[0],
                                                C.byref(k), float(self.lambda_geometric), sums.data_ptr(),
                                                pose.data_ptr(), C.byref(residual), C.byref(count),
                                                current_stream_ptr()))
        return pose, float(residual.value), int(count.value), sums

    def compute_transformation(self, source, target, correspondences, current_transform=None, iteration=0):
        """TransformationEstimation.cpp:382-432 -> 4x4 Float64 on CPU."""
        pose, _, _, _ = self.compute_pose(source, target, correspondences)
        p = np.ascontiguousarray(pose.cpu().numpy())
        T = np.zeros((4, 4), np.float64)
        lib.o3db_pose_to_transformation(dptr(p), dptr(T))
        return T


class TransformationEstimationSymmetric(TransformationEstimation):
    """TransformationEstimation.h:214-270 / TransformationEstimation.cpp:229-292: Rusinkiewicz's symmetric objective,
    residual (p - q) . (n_p +- n_q).  Both clouds need normals."""

    def __init__(self, kernel: RobustKernel | None = None):
        self.kernel = kernel if kernel is not None else RobustKernel()

    @staticmethod
    def _check(source, target):
        """AssertValidSymmetricInputs (TransformationEstimation.cpp:40-83)."""
        if not target.has_point_positions() or not source.has_point_positions():
            raise RuntimeError("Source and/or Target pointcloud is empty.")
        if "normals" not in source.point or "normals" not in target.point:
            raise RuntimeError("SymmetricICP requires both source and target to have normals.")
        for name, cloud in (("Source", source), ("Target", target)):
            p, n = cloud.point["positions"], cloud.point["normals"]
            if tuple(n.shape) != tuple(p.shape):
                raise RuntimeError(f"{name} normals shape {list(n.shape)} must match {name.lower()} positions shape "
                                   f"{list(p.shape)} for SymmetricICP.")

    def _inputs(self, source, target, correspondences):
        self._check(source, target)
        s, t = source.point["positions"], target.point["positions"]
        ns, nt = source.point["normals"], target.point["normals"]
        return s, t, ns, nt, _corr_arg(correspondences, s.shape[0])

    def compute_rmse(self, source, target, correspondences):
        """TransformationEstimation.cpp:229-274: sqrt(mean(((s - t) . (sign n_s + n_t))^2)) over the valid pairs, 0 with
        none (torch ops on the device, tensor ops upstream)."""
        s, t, ns, nt, corr = self._inputs(source, target, correspondences)
        if bool(((corr < -1) | (corr >= t.shape[0])).any()):
            raise RuntimeError(f"SymmetricICP correspondences must be -1 or a target point index in [0, {t.shape[0]}), "
                               "but an out-of-range value was found.")
        valid = corr != -1
        idx = corr[valid]
        if idx.shape[0] == 0:
            return 0.0
        vs, vt, vns, vnt = s[valid], t[idx], ns[valid], nt[idx]
        dot = (vns * vnt).sum(1, keepdim=True)
        direction = torch.where(dot < 0, -1.0, 1.0).to(dot.dtype)
        r = ((vs - vt) * (vns * direction + vnt)).sum(1)
        return float(torch.sqrt((r * r).mean().to(torch.float64)))

    def compute_pose(self, source, target, correspondences, source_mean, target_mean):
        """kernel::ComputePoseSymmetric (RegistrationCPU.cpp:124-218) about the given means, through the C ABI seam
        o3db_compute_pose_symmetric: pose [6] f64 on the device, residual (sum of squared objective residuals),
        inlier_count and the 29 sums."""
        s, t, ns, nt, corr = self._inputs(source, target, correspondences)
        ms = (C.c_float * 3)(*[float(v) for v in np.asarray(source_mean, np.float32).reshape(3)])
        mt = (C.c_float * 3)(*[float(v) for v in np.asarray(target_mean, np.float32).reshape(3)])
        pose = torch.zeros(6, dtype=torch.float64, device=s.device)
        sums = torch.zeros(29, dtype=torch.float64, device=s.device)
        residual, count = C.c_float(0), C.c_int(0)
        k = self.kernel._c()
        check(lib.o3db_compute_pose_symmetric(s.data_ptr(), t.data_ptr(), ns.data_ptr(), nt.data_ptr(), corr.data_ptr(),
                                              s.shape[0], t.shape[0], ms, mt, C.byref(k), sums.data_ptr(),
                                              pose.data_ptr(), C.byref(residual), C.byref(count), current_stream_ptr()))
        return pose, float(residual.value), int(count.value), sums

    def compute_transformation(self, source, target, correspondences, current_transform=None, iteration=0):
        """TransformationEstimation.cpp:276-292 (kernel::ComputeTransformationSymmetric) -> 4x4 Float64 on CPU; the
        identity when no correspondence is valid."""
        s, t, ns, nt, corr = self._inputs(source, target, correspondences)
        T = np.zeros((4, 4), np.float64)
        k = self.kernel._c()
        check(lib.o3db_compute_transformation_symmetric(s.data_ptr(), t.data_ptr(), ns.data_ptr(), nt.data_ptr(),
                                                        corr.data_ptr(), s.shape[0], t.shape[0], C.byref(k), dptr(T),
                                                        None, current_stream_ptr()))
        return T


class TransformationEstimationForDopplerICP(TransformationEstimation):
    """TransformationEstimation.h:356-470 / TransformationEstimation.cpp:434-523: point-to-plane ICP plus the FMCW
    Doppler term of DICP (Hexsel, Vhavle and Chen, RSS 2022), energy (1 - lambda) E_G + lambda E_D.  The source needs
    "dopplers" ([N] or [N, 1] Float32, radial velocities) and "directions" ([N, 3] Float32, unit rays in the vehicle
    frame, never transformed), the target normals.  The arguments are the C++ constructor's; upstream's one-argument
    Python overload, which passes its value to `period`, is not reproduced.  Each kernel is L2 or Tukey, the two that
    upstream's dual dispatch accepts."""

    def __init__(self, period: float = 0.1, lambda_doppler: float = 0.01, reject_dynamic_outliers: bool = False,
                 doppler_outlier_threshold: float = 2.0, outlier_rejection_min_iteration: int = 2,
                 geometric_robust_loss_min_iteration: int = 0, doppler_robust_loss_min_iteration: int = 2,
                 geometric_kernel: RobustKernel | None = None, doppler_kernel: RobustKernel | None = None,
                 transform_vehicle_to_sensor=None):
        T = np.eye(4) if transform_vehicle_to_sensor is None else transform_vehicle_to_sensor
        if isinstance(T, torch.Tensor):
            T = T.detach().cpu().numpy()
        T = np.asarray(T, np.float64)
        if T.shape != (4, 4):   # core::AssertTensorShape(transform_vehicle_to_sensor, {4, 4})
            raise RuntimeError(f"Tensor has shape {list(T.shape)}, but is expected to have [4, 4].")
        if abs(period) < 1e-3:   # kMinTimePeriod
            raise RuntimeError("Time period too small.")
        if lambda_doppler < 0 or lambda_doppler > 1.0:
            lambda_doppler = 0.01
        self.period = float(period)
        self.lambda_doppler = float(lambda_doppler)
        self.reject_dynamic_outliers = bool(reject_dynamic_outliers)
        self.doppler_outlier_threshold = float(doppler_outlier_threshold)
        self.outlier_rejection_min_iteration = int(outlier_rejection_min_iteration)
        self.geometric_robust_loss_min_iteration = int(geometric_robust_loss_min_iteration)
        self.doppler_robust_loss_min_iteration = int(doppler_robust_loss_min_iteration)
        self.geometric_kernel = geometric_kernel if geometric_kernel is not None else RobustKernel()
        self.doppler_kernel = doppler_kernel if doppler_kernel is not None else RobustKernel()
        self.transform_vehicle_to_sensor = T.copy()

    @property
    def kernel(self):   # the search options' kernel slot (the Doppler handle reads both kernels from _params)
        return self.geometric_kernel

    def __repr__(self):
        return f"TransformationEstimationForDopplerICP with lambda_doppler: {self.lambda_doppler:f}"

    def _params(self):
        p = DopplerParams()
        p.period, p.lambda_doppler = float(self.period), float(self.lambda_doppler)
        p.reject_dynamic_outliers = int(bool(self.reject_dynamic_outliers))
        p.doppler_outlier_threshold = float(self.doppler_outlier_threshold)
        p.outlier_rejection_min_iteration = int(self.outlier_rejection_min_iteration)
        p.geometric_robust_loss_min_iteration = int(self.geometric_robust_loss_min_iteration)
        p.doppler_robust_loss_min_iteration = int(self.doppler_robust_loss_min_iteration)
        p.geometric_kernel, p.doppler_kernel = self.geometric_kernel._c(), self.doppler_kernel._c()
        T = np.asarray(self.transform_vehicle_to_sensor, np.float64)
        if T.shape != (4, 4):
            raise RuntimeError(f"Tensor has shape {list(T.shape)}, but is expected to have [4, 4].")
        p.transform_vehicle_to_sensor[:] = [float(v) for v in T.reshape(16)]
        return p

    @staticmethod
    def _check(source, target):
        """TransformationEstimation.cpp:469-499 (and the positions' dtype, which every estimator here requires)."""
        if not source.has_point_positions() or not target.has_point_positions():
            raise RuntimeError("Source and/or Target pointcloud is empty.")
        if not target.has_point_normals():
            raise RuntimeError("Target pointcloud missing normals attribute.")
        if "dopplers" not in source.point:
            raise RuntimeError("Source pointcloud missing dopplers attribute.")
        if "directions" not in source.point:
            raise RuntimeError("Source pointcloud missing directions attribute.")
        return TransformationEstimationForDopplerICP._doppler_inputs(source)

    @staticmethod
    def _doppler_inputs(source):
        """(dopplers [N], directions [N, 3]) as contiguous Float32 on the device; raises on any other dtype or shape."""
        s, d, r = source.point["positions"], source.point["dopplers"], source.point["directions"]
        n = s.shape[0]
        for name, v in (("positions", s), ("dopplers", d), ("directions", r)):
            if v.dtype != torch.float32:
                raise RuntimeError(f"DopplerICP: source {name} must be Float32, got {v.dtype} (Float64 clouds are not "
                                   "supported).")
        if not (tuple(d.shape) == (n,) or tuple(d.shape) == (n, 1)):
            raise RuntimeError(f"DopplerICP: source dopplers must have shape [{n}] or [{n}, 1], got {list(d.shape)}.")
        if tuple(r.shape) != (n, 3):
            raise RuntimeError(f"DopplerICP: source directions must have shape [{n}, 3], got {list(r.shape)}.")
        return d.reshape(-1).cuda().contiguous(), r.cuda().contiguous()

    def compute_rmse(self, source, target, correspondences):
        """TransformationEstimation.cpp:434-467: the point-to-plane RMSE over the valid pairs (torch ops on the
        device, tensor ops upstream)."""
        self._check(source, target)
        s, t, n = source.point["positions"], target.point["positions"], target.point["normals"]
        corr = _corr_arg(correspondences, s.shape[0])
        valid = corr != -1
        idx = corr[valid]
        e = ((s[valid] - t[idx]) * n[idx]) ** 2
        return float(torch.sqrt(e.sum(dtype=torch.float64) / idx.shape[0]))

    def compute_pose(self, source, target, correspondences, current_transform=None, iteration=0):
        """kernel::ComputePoseDopplerICP (kernel/Registration.cpp:193-312) through the C ABI seam
        o3db_compute_pose_doppler_icp: pose [6] f64 on the device, residual, inlier_count and the 29 sums."""
        dops, dirs = self._check(source, target)
        s, t, n = source.point["positions"], target.point["positions"], target.point["normals"]
        corr = _corr_arg(correspondences, s.shape[0])
        T = as_host_f64_4x4(np.eye(4) if current_transform is None else current_transform, "current_transform")
        pose = torch.zeros(6, dtype=torch.float64, device=s.device)
        sums = torch.zeros(29, dtype=torch.float64, device=s.device)
        residual, count = C.c_float(0), C.c_int(0)
        p = self._params()
        check(lib.o3db_compute_pose_doppler_icp(s.data_ptr(), dops.data_ptr(), dirs.data_ptr(), t.data_ptr(),
                                                n.data_ptr(), corr.data_ptr(), s.shape[0], dptr(T), int(iteration),
                                                C.byref(p), sums.data_ptr(), pose.data_ptr(), C.byref(residual),
                                                C.byref(count), current_stream_ptr()))
        return pose, float(residual.value), int(count.value), sums

    def compute_transformation(self, source, target, correspondences, current_transform=None, iteration=0):
        """TransformationEstimation.cpp:469-519 -> 4x4 Float64 on CPU (PoseToTransformation of the seam's pose)."""
        pose, _, _, _ = self.compute_pose(source, target, correspondences, current_transform, iteration)
        p = np.ascontiguousarray(pose.cpu().numpy())
        T = np.zeros((4, 4), np.float64)
        lib.o3db_pose_to_transformation(dptr(p), dptr(T))
        return T


def pose_to_symmetric_transformation(pose, source_mean, target_mean):
    """kernel::PoseToSymmetricTransformation (TransformationConverter.cpp:106-133, SymmetricICPImpl.h:19-43) on the
    host in f64 -> 4x4."""
    p = np.ascontiguousarray(np.asarray(pose, np.float64).reshape(6))
    ms = np.ascontiguousarray(np.asarray(source_mean, np.float64).reshape(3))
    mt = np.ascontiguousarray(np.asarray(target_mean, np.float64).reshape(3))
    T = np.zeros((4, 4), np.float64)
    lib.o3db_pose_to_symmetric_transformation(dptr(p), dptr(ms), dptr(mt), dptr(T))
    return T


def _options(max_correspondence_distance, criteria, kernel):
    o = IcpOptions()
    o.max_correspondence_distance = float(max_correspondence_distance)
    o.max_iteration = int(criteria.max_iteration)
    o.relative_fitness = float(criteria.relative_fitness)
    o.relative_rmse = float(criteria.relative_rmse)
    o.kernel = kernel._c()
    o.cell_scale = 0.0
    return o


def _assert_inputs(source, target, estimation_method, max_correspondence_distance, scale_idx=0):
    # Registration.cpp:119-219 AssertInputMultiScaleICP
    colored = isinstance(estimation_method, TransformationEstimationForColoredICP)
    if not colored and not isinstance(estimation_method, (TransformationEstimationPointToPoint,
                                                          TransformationEstimationPointToPlane,
                                                          TransformationEstimationSymmetric,
                                                          TransformationEstimationForDopplerICP)):
        raise RuntimeError("open3d_b200 implements TransformationEstimationPointToPoint, ...Symmetric, ...ForDopplerICP, "
                           "...PointToPlane and ...ForColoredICP; other estimators are outside this build's scope "
                           "(SURVEY.md §8f).")
    if not target.has_point_positions() or not source.has_point_positions():
        raise RuntimeError("Source and/or Target pointcloud is empty.")
    if colored:
        if not target.has_point_normals():
            raise RuntimeError("ColoredICP requires target pointcloud to have normals.")
        if not target.has_point_colors():
            raise RuntimeError("ColoredICP requires target pointcloud to have colors.")
        if not source.has_point_colors():
            raise RuntimeError("ColoredICP requires source pointcloud to have colors.")
    elif isinstance(estimation_method, TransformationEstimationPointToPlane) and not target.has_point_normals():
        raise RuntimeError("TransformationEstimationPointToPlane require pre-computed normal vectors for target "
                           "PointCloud.")
    elif isinstance(estimation_method, TransformationEstimationSymmetric):
        TransformationEstimationSymmetric._check(source, target)
    elif isinstance(estimation_method, TransformationEstimationForDopplerICP):
        if not target.has_point_normals():
            raise RuntimeError("DopplerICP requires target pointcloud to have normals.")
        if "dopplers" not in source.point:
            raise RuntimeError("DopplerICP requires source pointcloud to have Doppler velocities.")
        if "directions" not in source.point:
            raise RuntimeError("DopplerICP requires source pointcloud to have pre-computed direction vectors.")
        TransformationEstimationForDopplerICP._doppler_inputs(source)
    if max_correspondence_distance <= 0.0:
        raise RuntimeError(" Max correspondence distance must be greater than 0, but got "
                           f"{max_correspondence_distance} in scale: {scale_idx}.")


def _run_single_scale(source, target, max_dist, init, estimation, criteria, callback, iteration_offset, scale_idx,
                      final_evaluation=True, comm=None):
    """DoSingleScaleICPIterations (Registration.cpp:275-360) as one device-resident loop.  final_evaluation: also
    run ComputeRegistrationResult for the final transformation (MultiScaleICP does so after the LAST scale only,
    Registration.cpp:424-431; between scales the last iteration's own fitness / rmse / transformation are kept).
    comm: this process holds a SHARD of the source (rows shard_range(n, rank, world) of the cloud every rank has in
    full); the target is replicated and every iteration exchanges the 30-double system (SURVEY.md 8e)."""
    s = source.point["positions"]
    t = target.point["positions"]
    opt = _options(max_dist, criteria, estimation.kernel)
    stream = current_stream_ptr()
    handle = C.c_void_p()
    T0 = np.ascontiguousarray(init, dtype=np.float64)
    if isinstance(estimation, TransformationEstimationForColoredICP):
        estimation._check(source, target)
        n = target.point["normals"]
        sc, tc, tg = source.point["colors"], target.point["colors"], target.point["color_gradients"]
        if comm is not None:
            b, e = _shard(s.shape[0], comm)
            s, sc = s[b:e].contiguous(), sc[b:e].contiguous()
        check(lib.o3db_icp_create_colored(s.data_ptr(), sc.data_ptr(), s.shape[0], t.data_ptr(), n.data_ptr(),
                                          tc.data_ptr(), tg.data_ptr(), t.shape[0], dptr(T0), C.byref(opt),
                                          float(estimation.lambda_geometric), comm.handle if comm is not None else None,
                                          stream, C.byref(handle)))
    else:
        if comm is not None:
            b, e = _shard(s.shape[0], comm)
            s = s[b:e].contiguous()
        if isinstance(estimation, TransformationEstimationPointToPoint):
            check(lib.o3db_icp_create_point_to_point(s.data_ptr(), s.shape[0], t.data_ptr(), t.shape[0], dptr(T0),
                                                     C.byref(opt), comm.handle if comm is not None else None, stream,
                                                     C.byref(handle)))
        elif isinstance(estimation, TransformationEstimationSymmetric):
            estimation._check(source, target)
            ns, nt = source.point["normals"], target.point["normals"]
            check(lib.o3db_icp_create_symmetric(s.data_ptr(), ns.data_ptr(), s.shape[0], t.data_ptr(), nt.data_ptr(),
                                                t.shape[0], dptr(T0), C.byref(opt), None, stream, C.byref(handle)))
        elif isinstance(estimation, TransformationEstimationForDopplerICP):
            dops, dirs = estimation._check(source, target)
            nt, p = target.point["normals"], estimation._params()
            check(lib.o3db_icp_create_doppler(s.data_ptr(), dops.data_ptr(), dirs.data_ptr(), s.shape[0], t.data_ptr(),
                                              nt.data_ptr(), t.shape[0], dptr(T0), C.byref(opt), C.byref(p), None,
                                              stream, C.byref(handle)))
        else:
            n = target.point["normals"]
            check(lib.o3db_icp_create(s.data_ptr(), s.shape[0], t.data_ptr(), n.data_ptr(), t.shape[0], dptr(T0),
                                      C.byref(opt), comm.handle if comm is not None else None, stream, C.byref(handle)))
    try:
        check(lib.o3db_icp_iterate(handle, opt.max_iteration, stream))
        res = IcpResult()
        corr = torch.empty(s.shape[0], dtype=torch.int64, device=s.device)
        per_iter = np.zeros((max(opt.max_iteration, 1), 2), np.float64)
        if final_evaluation:
            rc = lib.o3db_icp_finish(handle, C.byref(res), corr.data_ptr(), dptr(per_iter), stream)
        else:
            corr = None
            rc = lib.o3db_icp_state(handle, C.byref(res), dptr(per_iter), stream)
        if rc == ERR_SINGULAR:
            raise O3DBError(rc, "Singular 6x6 linear system detected, tracking failed.")
        check(rc)
    finally:
        lib.o3db_icp_destroy(handle)
    out = RegistrationResult(np.array(res.transformation, np.float64).reshape(4, 4), corr, res.inlier_rmse,
                             res.fitness, bool(res.converged), int(res.num_iterations))
    executed = out.num_iterations + (1 if out.converged else 0)
    if callback is not None:
        # Registration.cpp:330-345 — replayed after the device-resident loop (the per-iteration
        # transformation is not retained; the final one is passed with the last entry).
        for k in range(executed):
            callback({"iteration_index": iteration_offset + k, "scale_index": scale_idx,
                      "scale_iteration_index": k, "inlier_rmse": float(per_iter[k, 1]),
                      "fitness": float(per_iter[k, 0]),
                      "transformation": out.transformation if k == executed - 1 else None})
    return out, executed, per_iter[:executed]


def evaluate_registration(source, target, max_correspondence_distance, transformation=None):
    """EvaluateRegistration (Registration.cpp:64-91): zero ICP iterations.  Runs on the point-to-point handle: the
    evaluation pass is the same for every estimator and this one asks for positions only, as upstream does here."""
    T = as_host_f64_4x4(np.eye(4) if transformation is None else transformation)
    crit = ICPConvergenceCriteria(0, 0, 0)
    est = TransformationEstimationPointToPoint()
    if not target.has_point_positions() or not source.has_point_positions():
        raise RuntimeError("Source and/or Target pointcloud is empty.")
    res, _, _ = _run_single_scale(source, target, max_correspondence_distance, T, est, crit, None, 0, 0)
    res.transformation = T.copy()
    return res


def compute_fpfh_feature(input, max_nn=100, radius=None, indices=None):
    """ComputeFPFHFeature (t/pipelines/registration/Feature.cpp:23-277; pybind feature.cpp) -> torch.float32 [rows, 33]
    on the cloud's device.  With max_nn and radius (the recommended hybrid call) each point's neighbours are the
    max_nn nearest within radius; with radius=None the min(max_nn, n) nearest.  max_nn must be in 4..128; radius-only
    mode (max_nn=None) raises, because the fixed-radius search is not built.  indices (any int sequence or tensor)
    selects rows: one per distinct index, in ascending point order, each equal to that point's row without indices.
    f64 clouds, non-finite positions and non-finite normal components raise (DESIGN.md §4.24, §7)."""
    if max_nn is not None and int(max_nn) <= 3:
        raise RuntimeError("max_nn must be greater than 3.")
    if radius is not None and not float(radius) > 0:
        raise RuntimeError("radius must be greater than 0.")
    if radius is not None and not math.isfinite(float(radius)):
        raise RuntimeError(f"ComputeFPFHFeature: radius must be finite (got {float(radius)})")
    p = input._positions_f32("ComputeFPFHFeature")
    n = int(p.shape[0])
    # an empty cloud has no normal rows to check: it gives [0, 33] (DESIGN.md §7)
    if n > 0 and not input.has_point_normals():
        raise RuntimeError("The input point cloud has no normal.")
    if max_nn is None and radius is None:
        raise RuntimeError("Both max_nn and radius are none.")
    if max_nn is None:
        raise RuntimeError("ComputeFPFHFeature: radius-only search is not supported by open3d_b200; use the hybrid "
                           "call compute_fpfh_feature(input, max_nn=100, radius=radius)")
    max_nn = int(max_nn)
    if max_nn > 128:
        raise RuntimeError(f"ComputeFPFHFeature: max_nn = {max_nn} exceeds the largest list this search supports (128)")
    if n == 0:
        return torch.zeros((0, 33), dtype=torch.float32, device=p.device)
    nrm = input._normals_f32(n)
    sel = None
    if indices is not None:
        sel = torch.as_tensor(indices, device=p.device).reshape(-1)
        if sel.numel() == 0:   # an empty sequence has no dtype of its own
            return torch.zeros((0, 33), dtype=torch.float32, device=p.device)
        if sel.dtype.is_floating_point or sel.dtype.is_complex or sel.dtype == torch.bool:
            raise RuntimeError(f"ComputeFPFHFeature: indices must be integers (got {sel.dtype})")
        sel = sel.to(torch.int64).contiguous()
    rows = n if sel is None else min(n, int(sel.numel()))
    out = torch.zeros((rows, 33), dtype=torch.float32, device=p.device)
    got = C.c_int64(0)
    check(lib.o3db_compute_fpfh_feature(p.data_ptr(), nrm.data_ptr(), n, max_nn,
                                        0.0 if radius is None else float(radius),
                                        None if sel is None else sel.data_ptr(), -1 if sel is None else int(sel.numel()),
                                        out.data_ptr() if rows else None, C.byref(got), current_stream_ptr()))
    return out[:got.value]


def correspondences_from_features(source_features, target_features, mutual_filter=False,
                                  mutual_consistency_ratio=0.1):
    """CorrespondencesFromFeatures (t/pipelines/registration/Feature.cpp:279-333) -> torch.int64 [K, 2] on the device:
    (source row, nearest target row) by the f32 squared feature distance, ties to the lowest target index.  With
    mutual_filter only the mutual pairs are kept, when there are more than mutual_consistency_ratio * N of them; else
    every pair, with upstream's warning.  Features are [N, D] and [M, D] Float32 with the same D >= 1."""
    def _rows(x, name):
        x = torch.as_tensor(x)
        if x.dtype != torch.float32 or x.dim() != 2 or x.shape[1] < 1:
            raise RuntimeError(f"{name} must be a [N, D] Float32 tensor with D >= 1 (got {tuple(x.shape)} {x.dtype})")
        if not x.is_cuda and torch.cuda.is_available():
            x = x.cuda()
        return x.contiguous()
    s, t = _rows(source_features, "source_features"), _rows(target_features, "target_features")
    if s.shape[1] != t.shape[1]:
        raise RuntimeError(f"source and target features have different dimensions ({s.shape[1]} and {t.shape[1]})")
    n = int(s.shape[0])
    out = torch.empty((n, 2), dtype=torch.int64, device=s.device)
    k, mutual = C.c_int64(0), C.c_int64(0)
    ratio = float(np.float32(mutual_consistency_ratio))
    check(lib.o3db_correspondences_from_features(s.data_ptr(), n, t.data_ptr(), int(t.shape[0]), int(s.shape[1]),
                                                 int(bool(mutual_filter)), ratio, out.data_ptr() if n else None,
                                                 C.byref(k), C.byref(mutual), current_stream_ptr()))
    if mutual_filter and n and k.value == n and not np.float32(mutual.value) > np.float32(ratio) * np.float32(n):
        print(f"[Open3D WARNING] Too few correspondences ({mutual.value:d}) after mutual filter, fall back to "
              "original correspondences.")
    return out[:k.value]


class RANSACConvergenceCriteria:
    """RANSACConvergenceCriteria (pipelines/registration/Registration.h:54-76; pybind registration.cpp:877-905):
    max_iteration hypotheses at most, and the confidence that sets the early stop, clamped to [0, 1] (a NaN stays
    NaN, as std::max(std::min(c, 1.0), 0.0) leaves it)."""

    def __init__(self, max_iteration=100000, confidence=0.999):
        self.max_iteration = int(max_iteration)
        c = float(confidence)
        self.confidence = c if math.isnan(c) else max(min(c, 1.0), 0.0)

    def __repr__(self):
        return (f"RANSACConvergenceCriteria[max_iteration_={self.max_iteration:d}, "
                f"confidence_={self.confidence:e}].")


class CorrespondenceChecker:
    """CorrespondenceChecker (pipelines/registration/CorrespondenceChecker.h:28-63): the checkers RANSAC runs on each
    sample before validating it.  Only the three subclasses below run on the device."""
    require_pointcloud_alignment = False


class CorrespondenceCheckerBasedOnEdgeLength(CorrespondenceChecker):
    """Rejects a sample when an edge between two of its source points and the matching target edge differ by more than
    the similarity ratio (CorrespondenceChecker.cpp:19-40)."""

    def __init__(self, similarity_threshold=0.9):
        self.similarity_threshold = float(similarity_threshold)


class CorrespondenceCheckerBasedOnDistance(CorrespondenceChecker):
    """Rejects a sample when a transformed source point lies farther than distance_threshold from its target
    point (CorrespondenceChecker.cpp:42-57)."""
    require_pointcloud_alignment = True

    def __init__(self, distance_threshold):
        self.distance_threshold = float(distance_threshold)


class CorrespondenceCheckerBasedOnNormal(CorrespondenceChecker):
    """Rejects a sample when a rotated source normal and its target normal are more than normal_angle_threshold
    (radians) apart (CorrespondenceChecker.cpp:59-80).  Passes, with upstream's warning, when a cloud has no
    normals."""
    require_pointcloud_alignment = True

    def __init__(self, normal_angle_threshold):
        self.normal_angle_threshold = float(normal_angle_threshold)


def _ransac_checkers(checkers):
    """The C checker struct.  Several checkers of one kind reject what any of them rejects: the smallest distance, the
    largest similarity and the largest cosine, leaving out NaN thresholds, which reject nothing."""
    from ...._lib import RansacCheckers
    edge, dist, cosn = [], [], []
    for c in checkers or ():
        if type(c) is CorrespondenceCheckerBasedOnEdgeLength:
            edge.append(c.similarity_threshold)
        elif type(c) is CorrespondenceCheckerBasedOnDistance:
            dist.append(c.distance_threshold)
        elif type(c) is CorrespondenceCheckerBasedOnNormal:
            cosn.append(math.cos(c.normal_angle_threshold))
        else:
            raise RuntimeError(f"RegistrationRANSAC: unsupported checker {type(c).__name__}; the supported ones are "
                               "CorrespondenceCheckerBasedOnEdgeLength, CorrespondenceCheckerBasedOnDistance and "
                               "CorrespondenceCheckerBasedOnNormal")

    def pick(vals, f):
        finite = [v for v in vals if not math.isnan(v)]
        return f(finite) if finite else math.nan
    return RansacCheckers(int(bool(edge)), int(bool(dist)), int(bool(cosn)), pick(edge, max), pick(dist, min),
                          pick(cosn, max))


def _ransac_correspondences(corres, device):
    c = torch.as_tensor(corres)
    if c.dtype not in (torch.int32, torch.int64) or c.dim() != 2 or c.shape[1] != 2:
        raise RuntimeError(f"RegistrationRANSAC: corres must be an Int32 or Int64 [K, 2] tensor (got "
                           f"{tuple(c.shape)} {c.dtype})")
    return c.to(device=device, dtype=torch.int64).contiguous()


def _registration_ransac(source, target, corres, max_correspondence_distance, estimation_method, ransac_n, checkers,
                         criteria):
    """o3db_registration_ransac -> (RegistrationResult, RansacStats)."""
    from ...._lib import RansacStats
    if estimation_method is not None and (type(estimation_method) is not TransformationEstimationPointToPoint or
                                           getattr(estimation_method, "with_scaling", False)):
        raise RuntimeError("RegistrationRANSAC: only TransformationEstimationPointToPoint() without scaling is "
                           f"supported (got {type(estimation_method).__name__})")
    criteria = RANSACConvergenceCriteria() if criteria is None else criteria
    ransac_n, max_iteration = int(ransac_n), int(criteria.max_iteration)
    for name, v in (("ransac_n", ransac_n), ("max_iteration", max_iteration)):
        if not -2 ** 31 <= v < 2 ** 31:
            raise TypeError(f"RegistrationRANSAC: {name} must fit in a 32-bit int (got {v})")
    chk = _ransac_checkers(checkers)
    s = source._positions_f32("RegistrationRANSAC")
    t = target._positions_f32("RegistrationRANSAC")
    n, m = int(s.shape[0]), int(t.shape[0])
    c = _ransac_correspondences(corres, s.device)
    sn = source._normals_f32(n) if source.has_point_normals() else None
    tn = target._normals_f32(m) if target.has_point_normals() else None
    if chk.use_normal and (sn is None or tn is None) and ransac_n >= 3 and c.shape[0] >= ransac_n and \
            max_correspondence_distance > 0 and max_iteration > 0:
        print("[Open3D WARNING] [CorrespondenceCheckerBasedOnNormal::Check] Pointcloud has no normals.")
    T = np.zeros(16, np.float64)
    out = torch.empty((n,), dtype=torch.int64, device=s.device)
    stats = RansacStats()
    check(lib.o3db_registration_ransac(s.data_ptr(), None if sn is None else sn.data_ptr(), n, t.data_ptr(),
                                       None if tn is None else tn.data_ptr(), m, c.data_ptr(), int(c.shape[0]),
                                       float(max_correspondence_distance), ransac_n, max_iteration,
                                       float(criteria.confidence), C.byref(chk), dptr(T),
                                       out.data_ptr() if n else None, C.byref(stats), current_stream_ptr()))
    res = RegistrationResult(T.reshape(4, 4), out, stats.inlier_rmse, stats.fitness)
    return res, stats


def registration_ransac_based_on_correspondence(source, target, corres, max_correspondence_distance,
                                                estimation_method=None, ransac_n=3, checkers=None, criteria=None):
    """RegistrationRANSACBasedOnCorrespondence (pipelines/registration/Registration.cpp:343-379; pybind
    registration.cpp), run as upstream runs it on one thread, on the device (o3db_registration_ransac).  corres is an
    Int32 or Int64 [K, 2] tensor or array of (source row, target row), as correspondences_from_features returns.
    Hypotheses draw from the library's random engine (open3d_b200.utility.random.seed).  estimation_method is None or
    TransformationEstimationPointToPoint(); checkers any of the three CorrespondenceChecker subclasses.  The result's
    transformation is 4x4 Float64 numpy; correspondence_set is Int64 [n] on the device, -1 for no match (upstream's
    pair list is its (nonzero, value)); converged and num_iterations are False and 0.  Float64 clouds, non-finite
    positions, a non-finite distance and pairs outside the clouds raise (DESIGN.md §4.25, §7)."""
    return _registration_ransac(source, target, corres, max_correspondence_distance, estimation_method, ransac_n,
                                checkers, criteria)[0]


def registration_ransac_based_on_feature_matching(source, target, source_feature, target_feature, mutual_filter,
                                                  max_correspondence_distance, estimation_method=None, ransac_n=3,
                                                  checkers=None, criteria=None):
    """RegistrationRANSACBasedOnFeatureMatching (pipelines/registration/Registration.cpp:381-404): the identity for
    ransac_n < 3 or max_correspondence_distance <= 0, else correspondences_from_features(source_feature,
    target_feature, mutual_filter) and registration_ransac_based_on_correspondence.  Features are [N, D] Float32,
    as compute_fpfh_feature returns them, with one row per point of their cloud."""
    if int(ransac_n) < 3 or max_correspondence_distance <= 0.0:
        s = source._positions_f32("RegistrationRANSAC")
        return RegistrationResult(np.eye(4), torch.full((int(s.shape[0]),), -1, dtype=torch.int64, device=s.device))
    for f, cloud, name in ((source_feature, source, "source"), (target_feature, target, "target")):
        rows = int(torch.as_tensor(f).shape[0])
        npts = int(cloud._positions_f32("RegistrationRANSAC").shape[0])
        if rows != npts:
            raise RuntimeError(f"RegistrationRANSAC: the {name} feature has {rows} rows for {npts} points")
    corres = correspondences_from_features(source_feature, target_feature, mutual_filter)
    return registration_ransac_based_on_correspondence(source, target, corres, max_correspondence_distance,
                                                       estimation_method, ransac_n, checkers, criteria)


class FastGlobalRegistrationOption:
    """FastGlobalRegistrationOption (pipelines/registration/FastGlobalRegistration.h:28-90) with the defaults of
    upstream's Python binding (pybind registration.cpp), where decrease_mu is False."""

    def __init__(self, division_factor=1.4, use_absolute_scale=False, decrease_mu=False,
                 maximum_correspondence_distance=0.025, iteration_number=64, tuple_scale=0.95,
                 maximum_tuple_count=1000, tuple_test=True):
        self.division_factor = float(division_factor)
        self.use_absolute_scale = bool(use_absolute_scale)
        self.decrease_mu = bool(decrease_mu)
        self.maximum_correspondence_distance = float(maximum_correspondence_distance)
        self.iteration_number = int(iteration_number)
        self.tuple_scale = float(tuple_scale)
        self.maximum_tuple_count = int(maximum_tuple_count)
        self.tuple_test = bool(tuple_test)

    def __repr__(self):
        def num(x):   # fmt's {} of a double: the shortest round trip, without a trailing ".0"
            r = repr(float(x))
            return r[:-2] if r.endswith(".0") else r

        def b(x):
            return "true" if x else "false"
        return (f"FastGlobalRegistrationOption(\ndivision_factor={num(self.division_factor)},"
                f"\nuse_absolute_scale={b(self.use_absolute_scale)},\ndecrease_mu={b(self.decrease_mu)},"
                f"\nmaximum_correspondence_distance={num(self.maximum_correspondence_distance)},"
                f"\niteration_number={self.iteration_number:d},\ntuple_scale={num(self.tuple_scale)},"
                f"\nmaximum_tuple_count={self.maximum_tuple_count:d},\ntuple_test={b(self.tuple_test)},\n)")

    def _c(self):
        from ...._lib import FgrOption
        for name in ("iteration_number", "maximum_tuple_count"):
            v = getattr(self, name)
            if not -2 ** 31 <= v < 2 ** 31:
                raise TypeError(f"FastGlobalRegistrationOption: {name} must fit in a 32-bit int (got {v})")
        return FgrOption(self.division_factor, int(self.use_absolute_scale), int(self.decrease_mu),
                         self.maximum_correspondence_distance, self.iteration_number, self.tuple_scale,
                         self.maximum_tuple_count, int(self.tuple_test))


def _registration_fgr(source, target, corres, source_feature, target_feature, option):
    """o3db_registration_fgr -> (RegistrationResult, FgrStats)."""
    from ...._lib import FgrStats
    # upstream binds both functions with "option"_a = FastGlobalRegistrationOption() built by the C++ constructor,
    # whose decrease_mu is true, unlike the Python class's default (FastGlobalRegistration.h:48-56)
    option = FastGlobalRegistrationOption(decrease_mu=True) if option is None else option
    opt = option._c()
    s = source._positions_f32("FastGlobalRegistration")
    t = target._positions_f32("FastGlobalRegistration")
    n, m = int(s.shape[0]), int(t.shape[0])
    c = fs = ft = None
    dim = 0
    if corres is not None:
        c = torch.as_tensor(corres)
        if c.dtype not in (torch.int32, torch.int64) or c.dim() != 2 or c.shape[1] != 2:
            raise RuntimeError(f"FastGlobalRegistration: corres must be an Int32 or Int64 [K, 2] tensor (got "
                               f"{tuple(c.shape)} {c.dtype})")
        c = c.to(device=s.device, dtype=torch.int64).contiguous()
    else:
        fs, ft = torch.as_tensor(source_feature), torch.as_tensor(target_feature)
        for f, rows, name in ((fs, n, "source"), (ft, m, "target")):
            if f.dtype != torch.float32 or f.dim() != 2 or f.shape[1] < 1:
                raise RuntimeError(f"FastGlobalRegistration: the {name} feature must be a [N, D] Float32 tensor "
                                   f"(got {tuple(f.shape)} {f.dtype})")
            if int(f.shape[0]) != rows:
                raise RuntimeError(f"FastGlobalRegistration: the {name} feature has {int(f.shape[0])} rows for "
                                   f"{rows} points")
        if fs.shape[1] != ft.shape[1]:
            raise RuntimeError(f"FastGlobalRegistration: source and target features have different dimensions "
                               f"({fs.shape[1]} and {ft.shape[1]})")
        dim = int(fs.shape[1])
        fs = fs.to(s.device).contiguous()
        ft = ft.to(s.device).contiguous()
    T = np.zeros(16, np.float64)
    out = torch.empty((n,), dtype=torch.int64, device=s.device)
    stats = FgrStats()
    check(lib.o3db_registration_fgr(s.data_ptr(), n, t.data_ptr(), m, None if c is None else c.data_ptr(),
                                    0 if c is None else int(c.shape[0]), None if fs is None else fs.data_ptr(),
                                    None if ft is None else ft.data_ptr(), dim, C.byref(opt), dptr(T),
                                    out.data_ptr() if n else None, C.byref(stats), current_stream_ptr()))
    return RegistrationResult(T.reshape(4, 4), out, stats.inlier_rmse, stats.fitness), stats


def registration_fgr_based_on_correspondence(source, target, corres, option=None):
    """FastGlobalRegistrationBasedOnCorrespondence (pipelines/registration/FastGlobalRegistration.cpp:285-327),
    run as upstream runs it on one thread, on the device (o3db_registration_fgr).  corres is an Int32 or Int64 [K, 2]
    tensor or array of (source row, target row).  The tuple test draws from the library's random engine
    (open3d_b200.utility.random.seed).  The result's transformation is 4x4 Float64 numpy; correspondence_set is Int64
    [n] on the device, -1 for no match; converged and num_iterations are False and 0.  Without option the call uses
    upstream's C++ defaults, as its binding does: those of FastGlobalRegistrationOption() except decrease_mu=True.
    Float64 clouds, non-finite positions and pairs outside the clouds raise (DESIGN.md §4.26, §7)."""
    return _registration_fgr(source, target, corres, None, None, option)[0]


def registration_fgr_based_on_feature_matching(source, target, source_feature, target_feature, option=None):
    """FastGlobalRegistrationBasedOnFeatureMatching (pipelines/registration/FastGlobalRegistration.cpp:329-391): the
    mutual nearest feature rows (f32 distances, ties to the lowest row), then the tuple test and the optimisation as
    registration_fgr_based_on_correspondence.  Features are [N, D] Float32 with one row per point of their cloud, as
    compute_fpfh_feature returns them.  Without option, upstream's C++ defaults (decrease_mu=True) as above."""
    return _registration_fgr(source, target, None, source_feature, target_feature, option)[0]


def get_information_matrix(source, target, max_correspondence_distance, transformation):
    """GetInformationMatrix (Registration.cpp:446-485; pybind registration.get_information_matrix): 6x6 Float64 GTG
    of the target points matched by the transformed source, on the host like upstream."""
    if not target.has_point_positions() or not source.has_point_positions():
        raise RuntimeError("Source and/or Target pointcloud is empty.")
    T = as_host_f64_4x4(transformation, "transformation")
    s, t = source.point["positions"], target.point["positions"]
    info = np.zeros((6, 6), np.float64)
    check(lib.o3db_get_information_matrix(s.data_ptr(), s.shape[0], t.data_ptr(), t.shape[0],
                                          float(max_correspondence_distance), dptr(T), dptr(info), current_stream_ptr()))
    return info


def icp(source, target, max_correspondence_distance, init_source_to_target=None,
        estimation_method=None, criteria=None, voxel_size=-1.0, callback_after_iteration=None, comm=None):
    """ICP() (Registration.cpp:93-106) == MultiScaleICP with one scale."""
    return multi_scale_icp(source, target, [voxel_size], [criteria or ICPConvergenceCriteria()],
                           [max_correspondence_distance], init_source_to_target, estimation_method,
                           callback_after_iteration, comm)


def registration_symmetric_icp(source, target, max_correspondence_distance, init_source_to_target=None,
                               estimation_method=None, criteria=None):
    """registration_symmetric_icp (pybind/t/pipelines/registration/registration.cpp): ICP with
    TransformationEstimationSymmetric() unless another symmetric estimator (e.g. with a robust kernel) is given."""
    if estimation_method is None:
        estimation_method = TransformationEstimationSymmetric()
    return icp(source, target, max_correspondence_distance, init_source_to_target, estimation_method,
               criteria or ICPConvergenceCriteria())


def _shard(n, comm):
    from ....distributed import shard_range
    return shard_range(int(n), comm.rank, comm.world)


def _replicate_from_rank0(cloud, comm):
    """Every rank built the same pyramid level, but VoxelDownSample's output ORDER is unspecified (hash-map slot
    order, as upstream) and its f32 means depend on the atomics' order: rank 0's level is broadcast so that all ranks
    shard one and the same cloud.  One-off per level, outside the iteration loop."""
    import torch.distributed as dist
    n = torch.tensor([cloud.point["positions"].shape[0]], dtype=torch.int64, device="cuda")
    dist.broadcast(n, src=0)
    out = type(cloud)()
    for key in sorted(cloud.point):
        v = cloud.point[key]
        buf = v.contiguous() if comm.rank == 0 else torch.empty((int(n.item()),) + tuple(v.shape[1:]), dtype=v.dtype, device=v.device)
        dist.broadcast(buf, src=0)
        out.point[key] = buf
    return out


def _doppler_voxel_down_sample(cloud, voxel_size):
    """A Doppler source's pyramid level: positions, directions and Doppler values averaged per voxel, as upstream's
    VoxelDownSample averages every attribute (PointCloud.cpp:536-552).  voxel_down_sample averages [N, 3] attributes,
    so the Doppler values ride as the first column of one; the directions are averaged, not renormalised, as upstream."""
    dops, dirs = TransformationEstimationForDopplerICP._doppler_inputs(cloud)
    tmp = PointCloud()
    tmp.point["positions"] = cloud.point["positions"]
    tmp.point["directions"] = dirs
    tmp.point["dopplers3"] = torch.nn.functional.pad(dops[:, None], (0, 2))
    out = tmp.voxel_down_sample(voxel_size)
    out.point["dopplers"] = out.point.pop("dopplers3")[:, 0].contiguous()
    return out


def multi_scale_icp(source, target, voxel_sizes, criteria_list, max_correspondence_distances,
                    init_source_to_target=None, estimation_method=None, callback_after_iteration=None, comm=None):
    """MultiScaleICP (Registration.cpp:362-444).

    comm (extension; upstream is single-device): an open3d_b200.distributed.Communicator.  Every rank passes the SAME
    full clouds; the voxel pyramid and the colour gradients are built once (rank 0's levels are broadcast), each
    level's source is split by rows over the ranks and every iteration exchanges the 30-double system, so all ranks
    return the same transformation / fitness / rmse (correspondence_set covers the rank's own rows)."""
    if estimation_method is None:
        estimation_method = TransformationEstimationPointToPoint()   # Registration.h:140, 205
    if comm is not None and isinstance(estimation_method, TransformationEstimationSymmetric):
        # the multi-GPU exchange carries the 30 sums of one line; this estimator also sums both clouds' points
        raise RuntimeError("TransformationEstimationSymmetric does not run multi-GPU: pass comm=None.")
    if comm is not None and isinstance(estimation_method, TransformationEstimationForDopplerICP):
        raise RuntimeError("TransformationEstimationForDopplerICP does not run multi-GPU: pass comm=None.")
    n_scales = len(criteria_list)
    if len(voxel_sizes) != n_scales or len(max_correspondence_distances) != n_scales:
        raise RuntimeError(" [MultiScaleICP]: Size of criterias, voxel_size, max_correspondence_distances vectors "
                           "must be same.")
    T = as_host_f64_4x4(np.eye(4) if init_source_to_target is None else init_source_to_target,
                        "init_source_to_target")
    for i, d in enumerate(max_correspondence_distances):
        _assert_inputs(source, target, estimation_method, d, i)
    for i in range(n_scales - 1):   # Registration.cpp:190-200: voxel_sizes[i + 1] >= voxel_sizes[i] is an error
        if voxel_sizes[i + 1] >= voxel_sizes[i]:
            raise RuntimeError(" [MultiScaleICP]: Voxel sizes must be in strictly decreasing order.")
    # InitializePointCloudPyramidForMultiScaleICP (Registration.cpp:221-273)
    src_pyr, tgt_pyr = [None] * n_scales, [None] * n_scales
    doppler = isinstance(estimation_method, TransformationEstimationForDopplerICP)
    down_src = _doppler_voxel_down_sample if doppler else (lambda c, v: c.voxel_down_sample(v))
    if voxel_sizes[-1] <= 0:
        src_pyr[-1], tgt_pyr[-1] = source, target          # (the loop clones the source itself)
    else:
        src_pyr[-1], tgt_pyr[-1] = down_src(source, voxel_sizes[-1]), target.voxel_down_sample(voxel_sizes[-1])
    if isinstance(estimation_method, TransformationEstimationForColoredICP) and \
            "color_gradients" not in target.point:          # Registration.cpp:243-263
        if voxel_sizes[-1] <= 0:
            tgt_pyr[-1] = tgt_pyr[-1].clone()               # the caller's target is left untouched
            tgt_pyr[-1].estimate_color_gradients(30, max_correspondence_distances[-1] * 2.0)
        else:
            tgt_pyr[-1].estimate_color_gradients(30, voxel_sizes[-1] * 4.0)
    for k in range(n_scales - 2, -1, -1):
        src_pyr[k] = down_src(src_pyr[k + 1], voxel_sizes[k])
        tgt_pyr[k] = tgt_pyr[k + 1].voxel_down_sample(voxel_sizes[k])
    if comm is not None and comm.world > 1:
        src_pyr = [_replicate_from_rank0(c, comm) for c in src_pyr]
        tgt_pyr = [_replicate_from_rank0(c, comm) for c in tgt_pyr]
    else:
        comm = None
    result = RegistrationResult(T)
    total = 0
    for s_idx in range(n_scales):
        result, executed, _ = _run_single_scale(src_pyr[s_idx], tgt_pyr[s_idx], max_correspondence_distances[s_idx],
                                                result.transformation, estimation_method, criteria_list[s_idx],
                                                callback_after_iteration, total, s_idx,
                                                final_evaluation=(s_idx == n_scales - 1), comm=comm)
        total += result.num_iterations
        if result.fitness <= np.finfo(np.float64).tiny:   # Registration.cpp:434-438
            result.converged = False
            break
    result.num_iterations = total
    return result

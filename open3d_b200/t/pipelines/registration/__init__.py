"""Mirror of ``open3d.t.pipelines.registration`` for the point-to-point, point-to-plane and coloured ICP paths
(cpp/pybind/t/pipelines/registration/registration.cpp:96-140, 469-530;
cpp/open3d/t/pipelines/registration/{Registration,TransformationEstimation}.cpp).

The iteration loop itself runs device-resident inside libo3db200.so
(``o3db_icp_*``); this module only validates arguments the way
``AssertInputMultiScaleICP`` does (Registration.cpp:119-219) and marshals
results into the reference's result type.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from enum import IntEnum

import numpy as np
import torch

from ... import geometry as _geometry
from ...._lib import (ERR_SINGULAR, IcpOptions, IcpResult, O3DBError, RobustKernel as _CRobust, check, dptr, lib)
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
                                                          TransformationEstimationPointToPlane)):
        raise RuntimeError("open3d_b200 implements TransformationEstimationPointToPoint, ...PointToPlane and "
                           "...ForColoredICP; other estimators are outside this build's scope (SURVEY.md §8f).")
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


def multi_scale_icp(source, target, voxel_sizes, criteria_list, max_correspondence_distances,
                    init_source_to_target=None, estimation_method=None, callback_after_iteration=None, comm=None):
    """MultiScaleICP (Registration.cpp:362-444).

    comm (extension; upstream is single-device): an open3d_b200.distributed.Communicator.  Every rank passes the SAME
    full clouds; the voxel pyramid and the colour gradients are built once (rank 0's levels are broadcast), each
    level's source is split by rows over the ranks and every iteration exchanges the 30-double system, so all ranks
    return the same transformation / fitness / rmse (correspondence_set covers the rank's own rows)."""
    if estimation_method is None:
        estimation_method = TransformationEstimationPointToPoint()   # Registration.h:140, 205
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
    if voxel_sizes[-1] <= 0:
        src_pyr[-1], tgt_pyr[-1] = source, target          # (the loop clones the source itself)
    else:
        src_pyr[-1], tgt_pyr[-1] = source.voxel_down_sample(voxel_sizes[-1]), target.voxel_down_sample(voxel_sizes[-1])
    if isinstance(estimation_method, TransformationEstimationForColoredICP) and \
            "color_gradients" not in target.point:          # Registration.cpp:243-263
        if voxel_sizes[-1] <= 0:
            tgt_pyr[-1] = tgt_pyr[-1].clone()               # the caller's target is left untouched
            tgt_pyr[-1].estimate_color_gradients(30, max_correspondence_distances[-1] * 2.0)
        else:
            tgt_pyr[-1].estimate_color_gradients(30, voxel_sizes[-1] * 4.0)
    for k in range(n_scales - 2, -1, -1):
        src_pyr[k] = src_pyr[k + 1].voxel_down_sample(voxel_sizes[k])
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

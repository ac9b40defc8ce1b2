"""Host-side mirror of the pieces of ``open3d.t.geometry`` the hot path touches:
``PointCloud`` (positions / normals / colors + ``transform``), ``Image`` and
``VoxelBlockGrid`` (``compute_unique_block_coordinates``, ``integrate``,
``hashmap``/``attribute`` access).  Reference: cpp/open3d/t/geometry/
{PointCloud,VoxelBlockGrid}.cpp and cpp/pybind/t/geometry/voxel_block_grid.cpp:112-165.
"""
from __future__ import annotations

import ctypes as C
import enum
import math
import weakref

import numpy as np
import torch

from .. import _libshim as _s
from ..._lib import (COLOR_F32, COLOR_NONE, COLOR_U8, DEPTH_F32, DEPTH_U16, ERR_CAPACITY, METRIC_CHAMFER, METRIC_FSCORE,
                     METRIC_HAUSDORFF, O3DBError, check, dptr, lib)
from ._replay import FrameReplay
from ...core import as_device_f32_points, as_host_f64_4x4, current_stream_ptr


class Metric(enum.IntEnum):
    """t::geometry::Metric (t/geometry/Geometry.h:98-102)."""
    ChamferDistance = METRIC_CHAMFER
    HausdorffDistance = METRIC_HAUSDORFF
    FScore = METRIC_FSCORE


class MetricParameters:
    """t::geometry::MetricParameters (t/geometry/Geometry.h:104-113): the F-score radii, and the sample count that
    only mesh metrics use."""

    def __init__(self, fscore_radius=(0.01,), n_sampled_points=1000):
        self.fscore_radius = [float(r) for r in fscore_radius]
        self.n_sampled_points = int(n_sampled_points)


class PointCloud:
    """t::geometry::PointCloud restricted to positions / normals / colors
    (t/geometry/PointCloud.h).  Attributes live in ``self.point`` like upstream."""

    def __init__(self, positions=None, device=None):
        self.point = {}
        if positions is not None:
            self.point["positions"] = as_device_f32_points(positions, "positions")

    # accessors named as in pybind (t/geometry/pointcloud.cpp)
    @property
    def positions(self):
        return self.point.get("positions")

    def has_point_positions(self):
        return "positions" in self.point and self.point["positions"].shape[0] > 0

    def has_point_normals(self):
        return "normals" in self.point and self.point["normals"].shape[0] > 0

    def has_point_colors(self):
        return "colors" in self.point and self.point["colors"].shape[0] > 0

    def set_point_normals(self, normals):
        self.point["normals"] = as_device_f32_points(normals, "normals")
        return self

    def set_point_colors(self, colors):
        self.point["colors"] = as_device_f32_points(colors, "colors")
        return self

    def clone(self):
        out = PointCloud()
        out.point = {k: v.clone() for k, v in self.point.items()}
        return out

    def voxel_down_sample(self, voxel_size, reduction="mean"):
        """PointCloud::VoxelDownSample (t/geometry/PointCloud.cpp:496-560)."""
        if voxel_size <= 0:
            raise RuntimeError("voxel_size must be positive.")
        if reduction != "mean":
            raise RuntimeError("Reduction can only be 'mean' for VoxelDownSample.")
        import ctypes as C
        p = self.point["positions"]
        n = int(p.shape[0])
        # every [n,3] Float32 attribute is averaged per voxel (PointCloud.cpp:536-552)
        names = [k for k, v in self.point.items() if k != "positions"]
        for k in names:
            v = self.point[k]
            if v.dtype != torch.float32 or v.dim() != 2 or v.shape[1] != 3 or v.shape[0] != n:
                raise RuntimeError(f"voxel_down_sample: attribute '{k}' must be [N,3] Float32")
        if len(names) > 4:
            raise RuntimeError("voxel_down_sample: at most 4 attributes besides positions")
        ins = [self.point[k].contiguous() for k in names]
        outs = [torch.empty_like(v) for v in ins]
        po = torch.empty_like(p)
        m = C.c_int64(0)
        in_ptrs = (C.c_void_p * max(len(ins), 1))(*[v.data_ptr() for v in ins])
        out_ptrs = (C.c_void_p * max(len(outs), 1))(*[v.data_ptr() for v in outs])
        check(lib.o3db_voxel_down_sample_attrs(p.data_ptr(), in_ptrs, len(ins), n, float(voxel_size), po.data_ptr(),
                                               out_ptrs, C.byref(m), current_stream_ptr()))
        out = PointCloud()
        out.point["positions"] = po[: m.value].contiguous()
        for k, v in zip(names, outs):
            out.point[k] = v[: m.value].contiguous()
        return out

    def estimate_color_gradients(self, max_nn=30, radius=None, solver="reference"):
        """PointCloud::EstimateColorGradients (t/geometry/PointCloud.cpp:723-767), hybrid search: sets
        the "color_gradients" attribute ColoredICP reads on the target.  solver="reference" (default)
        reproduces upstream's solve_svd3x3<float> bit for bit; "exact" is the exact pseudo-inverse of
        the same f32 normal equations (an extension, not upstream behaviour)."""
        if solver not in ("reference", "exact"):
            raise ValueError("solver must be 'reference' or 'exact'")
        if not self.has_point_colors():
            raise RuntimeError("PointCloud must have colors attribute to estimate color gradients.")
        if not self.has_point_normals():
            raise RuntimeError("PointCloud must have normals attribute to estimate color gradients.")
        if radius is None:
            raise RuntimeError("open3d_b200 builds the hybrid-search variant: pass radius (upstream's KNN-only and "
                               "radius-only variants are outside this build's scope).")
        p, nrm, col = self.point["positions"], self.point["normals"], self.point["colors"]
        g = torch.empty_like(p)
        check(lib.o3db_estimate_color_gradients_solver(p.data_ptr(), nrm.data_ptr(), col.data_ptr(), int(p.shape[0]),
                                                       float(radius), int(max_nn), 0 if solver == "reference" else 1,
                                                       g.data_ptr(), current_stream_ptr()))
        self.point["color_gradients"] = g
        return self

    def estimate_normals(self, max_nn=30, radius=None):
        """PointCloud::EstimateNormals (t/geometry/PointCloud.cpp:856-984), hybrid search: sets "normals" in place.
        If the cloud already has normals, each new normal is flipped where it points against the old one, as
        upstream does; otherwise a point whose normal cannot be estimated gets (0, 0, 1)."""
        p = self._positions_f32("EstimateNormals")
        if radius is None or max_nn is None:
            raise RuntimeError("open3d_b200 builds the hybrid-search variant: pass max_nn and radius (upstream's "
                               "KNN-only and radius-only variants are outside this build's scope).")
        n = int(p.shape[0])
        has_normals = self.has_point_normals()
        if has_normals:
            nrm = self._normals_f32(n)
        else:
            nrm = torch.empty_like(p)
        check(lib.o3db_estimate_normals(p.data_ptr(), n, float(radius), int(max_nn), int(has_normals), nrm.data_ptr(),
                                        None, current_stream_ptr()))
        self.point["normals"] = nrm
        return self

    def orient_normals_to_align_with_direction(self, orientation_reference=(0.0, 0.0, 1.0)):
        """PointCloud::OrientNormalsToAlignWithDirection (t/geometry/PointCloud.cpp:986-1018): in place."""
        d = _vec3_f32(orientation_reference, "orientation_reference")
        if not self.has_point_normals():
            raise RuntimeError("No normals in the PointCloud. Call EstimateNormals() first.")
        nrm = self._normals_f32(int(self._positions_f32("OrientNormalsToAlignWithDirection").shape[0]))
        check(lib.o3db_orient_normals_to_align_with_direction(nrm.data_ptr(), int(nrm.shape[0]), d.ctypes.data,
                                                              current_stream_ptr()))
        self.point["normals"] = nrm
        return self

    def orient_normals_towards_camera_location(self, camera_location=(0.0, 0.0, 0.0)):
        """PointCloud::OrientNormalsTowardsCameraLocation (t/geometry/PointCloud.cpp:1020-1051): in place."""
        c = _vec3_f32(camera_location, "camera_location")
        if not self.has_point_normals():
            raise RuntimeError("No normals in the PointCloud. Call EstimateNormals() first.")
        p = self._positions_f32("OrientNormalsTowardsCameraLocation")
        nrm = self._normals_f32(int(p.shape[0]))
        check(lib.o3db_orient_normals_towards_camera_location(p.data_ptr(), nrm.data_ptr(), int(nrm.shape[0]),
                                                              c.ctypes.data, current_stream_ptr()))
        self.point["normals"] = nrm
        return self

    def compute_boundary_points(self, radius, max_nn=30, angle_threshold=90.0):
        """PointCloud::ComputeBoundaryPoints (t/geometry/PointCloud.cpp:803-853; pybind pointcloud.cpp:628-651) ->
        (PointCloud, mask): a point is on the boundary when the largest angular gap between its hybrid-search
        neighbours (radius, max_nn in 1..32), seen in the plane of its normal, exceeds angle_threshold degrees.  The
        mask is a torch.bool [n] on the device; every attribute is selected by it in the original order.  As upstream,
        the first neighbour of each list is taken to be the point itself, and a normal of exactly (0, 0, +-1), a zero
        normal or a NaN normal gives a NaN plane frame and never a boundary point (for angle_threshold >= 0), so an
        exactly z-facing plane has no boundary.  Non-finite positions and infinite normal components raise.  An empty
        cloud gives an empty cloud and an empty mask."""
        p = self._positions_f32("ComputeBoundaryPoints")
        n = int(p.shape[0])
        if n > 0 and not self.has_point_normals():
            raise RuntimeError("PointCloud must have normals attribute to compute boundary points.")
        radius, max_nn = float(radius), int(max_nn)
        if not radius > 0:
            raise RuntimeError(f"ComputeBoundaryPoints: radius must be positive (got {radius})")
        if not 1 <= max_nn <= 32:
            raise RuntimeError(f"ComputeBoundaryPoints: max_nn must be in 1..32, the hybrid search's limit (got "
                               f"{max_nn})")
        mask = torch.zeros((n,), dtype=torch.bool, device=p.device)
        if n > 0:
            nrm = self._normals_f32(n)
            check(lib.o3db_compute_boundary_points(p.data_ptr(), nrm.data_ptr(), n, radius, max_nn,
                                                   float(angle_threshold), mask.data_ptr(), None,
                                                   current_stream_ptr()))
        out = PointCloud()
        out.point = {k: v[mask] for k, v in self.point.items()}
        return out, mask

    @staticmethod
    def create_from_depth_image(depth, intrinsics, extrinsics=None, depth_scale=1000.0, depth_max=3.0, stride=1,
                                with_normals=False):
        """PointCloud::CreateFromDepthImage (t/geometry/PointCloud.cpp:1414-1442; pybind pointcloud.cpp:451-473): one
        point per strided pixel with 0 < depth / depth_scale < depth_max, in the world frame of extrinsics (default
        identity).  depth: Image, torch tensor or numpy array, [H,W] or [H,W,1] UInt16 / Float32.  Rows row-major over
        the strided grid (see o3db_unproject)."""
        return PointCloud._unproject(depth, None, intrinsics, extrinsics, depth_scale, depth_max, stride, with_normals)

    @staticmethod
    def create_from_rgbd_image(rgbd_image, intrinsics, extrinsics=None, depth_scale=1000.0, depth_max=3.0, stride=1,
                               with_normals=False):
        """PointCloud::CreateFromRGBDImage (PointCloud.cpp:1444-1469; pybind pointcloud.cpp:474-497): as
        create_from_depth_image, plus "colors" = the [H,W,3] UInt8 / Float32 colour pixel as Float32 without scaling
        (0..255 for UInt8, as upstream's color.To(Float32))."""
        return PointCloud._unproject(rgbd_image.depth, rgbd_image.color, intrinsics, extrinsics, depth_scale,
                                     depth_max, stride, with_normals)

    @staticmethod
    def _unproject(depth, color, intrinsics, extrinsics, depth_scale, depth_max, stride, with_normals):
        if with_normals:
            raise RuntimeError("with_normals=True is not built in open3d_b200: upstream's path filters the depth with "
                               "NPP's bilateral filter or PyrDown first, which this build does not reproduce. Create "
                               "the cloud without normals and call estimate_normals().")
        K = _k9(intrinsics)
        E = as_host_f64_4x4(np.eye(4) if extrinsics is None else extrinsics, "extrinsics")
        d = _image_tensor(depth)
        c = _image_tensor(color)
        if d is None:
            d = torch.empty((0, 0, 1), dtype=torch.uint16, device="cuda")
        if d.dim() == 2:
            d = d.unsqueeze(-1)
        if d.dim() != 3 or d.shape[2] != 1:
            raise RuntimeError(f"Depth image must have one channel, got shape {tuple(d.shape)}")
        rows, cols = int(d.shape[0]), int(d.shape[1])
        with_colors = color is not None
        if c is not None and (c.dim() != 3 or c.shape[2] != 3):
            raise RuntimeError(f"Color image must have three channels, got shape {tuple(c.shape)}")
        if with_colors and (rows, cols) != ((0, 0) if c is None else (int(c.shape[0]), int(c.shape[1]))):
            raise RuntimeError("Depth and color images have different sizes.")
        cap = (rows // stride) * (cols // stride) if stride >= 1 else 0
        pts = torch.empty((cap, 3), dtype=torch.float32, device=d.device)
        col = torch.empty((cap, 3), dtype=torch.float32, device=d.device) if with_colors else None
        n = C.c_int64(0)
        check(lib.o3db_unproject(d.data_ptr(), _depth_dtype(d), rows, cols, None if c is None else c.data_ptr(),
                                 _color_dtype(c), dptr(K), dptr(E), float(depth_scale), float(depth_max), int(stride),
                                 pts.data_ptr(), None if col is None else col.data_ptr(), C.byref(n),
                                 current_stream_ptr()))
        out = PointCloud()
        out.point["positions"] = pts[: n.value]
        if with_colors:
            out.point["colors"] = col[: n.value]
        return out

    def project_to_depth_image(self, width, height, intrinsics, extrinsics=None, depth_scale=1000.0, depth_max=3.0):
        """PointCloud::ProjectToDepthImage (PointCloud.cpp:1471-1492): an [height, width, 1] Float32 Image of
        zc * depth_scale, 0 where no point lands; each pixel keeps the nearest point (see o3db_project).  A cloud
        without positions gives an empty image, as upstream."""
        if not self.has_point_positions():
            return Image(torch.empty((0, 0, 1), dtype=torch.float32))
        depth, _ = self._project(width, height, intrinsics, extrinsics, depth_scale, depth_max, False)
        return Image(depth)

    def project_to_rgbd_image(self, width, height, intrinsics, extrinsics=None, depth_scale=1000.0, depth_max=3.0):
        """PointCloud::ProjectToRGBDImage (PointCloud.cpp:1494-1530): RGBDImage(color [height, width, 3], depth
        [height, width, 1]), both Float32; the colour of a pixel is that of the point whose depth it keeps."""
        if not self.has_point_positions():
            return RGBDImage(Image(torch.empty((0, 0, 1), dtype=torch.float32)),
                             Image(torch.empty((0, 0, 1), dtype=torch.float32)))
        if not self.has_point_colors():
            raise RuntimeError("Unable to project to RGBD without the Color attribute in the point cloud.")
        depth, color = self._project(width, height, intrinsics, extrinsics, depth_scale, depth_max, True)
        return RGBDImage(Image(color), Image(depth))

    def _project(self, width, height, intrinsics, extrinsics, depth_scale, depth_max, with_colors):
        p = self._positions_f32("Project")
        n = int(p.shape[0])
        K = _k9(intrinsics)
        E = as_host_f64_4x4(np.eye(4) if extrinsics is None else extrinsics, "extrinsics")
        width, height = int(width), int(height)
        if width < 0 or height < 0:
            raise RuntimeError(f"Invalid image size {width} x {height}")
        depth = torch.empty((height, width, 1), dtype=torch.float32, device=p.device)
        color = cols = None
        if with_colors:
            cols = self.point["colors"]
            if cols.dtype != torch.float32 or cols.dim() != 2 or cols.shape[1] != 3 or cols.shape[0] != n:
                raise RuntimeError(f"colors must be [{n}, 3] Float32, as the positions (got {tuple(cols.shape)} "
                                   f"{cols.dtype})")
            cols = cols.contiguous()
            color = torch.empty((height, width, 3), dtype=torch.float32, device=p.device)
        check(lib.o3db_project(p.data_ptr(), None if cols is None else cols.data_ptr(), n, dptr(K), dptr(E),
                               float(depth_scale), float(depth_max), height, width, depth.data_ptr(),
                               None if color is None else color.data_ptr(), current_stream_ptr()))
        return depth, color

    def remove_statistical_outliers(self, nb_neighbors, std_ratio):
        """PointCloud::RemoveStatisticalOutliers (t/geometry/PointCloud.cpp:678-714) -> (PointCloud, mask): keeps the
        points whose mean distance to their nb_neighbors (1..32) nearest points, itself included, is at most
        mean + std_ratio * std over the cloud.  The mask is a torch.bool on the device; every attribute is selected by
        it in the original order.  The cloud-wide sums are exact-order f64 (o3db_remove_statistical_outliers)."""
        if nb_neighbors < 1 or std_ratio <= 0:
            raise RuntimeError("Illegal input parameters, the number of neighbors and standard deviation ratio must "
                               "be positive.")
        p = self._positions_f32("RemoveStatisticalOutliers")
        n = int(p.shape[0])
        mask = torch.empty((n,), dtype=torch.bool, device=p.device)
        if n == 0:
            return PointCloud(), mask
        check(lib.o3db_remove_statistical_outliers(p.data_ptr(), n, int(nb_neighbors), float(std_ratio),
                                                   mask.data_ptr(), None, current_stream_ptr()))
        out = PointCloud()
        out.point = {k: v[mask] for k, v in self.point.items()}
        return out, mask

    def remove_radius_outliers(self, nb_points, search_radius):
        """PointCloud::RemoveRadiusOutliers (t/geometry/PointCloud.cpp:650-676; pybind pointcloud.cpp:264) ->
        (PointCloud, mask): keeps the points with at least nb_points points, themselves included, within
        search_radius, with the distance test of upstream's CUDA radius search (f32, dist <= radius^2).  The mask is a
        torch.bool [n] on the device; every attribute is selected by it in the original order.  A NaN or infinite
        radius raises, and so do non-finite positions (see remove_non_finite_points).  An empty cloud gives an empty
        cloud and an empty mask."""
        nb_points, search_radius = int(nb_points), float(search_radius)
        if nb_points < 1 or search_radius <= 0:
            raise RuntimeError("Illegal input parameters, number of points and radius must be positive")
        if not math.isfinite(search_radius):
            raise RuntimeError(f"RemoveRadiusOutliers: search_radius must be finite (got {search_radius})")
        p = self._positions_f32("RemoveRadiusOutliers")
        n = int(p.shape[0])
        mask = torch.empty((n,), dtype=torch.bool, device=p.device)
        if n > 0:
            check(lib.o3db_remove_radius_outliers(p.data_ptr(), n, nb_points, search_radius, mask.data_ptr(),
                                                  current_stream_ptr()))
        return self._select(mask), mask

    def remove_duplicated_points(self):
        """PointCloud::RemoveDuplicatedPoints (t/geometry/PointCloud.cpp:740-760) -> (PointCloud, mask): of the points
        whose three coordinates are equal bit for bit (so -0.0 and 0.0 differ, and NaNs with equal bits are equal), the
        one with the lowest index is kept.  The mask is a torch.bool [n] on the device; every attribute is selected by
        it in the original order."""
        p = self._positions_f32("RemoveDuplicatedPoints")
        n = int(p.shape[0])
        mask = torch.empty((n,), dtype=torch.bool, device=p.device)
        if n > 0:
            check(lib.o3db_remove_duplicated_points(p.data_ptr(), n, mask.data_ptr(), current_stream_ptr()))
        return self._select(mask), mask

    def remove_non_finite_points(self, remove_nan=True, remove_inf=True):
        """PointCloud::RemoveNonFinitePoints (t/geometry/PointCloud.cpp:716-738) -> (PointCloud, mask): removes the
        points with a NaN coordinate when remove_nan and those with an infinite one when remove_inf.  The mask is a
        torch.bool [n] on the device; every attribute is selected by it in the original order."""
        p = self._positions_f32("RemoveNonFinitePoints")
        n = int(p.shape[0])
        mask = torch.empty((n,), dtype=torch.bool, device=p.device)
        if n > 0:
            check(lib.o3db_remove_non_finite_points(p.data_ptr(), n, int(bool(remove_nan)), int(bool(remove_inf)),
                                                    mask.data_ptr(), current_stream_ptr()))
        return self._select(mask), mask

    def _select(self, mask):
        out = PointCloud()
        out.point = {k: v[mask] for k, v in self.point.items()}
        return out

    def compute_metrics(self, pcd2, metrics, params=None):
        """PointCloud::ComputeMetrics (t/geometry/PointCloud.cpp:1805-1835, kernel/Metrics.cpp) -> a CPU Float32
        tensor with the values of `metrics` in order, Metric.FScore giving one value per params.fscore_radius.  Both
        nearest-neighbour searches run on the device, where upstream copies the clouds to the CPU."""
        params = MetricParameters() if params is None else params
        if not self.has_point_positions() or not pcd2.has_point_positions():
            raise RuntimeError("One or both input point clouds are empty!")
        p1 = self._positions_f32("ComputeMetrics")
        p2 = pcd2._positions_f32("ComputeMetrics")
        ms = np.ascontiguousarray([int(Metric(m)) for m in metrics], np.int32)
        radius = np.ascontiguousarray(params.fscore_radius, np.float32)
        nval = sum(len(radius) if m == METRIC_FSCORE else 1 for m in ms)
        out = np.zeros(max(nval, 1), np.float32)
        check(lib.o3db_compute_metrics(p1.data_ptr(), int(p1.shape[0]), p2.data_ptr(), int(p2.shape[0]), ms.ctypes.data,
                                       len(ms), radius.ctypes.data, len(radius), out.ctypes.data, nval,
                                       current_stream_ptr()))
        return torch.from_numpy(out[:nval].copy())

    def smooth_laplacian(self, iterations=10, lambda_=0.5, max_nn=20, use_fixed_neighborhoods=False):
        """PointCloud::SmoothLaplacian (t/geometry/PointCloud.cpp:1106-1131) -> a new PointCloud: `iterations` passes
        of x_i <- x_i + lambda_ * (mean of its neighbours - x_i) over the max_nn + 1 nearest points (itself excluded),
        searched again before every pass unless use_fixed_neighborhoods.  Every other attribute is cloned."""
        return self._smooth_knn("SmoothLaplacian", iterations, (lambda_,), max_nn, use_fixed_neighborhoods)

    def smooth_taubin(self, iterations=10, lambda_=0.5, mu=-0.53, max_nn=20, use_fixed_neighborhoods=False):
        """PointCloud::SmoothTaubin (t/geometry/PointCloud.cpp:1133-1158) -> a new PointCloud: each iteration is a
        Laplacian pass with lambda_ and then one with mu (see smooth_laplacian)."""
        return self._smooth_knn("SmoothTaubin", iterations, (lambda_, mu), max_nn, use_fixed_neighborhoods)

    def smooth_mls(self, radius=0.05, max_nn=30):
        """PointCloud::SmoothMLS (t/geometry/PointCloud.cpp:1074-1104) -> a new PointCloud: each point projected onto
        the plane of the Gaussian-weighted PCA of its hybrid-search neighbours (radius <= 0: its max_nn nearest points,
        each of weight 1).  The cloud's normals, if it has them, become the planes' normals."""
        p = self._positions_f32("SmoothMLS")
        out = self.clone()
        n = int(p.shape[0])
        if n == 0:
            return out
        nrm = None
        if self.has_point_normals():
            nrm = out.point["normals"] = self._normals_f32(n).clone()
        pos = out.point["positions"] = torch.empty_like(p)
        check(lib.o3db_smooth_mls(p.data_ptr(), n, float(radius), int(max_nn), pos.data_ptr(),
                                  None if nrm is None else nrm.data_ptr(), current_stream_ptr()))
        return out

    def smooth_bilateral(self, radius=0.05, max_nn=30, sigma_s=0.05, sigma_r=0.05):
        """PointCloud::SmoothBilateral (t/geometry/PointCloud.cpp:1160-1198) -> a new PointCloud carrying the normals:
        each point becomes the mean of its hybrid-search neighbours weighted by their distance (sigma_s) and their
        offset along its normal (sigma_r).  The cloud must have normals (see estimate_normals)."""
        p = self._positions_f32("SmoothBilateral")
        n = int(p.shape[0])
        if n == 0:
            return self.clone()
        if sigma_s <= 0 or sigma_r <= 0:
            raise RuntimeError("Sigma values must be positive.")
        if not self.has_point_normals():
            raise RuntimeError("SmoothBilateral needs normals: upstream estimates missing ones with the KNN-only "
                               "EstimateNormals(), which open3d_b200 does not build. Call estimate_normals(max_nn, "
                               "radius) first.")
        out = self.clone()
        nrm = out.point["normals"] = self._normals_f32(n).clone()
        pos = out.point["positions"] = torch.empty_like(p)
        check(lib.o3db_smooth_bilateral(p.data_ptr(), nrm.data_ptr(), n, float(radius), int(max_nn), float(sigma_s),
                                        float(sigma_r), pos.data_ptr(), current_stream_ptr()))
        return out

    def cluster_dbscan(self, eps, min_points, print_progress=False):
        """PointCloud::ClusterDBSCAN (t/geometry/PointCloud.cpp:1634-1644, geometry/PointCloudCluster.cpp:21-97) -> a
        torch.int32 tensor [n] on the cloud's device: the DBSCAN cluster of every point, -1 for noise.  Points closer
        than eps are neighbours; a point with at least min_points neighbours, itself included, is a core point.  The
        clusters are numbered in the order of their smallest point index, and a border point takes the lowest cluster
        id among its core neighbours, so the labels are upstream's exactly.  print_progress is accepted and ignored."""
        del print_progress
        p = self._positions_f32("ClusterDBSCAN")
        n = int(p.shape[0])
        labels = torch.empty((n,), dtype=torch.int32, device=p.device)
        if n == 0:
            return labels
        check(lib.o3db_cluster_dbscan(p.data_ptr(), n, float(eps), int(min_points), labels.data_ptr(),
                                      current_stream_ptr()))
        return labels

    def segment_plane(self, distance_threshold=0.01, ransac_n=3, num_iterations=100, probability=0.999):
        """PointCloud::SegmentPlane (t/geometry/PointCloud.cpp:1646-1666, geometry/PointCloudSegmentation.cpp:157-279;
        pybind pointcloud.cpp:575-577) -> (plane_model, inliers) on the cloud's device: a torch.float64 [4] plane
        (a, b, c, d) with a*x + b*y + c*z + d = 0, and the torch.int64 indices of its inliers in ascending order.
        RANSAC over num_iterations samples of ransac_n points drawn from the library's random engine
        (open3d_b200.utility.random.seed), stopping early by upstream's rule for the given probability; the result is
        that of upstream's function run on one thread (o3db_segment_plane).  With no valid hypothesis the plane is
        (0, 0, 0, 0) and there are no inliers."""
        p = self._positions_f32("SegmentPlane")
        n = int(p.shape[0])
        ransac_n, num_iterations = int(ransac_n), int(num_iterations)
        for name, v in (("ransac_n", ransac_n), ("num_iterations", num_iterations)):
            if not -2 ** 31 <= v < 2 ** 31:
                # upstream's arguments are C ints, which its binding refuses to take from a larger int
                raise TypeError(f"segment_plane: {name} must fit in a 32-bit int (got {v})")
        plane = torch.empty((4,), dtype=torch.float64, device=p.device)
        inliers = torch.empty((max(n, 1),), dtype=torch.int64, device=p.device)
        k = C.c_int64()
        check(lib.o3db_segment_plane(p.data_ptr(), n, float(distance_threshold), ransac_n, num_iterations,
                                     float(probability), plane.data_ptr(), inliers.data_ptr(), C.byref(k), None,
                                     current_stream_ptr()))
        return plane, inliers[:k.value].clone()

    def farthest_point_down_sample(self, num_samples, start_index=0):
        """PointCloud::FarthestPointDownSample (t/geometry/PointCloud.cpp:612-648; pybind pointcloud.cpp:253-263) -> a
        new PointCloud of num_samples points, in ascending index order with every attribute: starting at start_index,
        each next point is the one farthest (upstream's f32 squared distance) from those already chosen, ties to the
        lowest index.  The whole selection runs in one launch (o3db_farthest_point_down_sample).  num_samples == 0
        gives an empty cloud and num_samples == len(cloud) a clone, before start_index is checked, as upstream."""
        num_samples, start_index = int(num_samples), int(start_index)
        if num_samples < 0 or start_index < 0:
            # upstream's arguments are size_t, which its binding refuses to take from a negative int
            raise RuntimeError(f"farthest_point_down_sample: num_samples and start_index must be non-negative (got "
                               f"{num_samples}, {start_index})")
        p = self._positions_f32("FarthestPointDownSample")
        n = int(p.shape[0])
        if num_samples == 0:
            return PointCloud()
        if num_samples == n:
            return self.clone()
        if num_samples > n:
            raise RuntimeError(f"Illegal number of samples: {num_samples}, must <= point size: {n}")
        if start_index >= n:
            raise RuntimeError(f"Illegal start index: {start_index}, must <= point size: {n}")
        selected = torch.empty((num_samples,), dtype=torch.int32, device=p.device)
        check(lib.o3db_farthest_point_down_sample(p.data_ptr(), n, num_samples, start_index, selected.data_ptr(),
                                                  current_stream_ptr()))
        idx = torch.sort(selected).values.long()
        out = PointCloud()
        out.point = {k: v[idx] for k, v in self.point.items()}
        return out

    def _smooth_knn(self, who, iterations, factors, max_nn, fixed):
        p = self._positions_f32(who)
        if iterations < 0:
            raise RuntimeError(f"{who}: iterations must be non-negative (upstream takes a size_t), got {iterations}")
        out = self.clone()
        n = int(p.shape[0])
        if n == 0:
            return out
        f = np.ascontiguousarray(factors, np.float64)
        pos = out.point["positions"] = torch.empty_like(p)
        check(lib.o3db_smooth_laplacian(p.data_ptr(), n, int(iterations), dptr(f), len(f), int(max_nn), int(bool(fixed)),
                                        pos.data_ptr(), current_stream_ptr()))
        return out

    def _positions_f32(self, who):
        p = self.point.get("positions")
        if p is None:
            raise RuntimeError(f"{who}: the PointCloud has no positions.")
        if p.dtype != torch.float32:
            # upstream also takes Float64; this build implements Float32
            raise RuntimeError(f"{who}: only Float32 point clouds are supported by open3d_b200 (got {p.dtype})")
        return p.contiguous()

    def _normals_f32(self, n):
        nrm = self.point["normals"]
        if nrm.dtype != torch.float32 or nrm.dim() != 2 or nrm.shape[1] != 3 or nrm.shape[0] != n:
            raise RuntimeError(f"normals must be [{n}, 3] Float32, as the positions (got {tuple(nrm.shape)} {nrm.dtype})")
        return nrm.contiguous()

    def transform(self, transformation):
        """PointCloud::Transform (t/geometry/PointCloud.cpp:352-371): in place on
        positions and, if present, normals."""
        T = as_host_f64_4x4(transformation)
        p = self.point["positions"]
        check(lib.o3db_transform_points(dptr(T), p.data_ptr(), p.shape[0], current_stream_ptr()))
        if self.has_point_normals():
            n = self.point["normals"]
            check(lib.o3db_transform_normals(dptr(T), n.data_ptr(), n.shape[0], current_stream_ptr()))
        return self


class TriangleMesh:
    """t::geometry::TriangleMesh as the TSDF extraction returns it: device tensors in ``vertex`` ("positions",
    "normals", "colors") and ``triangle`` ("indices", [T, 3] Int32), as upstream's attribute maps."""

    def __init__(self):
        self.vertex = {}
        self.triangle = {}


class Image:
    """t::geometry::Image as a thin holder of an [H,W,C] tensor."""

    def __init__(self, tensor=None):
        if tensor is None:
            tensor = torch.empty((0, 0, 1), dtype=torch.uint8)
        if isinstance(tensor, np.ndarray):
            tensor = torch.from_numpy(np.ascontiguousarray(tensor))
        if tensor.dim() == 2:
            tensor = tensor.unsqueeze(-1)
        self._t = tensor

    def as_tensor(self):
        return self._t

    @property
    def rows(self):
        return int(self._t.shape[0])

    @property
    def columns(self):
        return int(self._t.shape[1])

    @property
    def channels(self):
        return int(self._t.shape[2])

    # ---- the depth-pyramid members RGB-D odometry uses (t/geometry/Image.cpp:248-285, 409-520)
    def _f32_1ch(self, who):
        t = self._t
        if self.rows <= 0 or self.columns <= 0 or self.channels != 1:
            raise RuntimeError(f"Invalid shape, expected a 1 channel image, but got ({self.rows}, {self.columns}, "
                               f"{self.channels})")
        if t.dtype != torch.float32:
            raise RuntimeError(f"{who}: expected a Float32 image, got {t.dtype}")
        return t.cuda().contiguous()

    def clip_transform(self, scale, min_value, max_value, clip_fill=0.0):
        """Image::ClipTransform (Image.cpp:426-456): UInt16/Float32 -> Float32, in / scale, clipped values filled."""
        if self.rows <= 0 or self.columns <= 0 or self.channels != 1:
            raise RuntimeError(f"Invalid shape, expected a 1 channel image, but got ({self.rows}, {self.columns}, "
                               f"{self.channels})")
        t = self._t.cuda().contiguous()
        out = torch.empty((self.rows, self.columns, 1), dtype=torch.float32, device=t.device)
        check(lib.o3db_image_clip_transform(t.data_ptr(), _depth_dtype(t), self.rows, self.columns, float(scale),
                                            float(min_value), float(max_value), float(clip_fill), out.data_ptr(),
                                            current_stream_ptr()))
        return Image(out)

    def pyr_down_depth(self, diff_threshold, invalid_fill=0.0):
        """Image::PyrDownDepth (Image.cpp:409-424)."""
        t = self._f32_1ch("PyrDownDepth")
        out = torch.empty((self.rows // 2, self.columns // 2, 1), dtype=torch.float32, device=t.device)
        check(lib.o3db_image_pyr_down_depth(t.data_ptr(), self.rows, self.columns, float(diff_threshold),
                                            float(invalid_fill), out.data_ptr(), current_stream_ptr()))
        return Image(out)

    def create_vertex_map(self, intrinsics, invalid_fill=0.0):
        """Image::CreateVertexMap (Image.cpp:458-480)."""
        t = self._f32_1ch("CreateVertexMap")
        out = torch.empty((self.rows, self.columns, 3), dtype=torch.float32, device=t.device)
        check(lib.o3db_image_create_vertex_map(t.data_ptr(), self.rows, self.columns, dptr(_k9(intrinsics)),
                                               float(invalid_fill), out.data_ptr(), current_stream_ptr()))
        return Image(out)

    def create_normal_map(self, invalid_fill=0.0):
        """Image::CreateNormalMap (Image.cpp:482-500) of a vertex map."""
        if self.channels != 3 or self._t.dtype != torch.float32:
            raise RuntimeError(f"Invalid shape, expected a 3 channel Float32 image, but got ({self.rows}, "
                               f"{self.columns}, {self.channels})")
        t = self._t.cuda().contiguous()
        out = torch.empty_like(t)
        check(lib.o3db_image_create_normal_map(t.data_ptr(), self.rows, self.columns, float(invalid_fill),
                                               out.data_ptr(), current_stream_ptr()))
        return Image(out)

    def filter_bilateral(self, kernel_size=3, value_sigma=20.0, dist_sigma=10.0):
        """Image::FilterBilateral (Image.cpp:248-285) for 1-channel Float32 (NPP's documented definition; see
        o3db_image_filter_bilateral)."""
        if kernel_size < 3:
            raise RuntimeError(f"Kernel size must be >= 3, but got {kernel_size}.")
        t = self._f32_1ch("FilterBilateral")
        out = torch.empty_like(t)
        check(lib.o3db_image_filter_bilateral(t.data_ptr(), self.rows, self.columns, int(kernel_size),
                                              float(value_sigma), float(dist_sigma), out.data_ptr(),
                                              current_stream_ptr()))
        return Image(out)


class RGBDImage:
    """t::geometry::RGBDImage (t/geometry/RGBDImage.h): a colour / depth image pair."""

    def __init__(self, color=None, depth=None, aligned=True):
        self.color = color if isinstance(color, Image) else Image(color)
        self.depth = depth if isinstance(depth, Image) else Image(depth)
        self.aligned = aligned


def _image_tensor(img):
    if img is None:
        return None
    if isinstance(img, Image):
        img = img.as_tensor()
    if isinstance(img, np.ndarray):
        img = torch.from_numpy(np.ascontiguousarray(img))
    if img.numel() == 0:
        return None
    if not img.is_cuda:
        img = img.cuda()
    return img.contiguous()


def _depth_dtype(t):
    # CheckDepthTensor (t/geometry/Utility.h:25-44): UInt16 or Float32, one channel
    if t.dtype == torch.uint16:
        return DEPTH_U16
    if t.dtype == torch.float32:
        return DEPTH_F32
    raise RuntimeError(f"Unsupported depth image dtype {t.dtype}")


def _color_dtype(t):
    if t is None:
        return COLOR_NONE
    if t.dtype == torch.uint8:
        return COLOR_U8
    if t.dtype == torch.float32:
        return COLOR_F32
    raise RuntimeError(f"Unsupported color image dtype {t.dtype}")


def _vec3_f32(v, name):
    # the reference takes a 3-vector tensor and casts it to the cloud's dtype (PointCloud.cpp:990-996)
    if isinstance(v, torch.Tensor):
        v = v.detach().cpu().numpy()
    v = np.ascontiguousarray(np.asarray(v).astype(np.float32))
    if v.shape != (3,):
        raise RuntimeError(f"{name}: expected shape {{3}}, got {v.shape}")
    return v


def _k9(K):
    if isinstance(K, torch.Tensor):
        K = K.detach().cpu().numpy()
    K = np.ascontiguousarray(np.asarray(K, dtype=np.float64))
    if K.shape != (3, 3):
        raise RuntimeError(f"Unsupported intrinsic matrix shape {K.shape}")  # CheckIntrinsicTensor
    return K


class _BlockHashMap:
    """View of the grid's core::HashMap (int32x3 keys)."""

    def __init__(self, vbg):
        self._v = vbg

    def size(self):
        return self._v._replay.guard(lambda: int(check(lib.o3db_vbg_size(self._v._h, current_stream_ptr()))))

    def capacity(self):
        return int(lib.o3db_vbg_capacity(self._v._h))

    def reserve(self, capacity):
        check(lib.o3db_vbg_reserve(self._v._h, int(capacity), current_stream_ptr()))

    def _keys_arg(self, keys):
        if isinstance(keys, np.ndarray):
            keys = torch.from_numpy(np.ascontiguousarray(keys))
        if keys.dtype != torch.int32:
            raise RuntimeError(f"Unsupported block coordinate dtype {keys.dtype}")  # CheckBlockCoordinates
        return keys.cuda().contiguous().reshape(-1, 3)

    def activate(self, keys):
        """HashMap::Activate -> (buf_indices int32 [n], masks bool [n])."""
        keys = self._keys_arg(keys)
        n = keys.shape[0]
        buf = torch.empty(n, dtype=torch.int32, device=keys.device)
        masks = torch.empty(n, dtype=torch.uint8, device=keys.device)
        check(lib.o3db_vbg_activate(self._v._h, keys.data_ptr(), n, buf.data_ptr(), masks.data_ptr(),
                                    current_stream_ptr()))
        return buf, masks.bool()

    def find(self, keys):
        keys = self._keys_arg(keys)
        n = keys.shape[0]
        buf = torch.empty(n, dtype=torch.int32, device=keys.device)
        masks = torch.empty(n, dtype=torch.uint8, device=keys.device)
        check(lib.o3db_vbg_find(self._v._h, keys.data_ptr(), n, buf.data_ptr(), masks.data_ptr(),
                                current_stream_ptr()))
        return buf, masks.bool()

    def active_buf_indices(self):
        n = self.size()
        out = torch.empty(n, dtype=torch.int32, device="cuda")
        check(lib.o3db_vbg_active_indices(self._v._h, out.data_ptr(), n, current_stream_ptr()))
        return out

    def key_tensor(self):
        """HashMap::GetKeyTensor: [capacity, 3] int32 view of the key buffer."""
        return _s.device_view(lib.o3db_vbg_key_buffer(self._v._h), (self.capacity(), 3), torch.int32)


class VoxelBlockGrid:
    """t::geometry::VoxelBlockGrid for the slam::Model attribute layout
    (tsdf Float32[1], weight UInt16[1], color UInt16[3]; slam/Model.cpp:28-35)."""

    def __init__(self, attr_names=("tsdf", "weight", "color"),
                 attr_dtypes=(torch.float32, torch.uint16, torch.uint16),
                 attr_channels=((1,), (1,), (3,)), voxel_size=0.0058, block_resolution=16,
                 block_count=10000, device="cuda:0"):
        names = list(attr_names)
        if "tsdf" not in names or "weight" not in names:
            raise RuntimeError("TSDF and/or weight not allocated in blocks, please implement customized integration.")
        layout = dict(zip(names, attr_dtypes))
        if layout["tsdf"] != torch.float32 or layout["weight"] != torch.uint16 or \
                layout.get("color", torch.uint16) != torch.uint16:
            raise RuntimeError("open3d_b200 implements the slam::Model layout only: tsdf Float32, weight UInt16, "
                               "color UInt16")
        self.voxel_size = float(voxel_size)
        self.block_resolution = int(block_resolution)
        self._with_color = "color" in names
        h = C.c_void_p()
        check(lib.o3db_vbg_create(self.voxel_size, self.block_resolution, int(block_count), int(self._with_color),
                                  current_stream_ptr(), C.byref(h)))
        self._h = h
        # HashMap::Activate grows the map on demand (HashMap.cpp:166-181); the fused path reports a frame that did
        # not fit instead, and this puts the reference's behaviour back (see _replay.py).  auto_grow = False hands
        # the O3DB_ERR_CAPACITY error to the caller.
        me = weakref.proxy(self)             # no reference cycle: __del__ frees the device buffers promptly
        self._replay = FrameReplay(lambda *frame: me._submit_frame(*frame), lambda n: me.hashmap().reserve(n),
                                   lambda: me.hashmap().capacity(),
                                   lambda e: isinstance(e, O3DBError) and e.code == ERR_CAPACITY)

    @property
    def auto_grow(self):
        return self._replay.enabled

    @auto_grow.setter
    def auto_grow(self, on):
        self._replay.enabled = bool(on)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and lib is not None:     # (module globals are already torn down at interpreter exit)
            lib.o3db_vbg_destroy(h)
            self._h = None

    def hashmap(self):
        return _BlockHashMap(self)

    def attribute(self, name):
        """VoxelBlockGrid::GetAttribute: [capacity, res, res, res, C] view of a value buffer."""
        cap = int(lib.o3db_vbg_capacity(self._h))
        r = self.block_resolution
        if name == "tsdf":
            return _s.device_view(lib.o3db_vbg_tsdf_buffer(self._h), (cap, r, r, r, 1), torch.float32)
        if name == "weight":
            return _s.device_view(lib.o3db_vbg_weight_buffer(self._h), (cap, r, r, r, 1), torch.uint16)
        if name == "color" and self._with_color:
            return _s.device_view(lib.o3db_vbg_color_buffer(self._h), (cap, r, r, r, 3), torch.uint16)
        raise RuntimeError(f"Attribute {name} not found")

    def compute_unique_block_coordinates(self, depth, intrinsic, extrinsic, depth_scale=1000.0, depth_max=3.0,
                                         trunc_voxel_multiplier=8.0):
        """VoxelBlockGrid::GetUniqueBlockCoordinates(depth, ...) (VoxelBlockGrid.cpp:212-245)."""
        d = _image_tensor(depth)
        if d is None:
            raise RuntimeError("depth image is empty")
        rows, cols = int(d.shape[0]), int(d.shape[1])
        K, E = _k9(intrinsic), as_host_f64_4x4(extrinsic, "extrinsic")
        cap = (rows // 4) * (cols // 4) * 4
        out = torch.empty((cap, 3), dtype=torch.int32, device=d.device)
        n = C.c_int64(0)
        check(lib.o3db_vbg_unique_block_coordinates(self._h, d.data_ptr(), _depth_dtype(d), rows, cols, dptr(K),
                                                    dptr(E), float(depth_scale), float(depth_max),
                                                    float(trunc_voxel_multiplier), out.data_ptr(), cap,
                                                    C.byref(n), current_stream_ptr()))
        return out[: n.value]

    def integrate(self, block_coords, depth, color=None, depth_intrinsic=None, color_intrinsic=None, extrinsic=None,
                  depth_scale=1000.0, depth_max=3.0, trunc_voxel_multiplier=8.0):
        """VoxelBlockGrid::Integrate (VoxelBlockGrid.cpp:292-326)."""
        d = _image_tensor(depth)
        c = _image_tensor(color)
        if d is None:
            raise RuntimeError("depth image is empty")
        rows, cols = int(d.shape[0]), int(d.shape[1])
        if c is not None and (int(c.shape[0]) != rows or int(c.shape[1]) != cols or c.shape[-1] != 3):
            raise RuntimeError("Unsupported color image shape")
        bc = self.hashmap()._keys_arg(block_coords)
        dK = _k9(depth_intrinsic)
        cK = _k9(color_intrinsic if color_intrinsic is not None else depth_intrinsic)
        E = as_host_f64_4x4(extrinsic, "extrinsic")
        check(lib.o3db_vbg_integrate(self._h, bc.data_ptr(), bc.shape[0], d.data_ptr(), _depth_dtype(d),
                                     None if c is None else c.data_ptr(), _color_dtype(c), rows, cols, dptr(dK),
                                     dptr(cK), dptr(E), float(depth_scale), float(depth_max),
                                     float(trunc_voxel_multiplier), current_stream_ptr()))

    # fused path used by slam.Model.integrate
    def integrate_frame(self, depth, color, intrinsic, extrinsic, depth_scale=1000.0, depth_max=3.0,
                        trunc_voxel_multiplier=8.0):
        K, E = _k9(intrinsic), as_host_f64_4x4(extrinsic, "extrinsic").copy()
        host = (isinstance(depth, torch.Tensor) and not depth.is_cuda) or isinstance(depth, np.ndarray)
        if host:
            d = torch.from_numpy(np.ascontiguousarray(depth)) if isinstance(depth, np.ndarray) else depth.contiguous()
            c = None
            if color is not None and (not isinstance(color, torch.Tensor) or color.numel() > 0):
                c = torch.from_numpy(np.ascontiguousarray(color)) if isinstance(color, np.ndarray) else color.contiguous()
        else:
            d, c = _image_tensor(depth), _image_tensor(color)
        self._replay.submit(host, d, c, K, E, float(depth_scale), float(depth_max), float(trunc_voxel_multiplier))

    def _submit_frame(self, host, d, c, K, E, depth_scale, depth_max, trunc_voxel_multiplier):
        rows, cols = int(d.shape[0]), int(d.shape[1])
        fn = lib.o3db_vbg_integrate_frame_host if host else lib.o3db_vbg_integrate_frame
        check(fn(self._h, d.data_ptr(), _depth_dtype(d), None if c is None else c.data_ptr(), _color_dtype(c), rows,
                 cols, dptr(K), dptr(E), depth_scale, depth_max, trunc_voxel_multiplier, current_stream_ptr()))

    _RAYCAST_ATTRS = {"vertex": (3, torch.float32), "normal": (3, torch.float32), "depth": (1, torch.float32),
                      "color": (3, torch.float32), "index": (8, torch.int64), "mask": (8, torch.bool),
                      "interp_ratio": (8, torch.float32), "interp_ratio_dx": (8, torch.float32),
                      "interp_ratio_dy": (8, torch.float32), "interp_ratio_dz": (8, torch.float32)}

    def ray_cast(self, block_coords, intrinsic, extrinsic, width, height, render_attributes=("depth", "color"),
                 depth_scale=1000.0, depth_min=0.1, depth_max=3.0, weight_threshold=3.0,
                 trunc_voxel_multiplier=8.0, range_map_down_factor=8):
        """VoxelBlockGrid::RayCast (VoxelBlockGrid.cpp:328-402; pybind voxel_block_grid.cpp ray_cast) ->
        dict {"range": [h/d, w/d, 2], attr: [h, w, C]}.  block_coords=None takes the blocks touched by the
        last fused integrate_frame without a host round trip (slam::Model::frustum_block_coords_)."""
        from ..._lib import RaycastOutputs
        K, E = _k9(intrinsic), as_host_f64_4x4(extrinsic, "extrinsic")
        width, height, down = int(width), int(height), int(range_map_down_factor)
        out = {}
        ptrs = RaycastOutputs()
        for name in render_attributes:
            if name not in self._RAYCAST_ATTRS:
                raise RuntimeError(f"Unsupported attribute {name}, please implement customized ray casting.")
            ch, dt = self._RAYCAST_ATTRS[name]
            out[name] = torch.empty((height, width, ch), dtype=dt, device="cuda")
            setattr(ptrs, name, out[name].data_ptr())
        rng = torch.empty((max(height // max(down, 1), 0), max(width // max(down, 1), 0), 2), dtype=torch.float32,
                          device="cuda")
        bc = None if block_coords is None else self.hashmap()._keys_arg(block_coords)
        self._replay.guard(lambda: check(lib.o3db_vbg_ray_cast(
            self._h, None if bc is None else bc.data_ptr(), 0 if bc is None else bc.shape[0], dptr(K), dptr(E), width,
            height, C.byref(ptrs), float(depth_scale), float(depth_min), float(depth_max), float(weight_threshold),
            float(trunc_voxel_multiplier), down, rng.data_ptr(), current_stream_ptr())))
        out["range"] = rng
        return out

    def extract_point_cloud(self, weight_threshold=3.0, estimated_point_number=-1):
        """VoxelBlockGrid::ExtractPointCloud (VoxelBlockGrid.cpp:404-434; pybind voxel_block_grid.cpp:180-183): the
        zero crossings of the TSDF between voxels of weight > weight_threshold, as a PointCloud with "positions",
        "normals" and, when the grid has colour, "colors".  Rows in a fixed order (block slot, voxel, axis; see
        o3db_vbg_extract_point_cloud); estimated_point_number >= 0 keeps the first that many."""
        n = C.c_int64(0)
        pts, nrm, col = C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._replay.guard(lambda: check(lib.o3db_vbg_extract_point_cloud(
            self._h, float(weight_threshold), int(estimated_point_number), C.byref(n), C.byref(pts), C.byref(nrm),
            C.byref(col), current_stream_ptr())))
        rows = int(n.value)
        # the library's buffers are reused by the next call: copy out
        out = PointCloud()
        out.point["positions"] = _s.device_view(pts.value, (rows, 3), torch.float32).clone()
        out.point["normals"] = _s.device_view(nrm.value, (rows, 3), torch.float32).clone()
        if self._with_color:
            out.point["colors"] = _s.device_view(col.value, (rows, 3), torch.float32).clone()
        return out

    def extract_triangle_mesh(self, weight_threshold=3.0, estimated_vertex_number=-1):
        """VoxelBlockGrid::ExtractTriangleMesh (VoxelBlockGrid.cpp:436-472; pybind voxel_block_grid.cpp:185-188):
        marching cubes over the cubes whose 8 voxels all have weight > weight_threshold, as a TriangleMesh with
        vertex "positions", "normals", "colors" (grids with colour) and triangle "indices".  Vertices in
        extract_point_cloud's order, triangles by block, voxel and case table (see o3db_vbg_extract_triangle_mesh).
        estimated_vertex_number only sizes buffers: the mesh is always complete."""
        nv, nt = C.c_int64(0), C.c_int64(0)
        pts, nrm, col, tri = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._replay.guard(lambda: check(lib.o3db_vbg_extract_triangle_mesh(
            self._h, float(weight_threshold), int(estimated_vertex_number), C.byref(nv), C.byref(nt), C.byref(pts),
            C.byref(nrm), C.byref(col), C.byref(tri), current_stream_ptr())))
        verts, tris = int(nv.value), int(nt.value)
        # the library's buffers are reused by the next call: copy out
        out = TriangleMesh()
        out.vertex["positions"] = _s.device_view(pts.value, (verts, 3), torch.float32).clone()
        out.vertex["normals"] = _s.device_view(nrm.value, (verts, 3), torch.float32).clone()
        if self._with_color:
            out.vertex["colors"] = _s.device_view(col.value, (verts, 3), torch.float32).clone()
        out.triangle["indices"] = _s.device_view(tri.value, (tris, 3), torch.int32).clone()
        return out

    def last_frustum_block_coordinates(self):
        cap = 76800
        out = torch.empty((cap, 3), dtype=torch.int32, device="cuda")
        n = int(self._replay.guard(
            lambda: check(lib.o3db_vbg_last_frustum_blocks(self._h, out.data_ptr(), cap, current_stream_ptr()))))
        if n > cap:
            out = torch.empty((n, 3), dtype=torch.int32, device="cuda")
            check(lib.o3db_vbg_last_frustum_blocks(self._h, out.data_ptr(), n, current_stream_ptr()))
        return out[:n]

"""Mirror of ``open3d.t.pipelines.slam`` for the integration path
(cpp/open3d/t/pipelines/slam/{Model.cpp,Model.h,Frame.h};
cpp/pybind/t/pipelines/slam/slam.cpp:58-160).

``Model.integrate`` is the fused, host-sync-free pipeline
``o3db_vbg_integrate_frame`` (frustum touch + hash activate + TSDF fusion).
``synthesize_model_frame`` is ``o3db_vbg_ray_cast`` on the last frame's frustum and
``track_frame_to_model`` the device-resident PointToPlane RGB-D odometry of
``open3d_b200.t.pipelines.odometry``: together the dense-SLAM loop of
examples/python/t_reconstruction_system/dense_slam.py.
"""
from __future__ import annotations

import numpy as np
import torch

from ...geometry import Image, RGBDImage, VoxelBlockGrid
from ....core import as_host_f64_4x4


class Frame:
    """slam::Frame (slam/Frame.h): a named bag of image tensors + intrinsics."""

    def __init__(self, height, width, intrinsics, device="cuda:0"):
        self._h, self._w = int(height), int(width)
        K = intrinsics.detach().cpu().numpy() if isinstance(intrinsics, torch.Tensor) else np.asarray(intrinsics)
        self._K = np.ascontiguousarray(K, dtype=np.float64)
        self._data = {}

    def height(self):
        return self._h

    def width(self):
        return self._w

    def get_intrinsics(self):
        return self._K

    def set_data(self, name, data):
        self._data[name] = data

    def get_data(self, name):
        d = self._data.get(name)
        return torch.empty(0) if d is None else d

    def set_data_from_image(self, name, image):
        self._data[name] = image.as_tensor() if isinstance(image, Image) else image

    def get_data_as_image(self, name):
        return Image(self.get_data(name))


_IDENTITY = np.eye(4)   # TrackFrameToModel's initial guess (read only)


def _inverse_transformation(T):
    """t::geometry::InverseTransformation (t/geometry/Utility.h:77-115), f64 on the host: R^T and -R^T t, the
    translation summed in the reference's order (plain Python floats are IEEE doubles: same results as the numpy
    expression, a fraction of its cost on the frame loop's critical path)."""
    (r00, r01, r02, t0), (r10, r11, r12, t1), (r20, r21, r22, t2) = T[0].tolist(), T[1].tolist(), T[2].tolist()
    return np.array([[r00, r10, r20, -(r00 * t0 + r10 * t1 + r20 * t2)],
                     [r01, r11, r21, -(r01 * t0 + r11 * t1 + r21 * t2)],
                     [r02, r12, r22, -(r02 * t0 + r12 * t1 + r22 * t2)],
                     [0.0, 0.0, 0.0, 1.0]])


class Model:
    """slam::Model (slam/Model.cpp:23-36): owns a VoxelBlockGrid{tsdf f32, weight u16,
    color u16x3} and the current frame pose."""

    def __init__(self, voxel_size=0.0058, block_resolution=16, block_count=10000, transformation=None,
                 device="cuda:0"):
        self.voxel_grid = VoxelBlockGrid(("tsdf", "weight", "color"),
                                         (torch.float32, torch.uint16, torch.uint16), ((1,), (1,), (3,)),
                                         voxel_size, block_resolution, block_count, device)
        self.transformation_frame_to_world = as_host_f64_4x4(np.eye(4) if transformation is None else transformation)
        self._extrinsic_of = None            # (pose bytes, its inverse): integrate and ray cast use the same one
        self.frame_id = -1
        self._frustum_dirty = False

    def get_current_frame_pose(self):
        return self.transformation_frame_to_world

    def update_frame_pose(self, frame_id, T_frame_to_world):
        """Model::UpdateFramePose (slam/Model.h:99-108)."""
        if frame_id != self.frame_id + 1:
            print(f"[Warning] Skipped {frame_id - self.frame_id - 1} frames in update T!")
        self.frame_id = frame_id
        self.transformation_frame_to_world = as_host_f64_4x4(T_frame_to_world)

    def integrate(self, input_frame, depth_scale=1000.0, depth_max=3.0, trunc_voxel_multiplier=8.0):
        """Model::Integrate (slam/Model.cpp:91-106)."""
        depth = input_frame.get_data("depth")
        color = input_frame.get_data("color")
        E = self._extrinsic()
        if isinstance(color, torch.Tensor) and color.numel() == 0:
            color = None
        self.voxel_grid.integrate_frame(depth, color, input_frame.get_intrinsics(), E, depth_scale, depth_max,
                                        trunc_voxel_multiplier)
        self._frustum_dirty = True

    def _extrinsic(self):
        """world -> frame of the current pose (InverseTransformation), computed once per pose."""
        key = self.transformation_frame_to_world.tobytes()   # by value: the pose array may be updated in place
        if self._extrinsic_of is None or self._extrinsic_of[0] != key:
            self._extrinsic_of = (key, _inverse_transformation(self.transformation_frame_to_world))
        return self._extrinsic_of[1]

    @property
    def frustum_block_coords(self):
        """Model::frustum_block_coords_ — the block keys touched by the last integrated frame."""
        return self.voxel_grid.last_frustum_block_coordinates()

    def get_hashmap(self):
        return self.voxel_grid.hashmap()

    def extract_pointcloud(self, weight_threshold=3.0, estimated_number=-1):
        """Model::ExtractPointCloud (slam/Model.cpp:108-111; pybind slam.cpp:112-115)."""
        return self.voxel_grid.extract_point_cloud(weight_threshold, estimated_number)

    def extract_trianglemesh(self, weight_threshold=3.0, estimated_number=-1):
        """Model::ExtractTriangleMesh (slam/Model.cpp; pybind slam.cpp:119-122)."""
        return self.voxel_grid.extract_triangle_mesh(weight_threshold, estimated_number)

    def track_frame_to_model(self, input_frame, model_frame, depth_scale=1000.0, depth_max=3.0, depth_diff=0.07,
                             method=None, criteria=(6, 3, 1)):
        """Model::TrackFrameToModel (slam/Model.cpp:68-89): multi-scale RGB-D odometry of the input frame against
        the ray-cast model frame, identity initialisation; returns OdometryResult (source = input -> model)."""
        from .. import odometry
        method = odometry.Method.PointToPlane if method is None else method
        return odometry.rgbd_odometry_multi_scale(
            RGBDImage(input_frame.get_data_as_image("color"), input_frame.get_data_as_image("depth")),
            RGBDImage(model_frame.get_data_as_image("color"), model_frame.get_data_as_image("depth")),
            model_frame.get_intrinsics(), _IDENTITY, depth_scale, depth_max, criteria, method,
            odometry.OdometryLossParams(depth_diff))

    def synthesize_model_frame(self, raycast_frame, depth_scale=1000.0, depth_min=0.1, depth_max=3.0,
                               trunc_voxel_multiplier=8.0, enable_color=True, weight_threshold=-1.0):
        """Model::SynthesizeModelFrame (slam/Model.cpp:38-66): ray-cast the blocks of the last integrated
        frame from the current pose into raycast_frame's "depth" (and "color")."""
        if weight_threshold < 0:
            weight_threshold = min(self.frame_id * 1.0, 3.0)
        # upstream always renders {"depth", "color"} and drops the colour when !enable_color (Model.cpp:49-55);
        # the depth map does not depend on it, so the colour pass (8-corner trilinear gather) is skipped here
        attrs = ("depth", "color") if enable_color else ("depth",)
        res = self.voxel_grid.ray_cast(None, raycast_frame.get_intrinsics(), self._extrinsic(),
                                       raycast_frame.width(), raycast_frame.height(), attrs, depth_scale,
                                       depth_min, depth_max, weight_threshold, trunc_voxel_multiplier)
        raycast_frame.set_data("depth", res["depth"])
        if enable_color:
            raycast_frame.set_data("color", res["color"])
        elif raycast_frame.get_data("color").numel() == 0:
            # a dummy RGB frame keeps RGB-D odometry usable in TrackFrameToModel (Model.cpp:58-64)
            raycast_frame.set_data("color", torch.zeros((raycast_frame.height(), raycast_frame.width(), 3),
                                                        dtype=torch.float32, device="cuda"))

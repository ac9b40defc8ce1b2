"""ctypes binding of libo3db200.so (the C ABI in include/open3d_b200.h).

The library is the product: there is no Python/CPU fallback.  If the shared
object is missing or fails to load, importing this module raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libo3db200.so")

OK = 0
ERR_INVALID, ERR_CUDA, ERR_SINGULAR, ERR_CAPACITY, ERR_NO_BLOCKS, ERR_COMM, ERR_NO_INLIERS = -1, -2, -3, -4, -5, -6, -7
DEPTH_U16, DEPTH_F32 = 0, 1
COLOR_NONE, COLOR_U8, COLOR_F32 = 0, 1, 2
UNIQUE_ID_BYTES = 128

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "or open3d_b200/csrc/build.sh (needs nvcc, sm_90a). open3d_b200 has no CPU fallback.")

lib = C.CDLL(LIB_PATH)


class RobustKernel(C.Structure):
    _fields_ = [("method", C.c_int), ("scale", C.c_double), ("shape", C.c_double)]


class IcpOptions(C.Structure):
    _fields_ = [("max_correspondence_distance", C.c_double), ("max_iteration", C.c_int),
                ("relative_fitness", C.c_double), ("relative_rmse", C.c_double),
                ("kernel", RobustKernel), ("cell_scale", C.c_double)]


class IcpResult(C.Structure):
    _fields_ = [("transformation", C.c_double * 16), ("fitness", C.c_double),
                ("inlier_rmse", C.c_double), ("converged", C.c_int), ("num_iterations", C.c_int),
                ("status", C.c_int), ("num_correspondences", C.c_int64)]


class OdometryCriteria(C.Structure):
    _fields_ = [("max_iteration", C.c_int), ("relative_rmse", C.c_double), ("relative_fitness", C.c_double)]


class OdometryResult(C.Structure):
    _fields_ = [("transformation", C.c_double * 16), ("inlier_rmse", C.c_double), ("fitness", C.c_double),
                ("status", C.c_int), ("iterations", C.c_int)]


class RaycastOutputs(C.Structure):
    """o3db_raycast_outputs: device pointers, None = attribute not requested"""
    _fields_ = [(n, C.c_void_p) for n in ("depth", "vertex", "color", "normal", "index", "mask", "interp_ratio",
                                          "interp_ratio_dx", "interp_ratio_dy", "interp_ratio_dz")]


_vp = C.c_void_p
_i64 = C.c_int64
_dbl = C.c_double
_f = C.c_float
_i = C.c_int
_dp = C.c_void_p   # double* parameters: a plain address (see dptr) — ctypes also accepts POINTER(c_double) objects here

_SIGS = {
    "o3db_last_error": (C.c_char_p, []),
    "o3db_version": (_i, []),
    "o3db_kernel_launch_count": (C.c_uint64, []),
    "o3db_nns_create": (_i, [_vp, _i64, _dbl, _vp, C.POINTER(_vp)]),
    "o3db_nns_destroy": (None, [_vp]),
    "o3db_nns_hybrid_search": (_i, [_vp, _vp, _i64, _dbl, _i, _vp, _vp, _vp, _vp]),
    "o3db_compute_pose_point_to_plane": (_i, [_vp, _vp, _vp, _vp, _i64, C.POINTER(RobustKernel), _vp, _vp,
                                              C.POINTER(_f), C.POINTER(_i), _vp]),
    "o3db_compute_pose_colored_icp": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.POINTER(RobustKernel), _dbl,
                                           _vp, _vp, C.POINTER(_f), C.POINTER(_i), _vp]),
    "o3db_pose_to_transformation": (None, [_dp, _dp]),
    "o3db_transform_points": (_i, [_dp, _vp, _i64, _vp]),
    "o3db_transform_normals": (_i, [_dp, _vp, _i64, _vp]),
    "o3db_voxel_down_sample": (_i, [_vp, _vp, _vp, _i64, _dbl, _vp, _vp, _vp, C.POINTER(_i64), _vp]),
    "o3db_voxel_down_sample_attrs": (_i, [_vp, C.POINTER(_vp), _i, _i64, _dbl, _vp, C.POINTER(_vp), C.POINTER(_i64),
                                          _vp]),
    "o3db_estimate_color_gradients": (_i, [_vp, _vp, _vp, _i64, _dbl, _i, _vp, _vp]),
    "o3db_estimate_color_gradients_solver": (_i, [_vp, _vp, _vp, _i64, _dbl, _i, _i, _vp, _vp]),
    "o3db_estimate_normals": (_i, [_vp, _i64, _dbl, _i, _i, _vp, _vp, _vp]),
    "o3db_orient_normals_to_align_with_direction": (_i, [_vp, _i64, _vp, _vp]),
    "o3db_orient_normals_towards_camera_location": (_i, [_vp, _vp, _i64, _vp, _vp]),
    "o3db_icp_create_colored": (_i, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _dp, C.POINTER(IcpOptions), _dbl, _vp,
                                     _vp, C.POINTER(_vp)]),
    "o3db_icp_colored": (_i, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _dp, C.POINTER(IcpOptions), _dbl,
                              C.POINTER(IcpResult), _vp, _dp, _vp]),
    "o3db_icp_create": (_i, [_vp, _i64, _vp, _vp, _i64, _dp, C.POINTER(IcpOptions), _vp, _vp, C.POINTER(_vp)]),
    "o3db_icp_create_point_to_point": (_i, [_vp, _i64, _vp, _i64, _dp, C.POINTER(IcpOptions), _vp, _vp, C.POINTER(_vp)]),
    "o3db_icp_point_to_point": (_i, [_vp, _i64, _vp, _i64, _dp, C.POINTER(IcpOptions), C.POINTER(IcpResult), _vp, _dp,
                                     _vp]),
    "o3db_compute_rt_point_to_point": (_i, [_vp, _vp, _vp, _i64, _dp, _dp, C.POINTER(_i), _vp]),
    "o3db_get_information_matrix": (_i, [_vp, _i64, _vp, _i64, _dbl, _dp, _dp, _vp]),
    "o3db_compute_information_matrix": (_i, [_vp, _vp, _i64, _dp, _vp, _vp]),
    "o3db_icp_reset": (_i, [_vp, _vp]),
    "o3db_icp_iterate": (_i, [_vp, _i, _vp]),
    "o3db_icp_finish": (_i, [_vp, C.POINTER(IcpResult), _vp, _dp, _vp]),
    "o3db_icp_state": (_i, [_vp, C.POINTER(IcpResult), _dp, _vp]),
    "o3db_icp_destroy": (None, [_vp]),
    "o3db_icp_point_to_plane": (_i, [_vp, _i64, _vp, _vp, _i64, _dp, C.POINTER(IcpOptions), C.POINTER(IcpResult),
                                     _vp, _dp, _vp]),
    "o3db_icp_point_to_plane_host": (_i, [_vp, _i64, _vp, _vp, _i64, _dp, C.POINTER(IcpOptions),
                                          C.POINTER(IcpResult), _vp, _dp]),
    "o3db_comm_get_unique_id": (_i, [_vp]),
    "o3db_comm_create": (_i, [_vp, _i, _i, C.POINTER(_vp)]),
    "o3db_comm_uses_peer_memory": (_i, [_vp]),
    "o3db_comm_allreduce_f64": (_i, [_vp, _vp, _i, _vp]),
    "o3db_comm_destroy": (None, [_vp]),
    "o3db_vbg_create": (_i, [_f, _i, _i64, _i, _vp, C.POINTER(_vp)]),
    "o3db_vbg_destroy": (None, [_vp]),
    "o3db_vbg_size": (_i64, [_vp, _vp]),
    "o3db_vbg_exec_stats": (_i, [_vp, _dp, C.POINTER(_i64), _i, _vp]),
    "o3db_depth_touch": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _f, _f, _f, _f, _i, _vp, _i64, _vp, _vp]),
    "o3db_integrate_blocks": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _i64, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _f, _f,
                                   _f, _f, _vp]),
    "o3db_vbg_capacity": (_i64, [_vp]),
    "o3db_vbg_reserve": (_i, [_vp, _i64, _vp]),
    "o3db_vbg_activate": (_i, [_vp, _vp, _i64, _vp, _vp, _vp]),
    "o3db_vbg_find": (_i, [_vp, _vp, _i64, _vp, _vp, _vp]),
    "o3db_vbg_active_indices": (_i64, [_vp, _vp, _i64, _vp]),
    "o3db_vbg_key_buffer": (_vp, [_vp]),
    "o3db_vbg_tsdf_buffer": (_vp, [_vp]),
    "o3db_vbg_weight_buffer": (_vp, [_vp]),
    "o3db_vbg_color_buffer": (_vp, [_vp]),
    "o3db_hash_keys": (_i, [_vp, _i64, _vp, _vp]),
    "o3db_vbg_unique_block_coordinates": (_i, [_vp, _vp, _i, _i, _i, _dp, _dp, _f, _f, _f, _vp, _i64,
                                               C.POINTER(_i64), _vp]),
    "o3db_vbg_integrate": (_i, [_vp, _vp, _i64, _vp, _i, _vp, _i, _i, _i, _dp, _dp, _dp, _f, _f, _f, _vp]),
    "o3db_vbg_integrate_frame": (_i, [_vp, _vp, _i, _vp, _i, _i, _i, _dp, _dp, _f, _f, _f, _vp]),
    "o3db_vbg_integrate_frame_host": (_i, [_vp, _vp, _i, _vp, _i, _i, _i, _dp, _dp, _f, _f, _f, _vp]),
    "o3db_vbg_integrate_sequence": (_i, [_vp, _i64, _vp, _i, _vp, _i, _i, _i, _dp, _dp, _f, _f, _f, _i, _vp]),
    "o3db_vbg_last_frustum_blocks": (_i64, [_vp, _vp, _i64, _vp]),
    "o3db_image_clip_transform": (_i, [_vp, _i, _i, _i, _f, _f, _f, _f, _vp, _vp]),
    "o3db_image_pyr_down_depth": (_i, [_vp, _i, _i, _f, _f, _vp, _vp]),
    "o3db_image_create_vertex_map": (_i, [_vp, _i, _i, _dp, _f, _vp, _vp]),
    "o3db_image_create_normal_map": (_i, [_vp, _i, _i, _f, _vp, _vp]),
    "o3db_image_filter_bilateral": (_i, [_vp, _i, _i, _i, _f, _f, _vp, _vp]),
    "o3db_compute_odometry_result_point_to_plane": (_i, [_vp, _vp, _vp, _i, _i, _dp, _dp, _f, _f, _dp, _dp, _dp, _dp,
                                                         _vp]),
    "o3db_rgbd_odometry_multi_scale_point_to_plane": (_i, [_vp, _i, _vp, _i, _i, _i, _dp, _dp, _f, _f,
                                                           C.POINTER(OdometryCriteria), _i, _f, _f,
                                                           C.POINTER(OdometryResult), _dp, _vp]),
    "o3db_vbg_estimate_range": (_i, [_vp, _vp, _i64, _dp, _dp, _i, _i, _i, _f, _f, _vp, _vp]),
    "o3db_vbg_ray_cast": (_i, [_vp, _vp, _i64, _dp, _dp, _i, _i, C.POINTER(RaycastOutputs), _f, _f, _f, _f, _f, _i,
                               _vp, _vp]),
    "o3db_vbg_extract_point_cloud": (_i, [_vp, _f, _i64, C.POINTER(_i64), C.POINTER(_vp), C.POINTER(_vp),
                                          C.POINTER(_vp), _vp]),
    "o3db_unproject": (_i, [_vp, _i, _i, _i, _vp, _i, _dp, _dp, _f, _f, _i, _vp, _vp, C.POINTER(_i64), _vp]),
    "o3db_project": (_i, [_vp, _vp, _i64, _dp, _dp, _f, _f, _i, _i, _vp, _vp, _vp]),
    "o3db_vbg_profile": (_i, [_vp, _i]),
    "o3db_vbg_profile_read": (_i, [_vp, _dp, _dp, C.POINTER(_i64)]),
    "o3db_build_spatial_hash_table": (_i, [_vp, _i64, _dbl, C.c_uint32, _vp, _vp, _vp]),
}

EXPORTED_SYMBOLS = tuple(_SIGS)

for _name, (_res, _args) in _SIGS.items():
    _fn = getattr(lib, _name)  # AttributeError here = header / library mismatch: fail loudly
    _fn.restype = _res
    _fn.argtypes = _args


class O3DBError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(message)
        self.code = code


def last_error() -> str:
    return (lib.o3db_last_error() or b"").decode("utf-8", "replace")


def check(rc: int) -> int:
    """Open3D reports errors as std::runtime_error (utility/Logging.h:44-53) -> RuntimeError."""
    if rc < 0:
        raise O3DBError(rc, last_error() or f"open3d_b200 error {rc}")
    return rc


def dptr(arr):
    """Address of a contiguous float64 numpy array, for the double* parameters (the caller keeps the array alive)."""
    return arr.ctypes.data


def launch_count() -> int:
    return int(lib.o3db_kernel_launch_count())

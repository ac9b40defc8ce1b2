"""Cameras, image shapes and depth scales for the TSDF, ray-cast and odometry tests (CPU and GPU).

Every other TSDF / odometry test renders 640x480 frames with PRIMESENSE_K at depth_scale 1000.  The integrate kernel
chooses between code paths from the camera and the image, so each case here names the path it exists to reach, and
the helpers below compute, on the host, the condition that sends it there: a test asserts that condition, so that a
case cannot quietly stop testing what it names.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

import oracle
from tests.synth import PRIMESENSE_K, camera_pose, render_depth


def look_at(pos, yaw_deg, pitch_deg=0.0):
    """T_frame_to_world with the axes of synth.camera_pose (x right, y down, z forward), at `pos`, looking along
    yaw (about +z, 0 = +x) and pitch (positive = down)."""
    yaw, pitch = math.radians(yaw_deg), math.radians(pitch_deg)
    fwd = np.array([math.cos(yaw) * math.cos(pitch), math.sin(yaw) * math.cos(pitch), -math.sin(pitch)])
    right = np.cross(fwd, [0.0, 0.0, 1.0])
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    T = np.eye(4)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = right, down, fwd, pos
    return T


def intrinsic(fx, fy, cx, cy):
    return np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])


def scaled_k(K, f):
    """K of the same camera at f times the resolution (pixel centres stay pixel centres)."""
    K = np.array(K, np.float64)
    return intrinsic(K[0, 0] * f, K[1, 1] * f, (K[0, 2] + 0.5) * f - 0.5, (K[1, 2] + 0.5) * f - 0.5)


def shifted_k(K):
    """A colour camera that differs from the depth camera: fx x 1.01, principal point moved by a few pixels."""
    K = np.array(K, np.float64)
    return intrinsic(K[0, 0] * 1.01, K[1, 1], K[0, 2] + 3.25, K[1, 2] - 2.5)


QVGA_K = scaled_k(PRIMESENSE_K, 0.5)
HD_K = intrinsic(900.0, 900.0, 639.5, 359.5)
ODD_K = intrinsic(301.25, 297.5, 171.3, 118.7)      # fx != fy, principal point off-centre and not on a half pixel
SHORT_K = intrinsic(525.0, 525.0, 319.5, 39.5)

# a rejected depth scale (see fast_scale_ok): 1 / s overflows 65535 / s for every numerator above 3402, so the
# division-free sequence returns NaN where d / s is +inf.  NaN passes `depth > depth_max` and would be integrated as
# a full truncation distance; inf is rejected, as in the reference.  No other scale tried fails the check (every
# multiple of 1/8 up to 12500 and 30 000 random floats up to 65536: Markstein's correction step is exact there), so
# the fallback is only reachable at such an extreme scale.
REJECTED_SCALE = 1e-35


@dataclass(frozen=True)
class Case:
    name: str
    reaches: str                          # which kernel path the case exists to reach
    width: int
    height: int
    K: np.ndarray
    poses: tuple                          # T_frame_to_world per frame
    color_K: np.ndarray | None = None     # None: the depth intrinsics
    f32: bool = False                     # Float32 depth (mm) and colour (0..1) instead of UInt16 / UInt8
    scale: float = 1000.0
    depth_max: float = 3.0
    voxel: float = 0.008
    res: int = 16
    misaligned: bool = False              # images handed over as views whose data_ptr() % 16 == 2
    render_max: float = 3.0                # render_depth's depth_max (metres)

    @property
    def cK(self):
        return self.K if self.color_K is None else self.color_K


def _ring(*ids):
    return tuple(camera_pose(i) for i in ids)


# close-range poses: inside the room box (x in -3..3), 0.25 m and ~0.06 m from the x = 3 wall, looking at it
NEAR_POSES = (look_at([2.75, 0.1, 1.2], 8.0, 10.0), look_at([2.75, 0.0, 1.25], -6.0, 4.0))
TOUCH_POSES = (look_at([2.94, 0.2, 1.3], 5.0, 6.0), look_at([2.935, 0.15, 1.3], -4.0, -5.0))

CASES = {c.name: c for c in (
    Case("qvga", "TMA-staged tile on a small image; u16 depth + u8 colour", 320, 240, QVGA_K, _ring(0, 6, 12)),
    Case("hd", "TMA-staged tile, many work units per frame", 1280, 720, HD_K, _ring(50, 56)),
    Case("hd_f32", "TMA-staged f32 tile (64-pixel rows), many units", 1280, 720, HD_K, _ring(50, 56), f32=True),
    Case("odd", "no tensor map (cols * 2 % 16 != 0): direct reads; touch and range-map remainders", 333, 251, ODD_K,
         _ring(300, 306, 312)),
    Case("short", "no tensor map (rows < 96): direct reads", 640, 80, SHORT_K, _ring(700, 706)),
    Case("misaligned", "no tensor map (base pointer % 16 == 2): direct reads", 640, 480, PRIMESENSE_K, _ring(150, 154),
         misaligned=True),
    Case("near", "unit rectangles wider than the 128 x 96 tile: direct reads", 640, 480, PRIMESENSE_K, NEAR_POSES),
    Case("touching", "unit corners behind the camera (zc <= 1e-3): direct reads", 640, 480, PRIMESENSE_K,
         TOUCH_POSES),
    Case("qvga_colour_k", "same_k = 0 on the fast path (general colour projection)", 320, 240, QVGA_K, _ring(0, 6, 12),
         color_K=shifted_k(QVGA_K)),
    Case("odd_colour_k", "same_k = 0 on the fast path, direct reads", 333, 251, ODD_K, _ring(300, 306, 312),
         color_K=shifted_k(ODD_K)),
    Case("qvga_scale5000", "fast_scale on at depth_scale 5000 (depth x 5)", 320, 240, QVGA_K, _ring(0, 6), scale=5000.0),
    Case("qvga_res8", "generic kernel, block resolution 8", 320, 240, QVGA_K, _ring(0, 6), voxel=0.004, res=8),
    Case("qvga_res4", "generic kernel, block resolution 4", 320, 240, QVGA_K, _ring(0, 6), voxel=0.004, res=4),
    Case("qvga_v02", "16^3 kernel at voxel size 0.02", 320, 240, QVGA_K, _ring(0, 6), voxel=0.02),
    Case("qvga_res32", "generic kernel, res^3 = 32768 voxels per block (larger than the CTA)", 320, 240, QVGA_K,
         _ring(0, 6), voxel=0.02, res=32),
)}

TSDF_CASES = list(CASES)


def frames(case):
    """[(T, E, depth [H, W], colour [H, W, 3])] of the case, as numpy arrays in the case's dtypes and depth scale."""
    out = []
    for T in case.poses:
        depth, col = render_depth(T, K=case.K, width=case.width, height=case.height, depth_max=case.render_max,
                                  with_color=True)
        depth, col = depth.numpy(), col.numpy()
        if case.scale != 1000.0:
            depth = np.round(depth.astype(np.float64) * (case.scale / 1000.0)).astype(np.uint16)
        if case.f32:
            depth, col = depth.astype(np.float32), col.astype(np.float32) / np.float32(255.0)
        out.append((T, oracle.inverse_transformation(T), np.ascontiguousarray(depth), np.ascontiguousarray(col)))
    return out


# ------------------------------------------------------------------------ path conditions (host side)

TILE_ROWS, TILE_ROW_BYTES = 96, 256     # integrate16_kernel's staged tile: 128 u16 or 64 f32 pixels x 96 rows


def tensor_map_possible(data_ptr, rows, cols, elem_size):
    """make_depth_tensor_map's conditions: 16-byte base and pitch, at least one tile wide and high."""
    return data_ptr % 16 == 0 and (cols * elem_size) % 16 == 0 and cols >= TILE_ROW_BYTES // elem_size and \
        rows >= TILE_ROWS


def unit_rectangles(keys, K, E, voxel, elem_size, res=16):
    """For each (block, quarter-block unit) of a 16^3 volume: whether a corner lies behind the camera
    (zc <= 1e-3) and whether the bounding rectangle of its 8 projected corners (rounded as the kernel does) is too
    large for the staged tile.  Returns (n_units, n_behind, n_oversize)."""
    assert res == 16
    keys = np.asarray(keys, np.float64).reshape(-1, 1, 1, 3)
    unit = np.arange(4, dtype=np.float64).reshape(1, 4, 1)
    c = np.arange(8).reshape(1, 1, 8)
    vx = keys[..., 0] * 16 + np.where(c & 1, 15, 0)
    vy = keys[..., 1] * 16 + np.where(c & 2, 15, 0)
    vz = keys[..., 2] * 16 + unit * 4 + np.where(c & 4, 3, 0)
    p = np.stack(np.broadcast_arrays(vx, vy, vz), -1) * voxel
    E = np.asarray(E, np.float64)
    cam = p @ E[:3, :3].T + E[:3, 3]
    zc = cam[..., 2]
    behind = (zc <= 1e-3).any(-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        u = K[0, 0] * cam[..., 0] / zc + K[0, 2]
        v = K[1, 1] * cam[..., 1] / zc + K[1, 2]
    align = 16 // elem_size
    x0 = (np.floor(u.min(-1)).astype(np.int64) - 1) & ~(align - 1)
    x1 = np.floor(u.max(-1)).astype(np.int64) + 1
    y0 = np.floor(v.min(-1)).astype(np.int64) - 1
    y1 = np.floor(v.max(-1)).astype(np.int64) + 1
    oversize = ~behind & ((x1 - x0 >= TILE_ROW_BYTES // elem_size) | (y1 - y0 >= TILE_ROWS))
    return behind.size, int(behind.sum()), int(oversize.sum())


def _fma32(a, b, c):
    """fmaf on float32 arrays: a*b is exact in f64, TwoSum gives the exact a*b + c as s + e, and a tie of the final
    rounding to f32 (s exactly between two floats) is broken by the sign of e."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        s = p + c64
        bv = s - p
        e = (p - (s - bv)) + (c64 - bv)
        f = s.astype(np.float32)
        f64 = f.astype(np.float64)
        other = np.nextafter(f, np.where(s > f64, np.float32(np.inf), np.float32(-np.inf)))
        tie = np.isfinite(s) & (s == (f64 + other.astype(np.float64)) / 2) & (e != 0)
    return np.where(tie, np.where(e > 0, np.maximum(f, other), np.minimum(f, other)), f)


def fast_scale_failures(s):
    """The u16 numerators for which tsdf.cu's division-free depth / depth_scale (q = d y, r = fma(-q, s, d),
    q' = fma(r, y, q), y = RN(1 / s)) differs from RN(d / s).  The library enables that sequence for a scale only
    when this set is empty (verify_fast_scale)."""
    s = np.float32(s)
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        y = np.float32(1.0) / s
        d = np.arange(65536, dtype=np.float32)
        q = d * y
        r = _fma32(-q, np.full_like(d, s), d)
        fast = _fma32(r, np.full_like(d, y), q)
        exact = d / s
    same = (fast == exact) | (np.isnan(fast) & np.isnan(exact))
    same &= ~(np.isnan(fast) ^ np.isnan(exact))
    return np.nonzero(~same)[0]


def fast_scale_ok(s):
    return bool(s > 0) and math.isfinite(s) and len(fast_scale_failures(s)) == 0

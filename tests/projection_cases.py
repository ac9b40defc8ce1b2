"""Inputs of the point-cloud <-> image projection tests (CPU and GPU): depth / RGB-D frames to unproject and clouds to
project, each named for what it exercises.  Frames come from tests.synth.render_depth and the cameras of
tests.camera_cases; clouds from tests.synth.make_icp_pair, the unprojected frames and hand-placed points."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

import oracle
from tests import camera_cases as cc
from tests.synth import PRIMESENSE_K, camera_pose, make_colors, make_icp_pair, render_depth


@dataclass(frozen=True)
class Frame:
    depth: np.ndarray                 # [H, W] u16 or f32
    color: np.ndarray | None          # [H, W, 3] u8 or f32
    K: np.ndarray
    E: np.ndarray                     # world -> camera
    scale: float = 1000.0
    depth_max: float = 3.0
    stride: int = 1


def _room(i=0, K=PRIMESENSE_K, width=640, height=480):
    d, c = render_depth(camera_pose(i), K=K, width=width, height=height, with_color=True)
    return d.numpy(), c.numpy()


def inline_fixture():
    """The reference's own unit test (cpp/tests/t/geometry/PointCloud.cpp:993-1041): 2x2 u16 depth, f32 colour."""
    depth = np.array([[1000, 0], [1000, 1000]], np.uint16)
    color = np.array([[[0.0] * 3, [0.2] * 3], [[0.1] * 3, [0.3] * 3]], np.float32)
    K = np.array([[10.0, 0, 1], [0, 10, 1], [0, 0, 1]], np.float32).astype(np.float64)
    return Frame(depth, color, K, np.eye(4))


def _at_depth_max():
    """u16 depth whose values include 1999, 2000 and 2001 mm at depth_max = 2.0 m: 2000 / 1000 == 2.0 exactly and is
    excluded (the bound is strict)."""
    d, c = _room(3)
    d = d.copy()
    d[::3, ::5] = 2000
    d[1::7, ::3] = 1999
    d[2::11, 1::4] = 2001
    return Frame(d, c, PRIMESENSE_K, oracle.inverse_transformation(camera_pose(3)), depth_max=2.0)


def _f32_at_depth_max():
    d, _ = _room(4)
    d = d.astype(np.float32) / np.float32(1000.0)
    d[::4, ::4] = np.float32(2.5)
    return Frame(d, None, PRIMESENSE_K, np.eye(4), scale=1.0, depth_max=2.5)


def unproject_cases():
    """{name: Frame}"""
    d, c = _room(0)
    E0 = oracle.inverse_transformation(camera_pose(0))
    out = {
        "inline": inline_fixture(),
        "room_u16": Frame(d, None, PRIMESENSE_K, np.eye(4)),
        "room_u16_rgb8_pose": Frame(d, c, PRIMESENSE_K, E0),
        "room_f32_rgbf_pose": Frame(d.astype(np.float32), c.astype(np.float32) / np.float32(255.0), PRIMESENSE_K,
                                    E0),
        "room_f32_metres_scale1": Frame(d.astype(np.float32) / np.float32(1000.0), c, PRIMESENSE_K, E0, scale=1.0),
        "room_u16_scale5000": Frame(np.round(d.astype(np.float64) * 5).astype(np.uint16), c, PRIMESENSE_K, E0,
                                    scale=5000.0),
        "at_depth_max_u16": _at_depth_max(),
        "at_depth_max_f32": _f32_at_depth_max(),
    }
    for s in (2, 3, 4, 7):
        out[f"room_rgb8_pose_stride{s}"] = Frame(d, c, PRIMESENSE_K, E0, stride=s)
    for name, strides in (("qvga", (1, 3)), ("hd", (1, 4)), ("hd_f32", (2,)), ("odd", (1, 2, 7)),
                          ("short", (1, 3))):
        case = cc.CASES[name]
        _, E, depth, col = cc.frames(case)[0]
        for s in strides:
            out[f"{name}_stride{s}"] = Frame(depth, col, case.K, E, scale=case.scale, stride=s)
    return out


@dataclass(frozen=True)
class Cloud:
    points: np.ndarray                # [N, 3] f32
    colors: np.ndarray                # [N, 3] f32; column 0 holds the point index (exact below 2^24)
    K: np.ndarray
    E: np.ndarray
    width: int = 640
    height: int = 480
    scale: float = 1000.0
    depth_max: float = 3.0


def indexed_colors(points, seed=0):
    """Colours whose first channel is the point's index, so that an image says which point won each pixel."""
    with np.errstate(invalid="ignore"):   # NaN / inf points get NaN colours
        c = make_colors(points, seed)
    c[:, 0] = np.arange(len(points), dtype=np.float32)
    return np.ascontiguousarray(c, np.float32)


def _above(points, height):
    """World -> camera of a camera with the world's axes, `height` below the cloud's centre, looking along +z."""
    T = np.eye(4)
    T[:3, 3] = [points[:, 0].mean(), points[:, 1].mean(), -height]
    return oracle.inverse_transformation(T)


def _icp_cloud(n, seed=1):
    _, tgt, _, _ = make_icp_pair(n, seed=seed)
    return tgt


def _pixel_edges():
    """K = I and z = 1, so u = x and v = y exactly: half-pixel centres, the -0.5 / -0.49 pair (-0.5 rounds to -1 and
    is rejected, -0.49 to -0 and is kept), the far edges, and zc == depth_max (kept) next to the float above it."""
    xs = np.array([-0.5, -0.49, 0.0, 0.5, 1.5, 2.5, 7.5, 8.49, 8.5, 9.0], np.float32)   # width 10: 9.49 is the last
    ys = np.array([-0.5, -0.49, 0.5, 3.5, 5.49, 5.5], np.float32)                         # height 6
    x, y = np.meshgrid(xs, ys)
    z = np.ones_like(x)
    pts = [np.stack([x.ravel(), y.ravel(), z.ravel()], 1)]
    dm = np.float32(3.0)
    pts.append(np.array([[5.0 * dm, 2.0 * dm, dm], [6.0 * dm, 2.0 * dm, np.nextafter(dm, np.float32(4))]],
                        np.float32))   # (u, v) = (5, 2) at z = 3 and (6, 2) just beyond
    return np.ascontiguousarray(np.concatenate(pts), np.float32)


def _hostile(seed=5):
    """Points behind the camera, on its plane, NaN and inf coordinates among ordinary ones."""
    rng = np.random.default_rng(seed)
    p = rng.uniform([-2, -1.5, -2.0], [2, 1.5, 4.0], (20000, 3)).astype(np.float32)
    p[::97, 2] = 0.0
    p[1::89, 0] = np.nan
    p[2::83, 1] = np.inf
    p[3::79, 2] = -np.inf
    p[4::73, 2] = np.inf
    p[5::71] = np.nan
    return p


def _duplicates(seed=6):
    """Coincident points: each of 500 points repeated 4 times at scattered indices."""
    rng = np.random.default_rng(seed)
    base = rng.uniform([-1, -0.8, 1.0], [1, 0.8, 2.5], (500, 3)).astype(np.float32)
    p = np.concatenate([base] * 4)
    return np.ascontiguousarray(p[rng.permutation(len(p))], np.float32)


def project_cases():
    """{name: Cloud}"""
    out = {}
    tgt = _icp_cloud(200000)
    out["icp_200k"] = Cloud(tgt, indexed_colors(tgt), PRIMESENSE_K, _above(tgt, 4.0), depth_max=5.0)
    out["icp_200k_close"] = Cloud(tgt, indexed_colors(tgt, 1), PRIMESENSE_K, _above(tgt, 1.5))
    frames = unproject_cases()
    for name in ("room_u16_rgb8_pose", "room_rgb8_pose_stride3", "odd_stride1", "hd_stride4"):
        f = frames[name]
        pts, _ = oracle_unproject(f)
        rows, cols = f.depth.shape[:2]
        out[f"unprojected_{name}"] = Cloud(pts, indexed_colors(pts), f.K, f.E, cols, rows, f.scale, f.depth_max)
    edges = _pixel_edges()
    out["pixel_edges"] = Cloud(edges, indexed_colors(edges), np.eye(3), np.eye(4), 10, 6, 1000.0, 3.0)
    h = _hostile()
    out["behind_nan_inf"] = Cloud(h, indexed_colors(h), PRIMESENSE_K, np.eye(4))
    out["behind_nan_inf_pose"] = Cloud(h, indexed_colors(h), PRIMESENSE_K,
                                       oracle.inverse_transformation(cc.look_at([0.1, -0.2, 0.3], 80.0, 5.0)))
    dup = _duplicates()
    out["duplicates"] = Cloud(dup, indexed_colors(dup), PRIMESENSE_K, np.eye(4))
    return out


def oracle_unproject(f: Frame):
    """The oracle's (points, colors) of a frame; colors is None for a depth-only frame."""
    from oracle import projection
    r = projection.unproject(f.depth, f.K, f.E, f.scale, f.depth_max, f.stride, f.color)
    return r if f.color is not None else (r, None)

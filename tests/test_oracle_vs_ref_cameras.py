"""The oracle's TSDF, range-map, ray-cast and image-pyramid functions against the reference's own CPU code
(oracle/_ref/libo3dref.so) on the camera matrix of tests/camera_cases.py: other image sizes, non-square and
off-centre intrinsics, a colour camera that differs from the depth camera, other depth scales, block resolutions
and voxel sizes.  Every comparison is bit-exact.  CPU only."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle
from tests.camera_cases import CASES, ODD_K, QVGA_K, TSDF_CASES, frames
from tests.synth import camera_pose, render_depth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libo3dref.so")
pytestmark = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref not built (needs the reference source tree)")

TRUNC, DMIN = 8.0, 0.1
ATTRS = ("depth", "vertex", "color", "normal", "index", "mask", "interp_ratio", "interp_ratio_dx", "interp_ratio_dy",
         "interp_ratio_dz")
f32p, f64p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int32)
vp = C.c_void_p


def _p(a, t):
    return a.ctypes.data_as(t)


@pytest.fixture(scope="module")
def ref():
    L = C.CDLL(REF)
    L.ref_depth_touch.restype = C.c_int64
    L.ref_depth_touch.argtypes = [vp, C.c_int, C.c_int, C.c_int, f64p, f64p, C.c_int, C.c_float, C.c_float, C.c_float,
                                  C.c_float, C.c_int, i32p, C.c_int64]
    for name in ("ref_integrate", "ref_integrate_f32_values"):
        f = getattr(L, name)
        f.restype = None
        f.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, i32p, C.c_int64, i32p, C.c_int64, f32p, vp, vp, f64p, f64p,
                      f64p, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float]
    L.ref_estimate_range.restype = C.c_int64
    L.ref_estimate_range.argtypes = [i32p, C.c_int64, f64p, f64p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                     C.c_float, C.c_float, C.c_int64, f32p]
    L.ref_ray_cast.restype = None
    L.ref_ray_cast.argtypes = [i32p, C.c_int64, f32p, vp, vp, f32p, f64p, f64p, C.c_int, C.c_int, C.c_int, C.c_float,
                               C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int] + [vp] * 10
    L.ref_clip_transform.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, f32p]
    L.ref_pyr_down_depth.argtypes = [f32p, C.c_int, C.c_int, C.c_float, C.c_float, f32p]
    L.ref_create_vertex_map.argtypes = [f32p, C.c_int, C.c_int, f64p, C.c_float, f32p]
    L.ref_create_normal_map.argtypes = [f32p, C.c_int, C.c_int, C.c_float, f32p]
    return L


def _k9(K):
    return np.ascontiguousarray(np.asarray(K, np.float64).reshape(9))


def _e16(E):
    return np.ascontiguousarray(np.asarray(E, np.float64).reshape(16))


def _sorted(k):
    k = np.asarray(k, np.int32).reshape(-1, 3)
    return k[np.lexsort((k[:, 2], k[:, 1], k[:, 0]))]


def _same(a, b):
    a, b = np.ascontiguousarray(a).reshape(-1), np.ascontiguousarray(b).reshape(-1)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and \
        np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))


@pytest.mark.parametrize("name", TSDF_CASES)
def test_depth_touch_is_the_reference_block_set(ref, name):
    """DepthTouchCPU: identical block set (image sizes that are not multiples of the stride 4 included)."""
    case = CASES[name]
    for T, E, depth, _ in frames(case):
        out = np.zeros(((case.height // 4) * (case.width // 4) * 4 + 1, 3), np.int32)
        n = ref.ref_depth_touch(depth.ctypes.data, int(case.f32), case.height, case.width, _p(_k9(case.K), f64p),
                                _p(_e16(E), f64p), case.res, case.voxel, case.voxel * TRUNC, case.scale,
                                case.depth_max, 4, _p(out, i32p), len(out))
        got = oracle.depth_touch(depth, case.K, E, case.res, case.voxel, case.voxel * TRUNC, case.scale, case.depth_max,
                                 4)
        assert n > 0 and np.array_equal(got, _sorted(out[:n]))


def _fuse(ref, case, values_f32=False):
    """The case's frames fused by the oracle and by the reference's IntegrateCPU, with the case's colour K."""
    frs = frames(case)
    r3 = case.res ** 3
    cap = sum(len(oracle.depth_touch(d, case.K, E, case.res, case.voxel, case.voxel * TRUNC, case.scale,
                                     case.depth_max, 4)) for _, E, d, _ in frs) + 16
    vt = np.float32 if values_f32 else np.uint16
    keys = np.zeros((cap, 3), np.int32)
    o = dict(tsdf=np.zeros((cap, r3), np.float32), wt=np.zeros((cap, r3), vt), col=np.zeros((cap, r3, 3), vt))
    r = {k: v.copy() for k, v in o.items()}
    size = 0
    fn = ref.ref_integrate_f32_values if values_f32 else ref.ref_integrate
    for T, E, depth, col in frs:
        want = oracle.depth_touch(depth, case.K, E, case.res, case.voxel, case.voxel * TRUNC, case.scale,
                                  case.depth_max, 4)
        bi, _, size, rc = oracle.hashmap_activate(keys, size, want)
        assert rc == 0
        oracle.tsdf_integrate(depth, col, bi, keys, o["tsdf"], o["wt"], o["col"], case.K, case.cK, E, case.res,
                              case.voxel, case.voxel * TRUNC, case.scale, case.depth_max)
        bi = np.ascontiguousarray(bi, np.int32)
        fn(depth.ctypes.data, col.ctypes.data, int(case.f32), case.height, case.width, _p(bi, i32p), len(bi),
           _p(keys, i32p), cap, _p(r["tsdf"], f32p), r["wt"].ctypes.data, r["col"].ctypes.data, _p(_k9(case.K), f64p),
           _p(_k9(case.cK), f64p), _p(_e16(E), f64p), case.res, case.voxel, case.voxel * TRUNC, case.scale,
           case.depth_max)
    return keys, size, o, r, want, frs


@pytest.mark.parametrize("name", TSDF_CASES)
def test_integrate_is_the_reference_integrate(ref, name):
    """IntegrateCPU (UInt16 weight / colour) over the case's frames: tsdf bit for bit, weights and colours equal."""
    case = CASES[name]
    _, size, o, r, _, _ = _fuse(ref, case)
    assert (o["wt"] > 0).sum() > 1000
    assert np.array_equal(o["tsdf"].view(np.uint32), r["tsdf"].view(np.uint32))
    assert np.array_equal(o["wt"], r["wt"]) and np.array_equal(o["col"], r["col"])


@pytest.mark.parametrize("name", ["odd_colour_k", "qvga_colour_k", "near", "hd_f32", "qvga_res8"])
def test_integrate_float32_value_layout_is_the_reference_integrate(ref, name):
    """IntegrateCPU in the (Float32, Float32) value layout, with the case's colour K."""
    case = CASES[name]
    _, _, o, r, _, _ = _fuse(ref, case, values_f32=True)
    assert (o["wt"] > 0).sum() > 1000
    for k in ("tsdf", "wt", "col"):
        assert np.array_equal(o[k].view(np.uint32), r[k].view(np.uint32)), k


RAY_CASES = ["qvga", "hd", "odd", "short", "near", "qvga_res8", "qvga_res32", "odd_colour_k"]


@pytest.mark.parametrize("name", RAY_CASES)
def test_range_map_and_ray_cast_are_the_reference(ref, name):
    """EstimateRangeCPU and RayCastCPU (all ten renderings) at down factors 1, 2, 4 and 8 on the case's own camera,
    on the oracle-fused volume: the range cells cut by integer division (odd sizes) and voxel indices of other
    block resolutions included."""
    case = CASES[name]
    keys, size, o, _, frustum, frs = _fuse(ref, case)
    E = frs[-1][1]
    K9, E16 = _k9(case.K), _e16(E)
    h, w = case.height, case.width
    for down in (1, 2, 4, 8):
        want = np.zeros((h // down, w // down, 2), np.float32)
        fk = np.ascontiguousarray(frustum)
        ref.ref_estimate_range(_p(fk, i32p), len(fk), _p(K9, f64p), _p(E16, f64p), h, w, down, case.res, case.voxel,
                               DMIN, case.depth_max, 1 << 20, _p(want, f32p))
        rng = oracle.estimate_range(fk, case.K, E, h, w, down, case.res, case.voxel, DMIN, case.depth_max)
        assert (want[..., 0] < want[..., 1]).mean() > 0.5
        assert np.array_equal(rng.view(np.uint32), want.view(np.uint32)), down
        got = oracle.ray_cast(keys, size, o["tsdf"], o["wt"], o["col"], rng, case.K, E, h, w, ATTRS, case.res,
                              case.voxel, case.scale, DMIN, case.depth_max, 1.0, TRUNC, down)
        exp, ptrs = {}, []
        for a in ATTRS:
            c, dt = oracle.RAYCAST_ATTRS[a]
            exp[a] = np.full((h, w, c), 77, dt)
            ptrs.append(exp[a].ctypes.data)
        # Where the image is not a multiple of the down factor, the last partial row / column of pixels has no range
        # cell (h_down = h / down): upstream indexes cell (x / down, y / down) of the [h_down, w_down] map anyway, i.e.
        # up to ((h - 1) / down) * w_down + (w - 1) / down, past its end.  It is handed a map padded with empty
        # cells up to that index, so that it only reads memory the test owns; the oracle (and the CUDA kernel) clamp
        # to the last cell instead (oracle/tsdf_oracle.c).  The images are compared where upstream is defined.
        w_down = w // down
        cells = max(((h - 1) // down) * w_down + (w - 1) // down + 1, rng.shape[0] * w_down)
        padded = np.zeros((cells, 2), np.float32)
        padded[: rng.shape[0] * w_down] = rng.reshape(-1, 2)
        ref.ref_ray_cast(_p(keys, i32p), size, _p(o["tsdf"], f32p), o["wt"].ctypes.data, o["col"].ctypes.data,
                         _p(padded, f32p), _p(K9, f64p), _p(E16, f64p), h, w, case.res, case.voxel, case.scale, DMIN,
                         case.depth_max, 1.0, TRUNC, down, *ptrs)
        assert (exp["depth"][..., 0] > 0).mean() > 0.3
        hh, ww = (h // down) * down, (w // down) * down
        for a in ATTRS:
            x, y = got[a][:hh, :ww], exp[a][:hh, :ww]
            if a == "mask":
                y = y.astype(bool)
            assert np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x,
                                  y.view(np.uint32) if y.dtype == np.float32 else y), (a, down)


@pytest.mark.parametrize("shape", [(251, 333, ODD_K, 3), (120, 160, QVGA_K / 2, 3), (240, 320, QVGA_K, 4)])
def test_image_pyramid_is_the_reference(ref, shape):
    """ClipTransform, PyrDownDepth, CreateVertexMap and CreateNormalMap through every pyramid level of odd and small
    shapes (halving 333 x 251 leaves remainders at every level)."""
    h, w, K, levels = shape
    K = np.array(K, np.float64)
    K[2, 2] = 1.0
    depth = render_depth(camera_pose(410), K=K, width=w, height=h).numpy()
    depth[h // 5: h // 5 + 7, w // 3: w // 3 + 9] = 0
    nan = float("nan")
    want = np.empty((h, w), np.float32)
    ref.ref_clip_transform(depth.ctypes.data, 0, h, w, 1000.0, 0.0, 3.0, nan, _p(want, f32p))
    d = oracle.clip_transform(depth, 1000.0, 0.0, 3.0, nan)
    assert _same(d, want) and np.isnan(d).any()
    for lv in range(levels):
        r, c = d.shape
        Kp = np.ascontiguousarray(K)
        v_want = np.empty((r, c, 3), np.float32)
        ref.ref_create_vertex_map(_p(d, f32p), r, c, _p(Kp.reshape(9), f64p), nan, _p(v_want, f32p))
        v = oracle.create_vertex_map(d, Kp)
        assert _same(v, v_want), lv
        n_want = np.empty((r, c, 3), np.float32)
        ref.ref_create_normal_map(_p(v_want, f32p), r, c, nan, _p(n_want, f32p))
        assert _same(oracle.create_normal_map(v), n_want), lv
        if lv + 1 < levels:
            d_want = np.empty((r // 2, c // 2), np.float32)
            ref.ref_pyr_down_depth(_p(d, f32p), r, c, 0.14, nan, _p(d_want, f32p))
            d = oracle.pyr_down_depth(d, 0.14)
            assert _same(d, d_want) and np.isfinite(d).mean() > 0.8, lv
            K = K / 2
            K[2, 2] = 1.0

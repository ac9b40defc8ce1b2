"""TSDF fusion, ray casting and RGB-D odometry on cameras and image shapes other than the 640x480 PrimeSense frame
(tests/camera_cases.py): CUDA against the CPU oracle, bit for bit where the other GPU tests are, and each case asserts
on the host the condition that sends it down the kernel path it names."""
import itertools

import numpy as np
import pytest
import torch

import oracle
from tests.camera_cases import (CASES, ODD_K, QVGA_K, REJECTED_SCALE, TSDF_CASES, Case, fast_scale_failures,
                                fast_scale_ok, frames, look_at, scaled_k, tensor_map_possible, unit_rectangles)
from tests.synth import PRIMESENSE_K, camera_pose, render_depth

pytestmark = pytest.mark.gpu

TRUNC, DMIN = 8.0, 0.1
ALL_ATTRS = ("depth", "vertex", "color", "normal", "index", "mask", "interp_ratio", "interp_ratio_dx",
             "interp_ratio_dy", "interp_ratio_dz")


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


def _sorted_keys(k):
    k = np.asarray(k, np.int32).reshape(-1, 3)
    return k[np.lexsort((k[:, 2], k[:, 1], k[:, 0]))]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _misaligned(t):
    """A device copy of `t` as a view into a larger buffer, with data_ptr() % 16 == 2."""
    flat = t.reshape(-1)
    per = 2 // t.element_size()
    big = torch.zeros(flat.numel() + 16 * max(per, 1), dtype=t.dtype, device="cuda")
    off = next(o for o in range(16) if (big.data_ptr() + o * t.element_size()) % 16 == 2)
    v = big[off: off + flat.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == 2 and v.is_contiguous()
    return v


def _device_images(case, depth, col):
    d, c = torch.from_numpy(depth).cuda(), torch.from_numpy(col).cuda()
    if case.misaligned:
        d, c = _misaligned(d), _misaligned(c)
    return d, c


class OracleVolume:
    def __init__(self, case, cap, color=True, values_f32=False):
        r3 = case.res ** 3
        vt = np.float32 if values_f32 else np.uint16
        self.case, self.size = case, 0
        self.keys = np.zeros((cap, 3), np.int32)
        self.tsdf = np.zeros((cap, r3), np.float32)
        self.wt = np.zeros((cap, r3), vt)
        self.col = np.zeros((cap, r3, 3), vt) if color else None

    def integrate(self, depth, col, E, want=None, scale=None, depth_max=None, cK=None):
        c = self.case
        scale = c.scale if scale is None else scale
        depth_max = c.depth_max if depth_max is None else depth_max
        if want is None:
            want = oracle.depth_touch(depth, c.K, E, c.res, c.voxel, c.voxel * TRUNC, scale, depth_max, 4)
        bi, _, self.size, rc = oracle.hashmap_activate(self.keys, self.size, want)
        assert rc == 0
        oracle.tsdf_integrate(depth, col if self.col is not None else None, bi, self.keys, self.tsdf, self.wt, self.col,
                              c.K, c.cK if cK is None else cK, E, c.res, c.voxel, c.voxel * TRUNC, scale, depth_max)
        return want


def _compare(case, okeys, otsdf, owt, ocol, osize, gkeys, gtsdf, gwt, gcol):
    """Same block set; TSDF bit for bit; weights and colours equal (aligned by block key)."""
    r3 = case.res ** 3
    gkeys = np.asarray(gkeys)[:osize]
    assert np.array_equal(_sorted_keys(gkeys), _sorted_keys(okeys[:osize]))
    lut = {tuple(k): i for i, k in enumerate(okeys[:osize].tolist())}
    perm = np.array([lut[tuple(k)] for k in gkeys.tolist()])
    gt = np.asarray(gtsdf).reshape(-1, r3)[:osize]
    gw = np.asarray(gwt).reshape(-1, r3)[:osize]
    assert np.array_equal(_bits(gw), _bits(owt[perm]))
    assert np.array_equal(gt.view(np.uint32), otsdf[perm].view(np.uint32))
    if ocol is not None:
        gc = np.asarray(gcol).reshape(-1, r3, 3)[:osize]
        assert np.array_equal(_bits(gc), _bits(ocol[perm]))
    return int((gw > 0).sum())


def _compare_vbg(case, vbg, ov):
    hm = vbg.hashmap()
    assert hm.size() == ov.size
    return _compare(case, ov.keys, ov.tsdf, ov.wt, ov.col, ov.size, hm.key_tensor().cpu().numpy(),
                    vbg.attribute("tsdf").cpu().numpy(), vbg.attribute("weight").cpu().numpy(),
                    vbg.attribute("color").cpu().numpy() if ov.col is not None else None)


def _assert_path(case, depth_dev, want_keys, E):
    """The host-side condition that sends the case down the path it names."""
    es = 4 if case.f32 else 2
    tiled = tensor_map_possible(depth_dev.data_ptr(), case.height, case.width, es)
    if case.name in ("odd", "odd_colour_k", "short", "misaligned"):
        assert not tiled
    elif case.res == 16:
        assert tiled
    if case.res != 16:
        assert case.res in (4, 8, 32)                      # integrate_kernel, not integrate16_kernel
    if case.name in ("near", "touching") and case.res == 16:
        n, behind, oversize = unit_rectangles(want_keys, case.K, E, case.voxel, es)
        if case.name == "near":
            assert oversize > 0.05 * n, (n, behind, oversize)
        else:
            assert behind > 0, (n, behind, oversize)
    if case.color_K is not None:
        assert not np.array_equal(case.color_K, case.K)    # same_k = 0
    if not case.f32:
        assert fast_scale_ok(case.scale)                   # fast_scale = 1


def _cap(case, frs):
    return sum(len(oracle.depth_touch(d, case.K, E, case.res, case.voxel, case.voxel * TRUNC, case.scale,
                                      case.depth_max, 4)) for _, E, d, _ in frs) + 64


_FUSED = {}


def _fused(o3d, name):
    """The case's frames fused by VoxelBlockGrid.integrate_frame (CUDA) and by the oracle; cached per case."""
    if name in _FUSED:
        return _FUSED[name]
    case = CASES[name]
    frs = frames(case)
    cap = _cap(case, frs)
    vbg = o3d.t.geometry.VoxelBlockGrid(voxel_size=case.voxel, block_resolution=case.res, block_count=cap)
    ov = OracleVolume(case, cap)
    want = None
    for T, E, depth, col in frs:
        d, c = _device_images(case, depth, col)
        want = ov.integrate(depth, col, E, cK=case.K)     # the fused path has one camera
        _assert_path(case, d, want, E)
        vbg.integrate_frame(d, c, case.K, E, case.scale, case.depth_max, TRUNC)
        got = vbg.last_frustum_block_coordinates().cpu().numpy()
        assert np.array_equal(_sorted_keys(got), want)     # slam::Model::frustum_block_coords_
        torch.cuda.synchronize()
    _FUSED[name] = (vbg, ov, want, frs)
    return _FUSED[name]


FUSED_CASES = [n for n in TSDF_CASES if CASES[n].color_K is None]


@pytest.mark.parametrize("name", FUSED_CASES)
def test_fused_integrate_vs_oracle(o3d, name):
    vbg, ov, _, _ = _fused(o3d, name)
    updated = _compare_vbg(CASES[name], vbg, ov)
    assert updated > 1000


@pytest.mark.parametrize("name", TSDF_CASES)
def test_unfused_integrate_with_colour_intrinsics_vs_oracle(o3d, name):
    """compute_unique_block_coordinates + integrate with the case's colour K (distinct from the depth K for the
    *_colour_k cases: the fast kernel's general colour projection)."""
    case = CASES[name]
    frs = frames(case)
    cap = _cap(case, frs)
    vbg = o3d.t.geometry.VoxelBlockGrid(voxel_size=case.voxel, block_resolution=case.res, block_count=cap)
    ov = OracleVolume(case, cap)
    for T, E, depth, col in frs:
        d, c = _device_images(case, depth, col)
        bc = vbg.compute_unique_block_coordinates(d, case.K, E, case.scale, case.depth_max, TRUNC)
        want = ov.integrate(depth, col, E)
        assert np.array_equal(_sorted_keys(bc.cpu().numpy()), want)
        _assert_path(case, d, want, E)
        vbg.integrate(bc, d, c, case.K, case.cK, E, case.scale, case.depth_max, TRUNC)
    updated = _compare_vbg(case, vbg, ov)
    assert updated > 1000
    if case.color_K is not None:
        # the colour camera moved the lookups: the volume differs from one fused with the depth K
        ov2 = OracleVolume(case, cap)
        for T, E, depth, col in frs:
            ov2.integrate(depth, col, E, cK=case.K)
        assert not np.array_equal(ov2.col[: ov2.size], ov.col[: ov.size])


def test_rejected_depth_scale_falls_back_to_the_division(o3d):
    """A scale that verify_fast_scale rejects: 1 / 1e-35 makes d * y overflow for every numerator above 3402, and the
    division-free sequence returns NaN where d / s is +inf.  NaN would pass the depth_max test and be integrated as a
    full truncation distance; the reference's inf is rejected.  The blocks come from the same frame at scale 1000
    (depth_max 6 m), so that they hold voxels that read those pixels: nothing may be integrated, exactly as the
    oracle integrates nothing."""
    from open3d_b200 import _lib as L
    bad = fast_scale_failures(REJECTED_SCALE)
    assert not fast_scale_ok(REJECTED_SCALE) and len(bad) > 60000 and fast_scale_ok(1000.0) and fast_scale_ok(5000.0)
    # looking down the room's long axis: walls and floor up to 8 m away
    case = Case("qvga_rejected_scale", "fast_scale = 0", 320, 240, QVGA_K, (look_at([-2.4, 0.3, 1.4], 5.0, 8.0),),
                render_max=8.0)
    (T, E, depth, col), = frames(case)
    assert np.isin(depth, bad).sum() > 5000                  # the image holds those numerators
    want = oracle.depth_touch(depth, case.K, E, 16, case.voxel, case.voxel * TRUNC, 1000.0, 8.0, 4)
    vbg = o3d.t.geometry.VoxelBlockGrid(voxel_size=case.voxel, block_resolution=16, block_count=len(want) + 16)
    d, c = torch.from_numpy(depth).cuda(), torch.from_numpy(col).cuda()
    assert tensor_map_possible(d.data_ptr(), 240, 320, 2)
    vbg.integrate(torch.from_numpy(want).cuda(), d, c, case.K, case.K, E, REJECTED_SCALE, 3.0, TRUNC)
    ov = OracleVolume(case, len(want) + 16)
    ov.integrate(depth, col, E, want=want, scale=REJECTED_SCALE, depth_max=3.0)
    # voxels that read a rejected numerator: those the frame integrates at scale 1000 when every other pixel is 0
    probe = OracleVolume(case, len(want) + 16)
    probe.integrate(np.where(np.isin(depth, bad), depth, 0).astype(np.uint16), col, E, want=want, scale=1000.0,
                    depth_max=8.0)
    assert (probe.wt > 0).sum() > 10000
    assert not ov.wt.any()                                   # the reference integrates nothing
    _compare_vbg(case, vbg, ov)
    # the stateless entry point keeps its own record of the last checked scale
    keys = torch.from_numpy(np.ascontiguousarray(ov.keys[: ov.size])).cuda()
    idx = torch.arange(ov.size, dtype=torch.int32, device="cuda")
    tsdf = torch.zeros((ov.size, 4096), dtype=torch.float32, device="cuda")
    wt = torch.zeros((ov.size, 4096), dtype=torch.uint16, device="cuda")
    K9, E16 = np.ascontiguousarray(case.K), np.ascontiguousarray(E)
    for scale in (1000.0, REJECTED_SCALE):
        L.check(L.lib.o3db_integrate_blocks(d.data_ptr(), L.DEPTH_U16, None, 0, 240, 320, idx.data_ptr(), ov.size,
                                            keys.data_ptr(), tsdf.data_ptr(), wt.data_ptr(), None, 0, L.dptr(K9),
                                            L.dptr(K9), L.dptr(E16), 16, case.voxel, case.voxel * TRUNC, scale, 3.0, 0))
        if scale == 1000.0:
            torch.cuda.synchronize()
            w1 = wt.clone()
    torch.cuda.synchronize()
    assert bool(w1.int().any()) and torch.equal(wt.int(), w1.int())                  # the second call added nothing


@pytest.mark.parametrize("name,layout", [("odd", 0), ("odd", 1), ("near", 0), ("near", 1), ("odd_colour_k", 0),
                                         ("odd_colour_k", 1), ("hd_f32", 0), ("hd_f32", 1)])
def test_stateless_integrate_blocks_vs_oracle(o3d, name, layout):
    """o3db_integrate_blocks (the forwarders' entry point, the reference's hash map and buffers) in both value
    layouts: UInt16 weight / colour (integrate16_kernel) and Float32 (integrate_kernel)."""
    from open3d_b200 import _lib as L
    case = CASES[name]
    frs = frames(case)
    cap = _cap(case, frs)
    f32v = layout == 1
    ov = OracleVolume(case, cap, values_f32=f32v)
    vt = torch.float32 if f32v else torch.uint16
    r3 = case.res ** 3
    tsdf = torch.zeros((cap, r3), dtype=torch.float32, device="cuda")
    wt = torch.zeros((cap, r3), dtype=vt, device="cuda")
    col = torch.zeros((cap, r3, 3), dtype=vt, device="cuda")
    keys = torch.zeros((cap, 3), dtype=torch.int32, device="cuda")
    dK, cK = np.ascontiguousarray(case.K), np.ascontiguousarray(case.cK)
    for T, E, depth, c in frs:
        d, cd = _device_images(case, depth, c)
        want = oracle.depth_touch(depth, case.K, E, case.res, case.voxel, case.voxel * TRUNC, case.scale,
                                  case.depth_max, 4)
        _assert_path(case, d, want, E)
        ov.integrate(depth, c, E, want=want)
        bi, _, _, _ = oracle.hashmap_activate(ov.keys.copy(), ov.size, want)   # the slots of the now active keys
        keys.copy_(torch.from_numpy(ov.keys))
        idx = torch.from_numpy(np.ascontiguousarray(bi, np.int32)).cuda()
        E16 = np.ascontiguousarray(E)
        L.check(L.lib.o3db_integrate_blocks(d.data_ptr(), L.DEPTH_F32 if case.f32 else L.DEPTH_U16, cd.data_ptr(),
                                            L.COLOR_F32 if case.f32 else L.COLOR_U8, case.height, case.width,
                                            idx.data_ptr(), len(bi), keys.data_ptr(), tsdf.data_ptr(), wt.data_ptr(),
                                            col.data_ptr(), layout, L.dptr(dK), L.dptr(cK), L.dptr(E16), case.res,
                                            case.voxel, case.voxel * TRUNC, case.scale, case.depth_max, 0))
    torch.cuda.synchronize()
    n = ov.size
    _compare(case, ov.keys, ov.tsdf, ov.wt, ov.col, n, ov.keys, tsdf.cpu().numpy(), wt.cpu().numpy(),
             col.cpu().numpy())
    assert (ov.wt > 0).sum() > 1000


@pytest.mark.parametrize("host", [False, True])
def test_frame_size_changes_on_one_handle(o3d, host):
    """320x240 -> 640x480 -> 1024x768 -> 320x240 through ONE handle (K scaled with the image): the fused path's
    frustum lists and the host entry point's staging buffers are reallocated when a larger frame arrives, and must
    not be when a smaller one follows."""
    voxel, res = 0.008, 16
    seq = [(320, 240, 0.5, 0), (640, 480, 1.0, 4), (1024, 768, 1.6, 8), (320, 240, 0.5, 12)]
    vbg = o3d.t.geometry.VoxelBlockGrid(voxel_size=voxel, block_resolution=res, block_count=2000)
    case = Case("sizes", "reallocation", 0, 0, PRIMESENSE_K, ())
    ov = OracleVolume(case, 20000)
    for w, h, f, fid in seq:
        K = scaled_k(PRIMESENSE_K, f)
        T = camera_pose(fid)
        E = oracle.inverse_transformation(T)
        depth, col = render_depth(T, K=K, width=w, height=h, with_color=True)
        depth, col = depth.numpy(), col.numpy()
        if host:
            vbg.integrate_frame(torch.from_numpy(depth), torch.from_numpy(col), K, E, 1000.0, 3.0, TRUNC)
        else:
            vbg.integrate_frame(torch.from_numpy(depth).cuda(), torch.from_numpy(col).cuda(), K, E, 1000.0, 3.0, TRUNC)
        c2 = Case("sizes", "", w, h, K, ())
        ov.case = c2
        want = ov.integrate(depth, col, E)
        got = vbg.last_frustum_block_coordinates().cpu().numpy()
        assert np.array_equal(_sorted_keys(got), want)
    _compare_vbg(case, vbg, ov)


# ------------------------------------------------------------------------------------------------ ray cast

RAY_CASES = [n for n in FUSED_CASES if CASES[n].res in (8, 16, 32) and not CASES[n].f32] + ["hd_f32"]


@pytest.mark.parametrize("name", RAY_CASES)
def test_ray_cast_all_attributes_vs_oracle(o3d, name):
    """All ten renderings at down factors 1, 2, 4 and 8, from the case's last camera and from a pose moved by a few
    centimetres and degrees, on the fused volume: bit for bit."""
    case = CASES[name]
    vbg, ov, frustum, frs = _fused(o3d, name)
    T_last = frs[-1][0]
    moved = T_last.copy()
    moved[:3, 3] += (0.02, -0.015, 0.01)
    moved[:3, :3] = moved[:3, :3] @ np.array(
        [[np.cos(0.03), 0, np.sin(0.03)], [0, 1, 0], [-np.sin(0.03), 0, np.cos(0.03)]])
    r3 = case.res ** 3
    gkeys = vbg.hashmap().key_tensor()[: ov.size].contiguous()
    gk = gkeys.cpu().numpy()
    scale = case.scale
    dmin = 0.02 if name == "touching" else DMIN             # the wall is 6 cm away
    min_hit = 0.05 if name in ("near", "touching") else 0.2
    for T in (T_last, moved):
        E = oracle.inverse_transformation(T)
        for down in (1, 2, 4, 8):
            res = vbg.ray_cast(gkeys, case.K, E, case.width, case.height, ALL_ATTRS, scale, dmin, case.depth_max, 1.0,
                               TRUNC, down)
            rng = oracle.estimate_range(gk, case.K, E, case.height, case.width, down, case.res, case.voxel, dmin,
                                        case.depth_max)
            assert np.array_equal(_bits(res["range"].cpu().numpy()), _bits(rng)), down
            ref = oracle.ray_cast(ov.keys, ov.size, ov.tsdf, ov.wt, ov.col, rng, case.K, E, case.height, case.width,
                                  ALL_ATTRS, case.res, case.voxel, scale, dmin, case.depth_max, 1.0, TRUNC, down)
            hit = ref["depth"][..., 0] > 0
            assert hit.mean() > min_hit, (down, hit.mean())
            for attr in ALL_ATTRS:
                if attr in ("index", "mask"):
                    continue
                assert np.array_equal(_bits(res[attr].cpu().numpy()), _bits(ref[attr])), (attr, down)
            gmask = res["mask"].cpu().numpy()
            assert np.array_equal(gmask, ref["mask"])
            gi, oi = res["index"].cpu().numpy(), ref["index"]
            assert np.array_equal(gk[gi[gmask] // r3], ov.keys[oi[gmask] // r3]) and \
                np.array_equal(gi[gmask] % r3, oi[gmask] % r3)
            assert not gi[~gmask].any()
    # the frustum of the last fused frame taken on the device (block_coords=None)
    E = oracle.inverse_transformation(T_last)
    got = vbg.ray_cast(None, case.K, E, case.width, case.height, ("depth",), scale, DMIN, case.depth_max, 1.0, TRUNC,
                       4)["range"]
    want = oracle.estimate_range(frustum, case.K, E, case.height, case.width, 4, case.res, case.voxel, DMIN,
                                 case.depth_max)
    assert np.array_equal(_bits(got.cpu().numpy()), _bits(want))


# ------------------------------------------------------------------------------------------------ odometry

def _cluster_size():
    """What the odometry host code's cluster choice can be: 16 CTAs, else 8 (unknown before the device answers)."""
    return (16, 8)


def _kernel_launches(level_pixels, its):
    """Launches of o3db_rgbd_odometry_multi_scale_point_to_plane, worked out from its host code: one clip launch for
    both frames, one pyramid launch per level, then per level either ONE odometry_level_kernel launch (cluster
    resident: max_iteration >= 2 and at most cluster x 512 x 12 pixels) or max_iteration odometry_iteration_kernel
    launches.  Returns, per level, the set of launch counts the rule allows over both possible cluster sizes, and for
    each level which kernel that count means."""
    per_level = []
    for px, it in zip(level_pixels, its):
        options = set()
        for cl in _cluster_size():
            options.add(1 if (it >= 2 and px <= cl * 512 * 12) else it)
        per_level.append(options)
    return per_level


def _pyramid_maps(o3d, depth_src, depth_tgt, K, levels):
    """The GPU maps at every level from the stand-alone image kernels (the fused pyramid kernel runs the same device
    functions in the same order): [(sv, tv, tn, K)] fine to coarse."""
    Image = o3d.t.geometry.Image
    NAN = float("nan")
    ds = Image(torch.from_numpy(depth_src).cuda()).clip_transform(1000.0, 0.0, 3.0, NAN)
    dt = Image(torch.from_numpy(depth_tgt).cuda()).clip_transform(1000.0, 0.0, 3.0, NAN)
    K = np.array(K, np.float64)
    out = []
    for lv in range(levels):
        if lv:
            ds, dt = ds.pyr_down_depth(0.14, NAN), dt.pyr_down_depth(0.14, NAN)
            K = K / 2
            K[2, 2] = 1
        sv = ds.create_vertex_map(K, NAN).as_tensor()
        tv = dt.create_vertex_map(K, NAN).as_tensor()
        tn = dt.filter_bilateral(5, 5.0, 10.0).create_vertex_map(K, NAN).create_normal_map(NAN).as_tensor()
        out.append((sv, tv, tn, K.copy()))
    return out


ODO_CASES = {
    # name: (width, height, K, criteria coarse -> fine, expected kernel fine -> coarse or None = either,
    #        finest level's max_iteration in the `single` variant)
    "xga": (1024, 768, scaled_k(PRIMESENSE_K, 1.6), (4, 3, 2), ("iter", "iter", "cluster"), 2),
    # 1 + 1 + 5 steps on this pair leave the final pose 2e-4 from the oracle's: from the fourth step on the inlier
    # counts differ by one or two pixels (f32 sums against the oracle's f64 ones), and the following steps amplify
    # that.  One step on the finest level stays within the trajectory tolerance.
    "odd": (333, 251, ODD_K, (4, 3, 5), (None, "cluster", "cluster"), 1),
    "qqvga_1level": (160, 120, scaled_k(PRIMESENSE_K, 0.25), (4,), ("cluster",), 4),
    "vga_5levels": (640, 480, PRIMESENSE_K, (3, 3, 3, 3, 2), ("iter", None, "cluster", "cluster", "cluster"), 2),
}


@pytest.mark.parametrize("name,single", [(n, s) for n in ODO_CASES for s in (False, True)
                                         if not (s and len(ODO_CASES[n][3]) == 1)])
def test_rgbd_odometry_kernel_choice_vs_oracle(o3d, name, single):
    """RGBDOdometryMultiScale (PointToPlane) at other image sizes and level counts.  `single`: max_iteration = 1 on
    every level but the finest, which forces the per-iteration kernel there; its first step is then checked bit for
    bit against compute_odometry_result_point_to_plane (the same kernel, stand-alone) on the same maps."""
    from open3d_b200 import _lib as L
    odo, geo = o3d.t.pipelines.odometry, o3d.t.geometry
    w, h, K, crit, kinds, single_finest = ODO_CASES[name]
    crit = list(crit)
    if single:
        crit = [1] * (len(crit) - 1) + [single_finest]
    levels = len(crit)
    Ta, Tb = camera_pose(200), camera_pose(203)
    da = render_depth(Ta, K=K, width=w, height=h).numpy()
    db = render_depth(Tb, K=K, width=w, height=h).numpy()
    da[h // 10: h // 10 + h // 20, w // 6: w // 6 + w // 16] = 0
    # level sizes fine -> coarse, as the host code halves them
    sizes = [(h >> i, w >> i) for i in range(levels)]
    pixels = [r * c for r, c in sizes]
    its = list(reversed(crit))                                 # fine -> coarse
    allowed = _kernel_launches(pixels, its)
    for kind, px, it, opts in zip(kinds, pixels, its, allowed):
        if single and it == 1:
            assert opts == {1}                                 # per-iteration kernel, one launch
        elif kind == "cluster":
            assert opts == {1} and it >= 2 and px <= 8 * 512 * 12
        elif kind == "iter":
            assert opts == {it} and px > 16 * 512 * 12
        else:
            assert 8 * 512 * 12 < px <= 16 * 512 * 12          # depends on the cluster size the device allows
    src = geo.RGBDImage(None, torch.from_numpy(db).cuda())
    tgt = geo.RGBDImage(None, torch.from_numpy(da).cuda())
    C_ = odo.OdometryConvergenceCriteria
    n0 = L.launch_count()
    res, log = odo.rgbd_odometry_multi_scale(src, tgt, K, np.eye(4), 1000.0, 3.0, [C_(c, 0.0, 0.0) for c in crit],
                                             odo.Method.PointToPlane, odo.OdometryLossParams(), return_log=True)
    launches = L.launch_count() - n0
    possible = {1 + levels + sum(choice) for choice in itertools.product(*allowed)}
    assert launches in possible, (launches, possible)
    ref = oracle.rgbd_odometry_multi_scale_p2plane(db, da, K, criteria=[(c, 0.0, 0.0) for c in crit])
    assert ref["status"] == 0
    assert len(log) == len(ref["per_iteration"]) == sum(crit)
    # the coarsest level's first step sees identical inputs: the same inlier count, rmse to 1e-5
    assert log[0, 1] == ref["per_iteration"][0, 1]
    np.testing.assert_allclose(log[0, 0], ref["per_iteration"][0, 0], rtol=1e-5)
    np.testing.assert_allclose(log[:, 1], ref["per_iteration"][:, 1], atol=2e-4)
    np.testing.assert_allclose(log[:, 0], ref["per_iteration"][:, 0], rtol=2e-3, atol=1e-9)
    np.testing.assert_allclose(res.transformation, ref["transformation"], atol=2e-5)
    assert abs(res.fitness - ref["fitness"]) < 2e-4
    if single and levels > 1:
        # One step on the coarsest level and none elsewhere: max_iteration = 1 keeps that level on the per-iteration
        # kernel, so the result is the stand-alone step (the same kernel, the same grid) on the same maps, bit for bit.
        # The cluster kernel adds the same terms in another association; its f32 sums, and so the pose, differ.
        sv, tv, tn, Kc = _pyramid_maps(o3d, db, da, K, levels)[-1]
        one = odo.compute_odometry_result_point_to_plane(sv, tv, tn, Kc, np.eye(4), 0.07, 0.05)
        n0 = L.launch_count()
        res1, log1 = odo.rgbd_odometry_multi_scale(src, tgt, K, np.eye(4), 1000.0, 3.0,
                                                   [C_(1, 0.0, 0.0)] + [C_(0, 0.0, 0.0)] * (levels - 1),
                                                   odo.Method.PointToPlane, odo.OdometryLossParams(), return_log=True)
        assert L.launch_count() - n0 == 1 + levels + 1
        assert len(log1) == 1 and log1[0, 1] == log[0, 1] and log1[0, 0] == log[0, 0]
        assert one.fitness == log1[0, 1] and one.inlier_rmse == log1[0, 0]
        assert np.array_equal(res1.transformation, one.transformation)


def test_compute_odometry_result_on_the_odd_shape_vs_oracle(o3d):
    """One Gauss-Newton step on oracle maps of the 333x251 shape (and its 166x125 level): the 29 sums within 1e-5 of
    the oracle's f64 sums, the same inlier set, delta, rmse and fitness."""
    odo = o3d.t.pipelines.odometry
    Ta, Tb = camera_pose(300), camera_pose(303)
    da = render_depth(Ta, K=ODD_K, width=333, height=251).numpy()
    db = render_depth(Tb, K=ODD_K, width=333, height=251).numpy()
    T = np.linalg.inv(Ta) @ Tb
    T[:3, 3] += (0.01, -0.02, 0.015)
    ds, dt = oracle.clip_transform(db), oracle.clip_transform(da)
    K = np.array(ODD_K, np.float64)
    for level in range(2):
        if level:
            ds, dt = oracle.pyr_down_depth(ds, 0.14), oracle.pyr_down_depth(dt, 0.14)
            K = K / 2
            K[2, 2] = 1
        sv, tv = oracle.create_vertex_map(ds, K), oracle.create_vertex_map(dt, K)
        tn = oracle.create_normal_map(oracle.create_vertex_map(oracle.filter_bilateral(dt), K))
        res = odo.compute_odometry_result_point_to_plane(torch.from_numpy(sv).cuda(), torch.from_numpy(tv).cuda(),
                                                         torch.from_numpy(tn).cuda(), K, T, 0.07, 0.05)
        o = oracle.odometry_p2plane_sums(sv, tv, tn, K, T, 0.07, 0.05)
        assert res.sums29[28] == o["sums64"][28] > 0.3 * sv.shape[0] * sv.shape[1]
        err = np.abs(res.sums29 - o["sums64"])
        assert (err <= 1e-5 * o["abs64"] + 1e-300).all(), (err / (o["abs64"] + 1e-300)).max()
        rc, dT, rmse, fit = oracle.compute_odometry_result_p2plane(sv, tv, tn, K, T, 0.07, 0.05)
        assert rc == 0 and res.fitness == fit
        np.testing.assert_allclose(res.transformation, dT, atol=2e-6)
        np.testing.assert_allclose(res.inlier_rmse, rmse, rtol=1e-5)

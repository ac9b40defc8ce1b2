"""registration.compute_fpfh_feature and correspondences_from_features on the H100, bit for bit against the CPU oracle
(oracle/fpfh): every feature and every correspondence.  Lists: the wide KNN walk against brute force, and against the
public hybrid search for max_nn <= 32."""
import numpy as np
import pytest
import torch

import open3d_b200 as o3d
from oracle import fpfh as of
from tests import fpfh_cases as fc

pytestmark = pytest.mark.gpu
reg = o3d.t.pipelines.registration
CASES = fc.cases()


def _cloud(pts, nrm):
    return o3d.t.geometry.PointCloud(pts).set_point_normals(nrm)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


@pytest.mark.parametrize("name", sorted(CASES))
def test_fpfh_equals_oracle(name):
    pts, nrm, radius, max_nn = CASES[name]
    got = reg.compute_fpfh_feature(_cloud(pts, nrm), max_nn=max_nn, radius=radius)
    assert got.dtype == torch.float32 and tuple(got.shape) == (len(pts), 33) and got.is_cuda
    want = of.compute_fpfh_feature(pts, nrm, max_nn, radius)
    assert np.array_equal(_bits(got.cpu().numpy()), _bits(want))
    if name == "clusters":
        assert (np.abs(want[-80:]).sum(1) == 0).all()   # the isolated points: no neighbour but themselves
    sel = np.random.default_rng(5).integers(0, len(pts), 200)
    rows = reg.compute_fpfh_feature(_cloud(pts, nrm), max_nn=max_nn, radius=radius, indices=torch.from_numpy(sel))
    assert np.array_equal(_bits(rows.cpu().numpy()), _bits(want[np.unique(sel)]))


# On scan(3000, 36) the capped lists hold 4..17 points at radius 0.04, 22..84 at 0.1 (slots 0..2 of the wide list)
# and 47..128 at 0.15, where max_nn 80 / 100 / 128 cut most of them.
RADII = (None, 0.04, 0.1, 0.15)
MAX_NN = (4, 30, 64, 65, 80, 96, 100, 128)


@pytest.mark.parametrize("max_nn", MAX_NN)
def test_fpfh_max_nn(max_nn):
    pts, nrm = fc.scan(3000, 36)
    for radius in RADII:
        got = reg.compute_fpfh_feature(_cloud(pts, nrm), max_nn=max_nn, radius=radius)
        assert np.array_equal(_bits(got.cpu().numpy()), _bits(of.compute_fpfh_feature(pts, nrm, max_nn, radius)))


def _knn_index(p):
    from open3d_b200 import _lib as L
    import ctypes as C
    h = C.c_void_p()
    L.check(L.lib.o3db_knn_create(p.data_ptr(), int(p.shape[0]), None, C.byref(h)))
    return h


def _wide_lists(h, p, k, radius):
    from open3d_b200 import _lib as L
    kp = min(k, int(p.shape[0]))
    idx = torch.empty((p.shape[0], kp), dtype=torch.int32, device="cuda")
    d2 = torch.empty((p.shape[0], kp), dtype=torch.float32, device="cuda")
    cnt = torch.empty((p.shape[0],), dtype=torch.int32, device="cuda")
    L.check(L.lib.o3db_knn_search_lists(h, p.data_ptr(), int(p.shape[0]), k, 0.0 if radius is None else radius,
                                        idx.data_ptr(), d2.data_ptr(), cnt.data_ptr(), None))
    torch.cuda.synchronize()
    return idx.cpu().numpy(), d2.cpu().numpy(), cnt.cpu().numpy()


@pytest.mark.parametrize("k", [1, 8, 31, 32, 33, 63, 64, 65, 80, 96, 97, 100, 127, 128])
def test_wide_lists_equal_brute_force(k):
    """The wide list itself, in every slot configuration (k' - 1) // 32 = 0..3, uncapped and capped, against the oracle's
    brute-force lists; at radius 0.15 most capped lists reach k and are cut there."""
    from open3d_b200 import _lib as L
    pts, _ = fc.scan(3000, 36)
    p = torch.from_numpy(pts).cuda()
    h = _knn_index(p)
    try:
        for radius in RADII:
            idx, d2, cnt = _wide_lists(h, p, k, radius)
            widx, wd2, wcnt = of.lists(pts, k, radius)
            assert np.array_equal(cnt, wcnt) and np.array_equal(idx, widx), (k, radius)
            assert np.array_equal(_bits(d2), _bits(wd2)), (k, radius)
        _, _, cnt = _wide_lists(h, p, k, 0.15)
        assert (cnt == k).sum() > 0.5 * len(pts)
        bad = p.clone()
        bad[11, 2] = float("nan")
        with pytest.raises(RuntimeError, match="non-finite"):
            _wide_lists(h, bad, k, 0.1)
    finally:
        L.lib.o3db_knn_destroy(h)


def test_wide_lists_equal_hybrid_and_knn_search():
    """For k <= 32 the wide list equals the public hybrid search (radius > 0) and the public KNN search (no cap), bit
    for bit."""
    from open3d_b200 import _lib as L
    import ctypes as C
    pts, _ = fc.scan(6000, 38)
    p = torch.from_numpy(pts).cuda()
    h = _knn_index(p)
    try:
        for radius, k in ((0.03, 30), (0.03, 32), (0.05, 8), (0.08, 32), (None, 32), (None, 5)):
            idx, d2, cnt = _wide_lists(h, p, k, radius)
            hi = torch.empty((len(pts), k), dtype=torch.int32, device="cuda")
            hd = torch.empty((len(pts), k), dtype=torch.float32, device="cuda")
            if radius is None:
                L.check(L.lib.o3db_knn_search(h, p.data_ptr(), len(pts), k, L.INDEX_INT32, hi.data_ptr(),
                                              hd.data_ptr(), None))
                torch.cuda.synchronize()
                assert (cnt == k).all()
            else:
                nns = C.c_void_p()
                L.check(L.lib.o3db_nns_create(p.data_ptr(), len(pts), radius, None, C.byref(nns)))
                hc = torch.empty((len(pts),), dtype=torch.int32, device="cuda")
                L.check(L.lib.o3db_nns_hybrid_search(nns, p.data_ptr(), len(pts), radius, k, hi.data_ptr(),
                                                     hd.data_ptr(), hc.data_ptr(), None))
                torch.cuda.synchronize()
                L.lib.o3db_nns_destroy(nns)
                assert np.array_equal(hc.cpu().numpy(), cnt)
            assert np.array_equal(hi.cpu().numpy(), idx), (radius, k)
            assert np.array_equal(_bits(hd.cpu().numpy()), _bits(d2)), (radius, k)
    finally:
        L.lib.o3db_knn_destroy(h)


def test_fpfh_2m():
    """The 2 M-point scan (0.02 spacing) at radius 5 x spacing = 0.1, the recommended hybrid call, where lists hold about
    78 points: max_nn 100 keeps them whole, max_nn 30 cuts them."""
    pts, nrm = fc.scan_2m()
    cloud = _cloud(pts, nrm)
    sel = np.unique(np.random.default_rng(6).integers(0, len(pts), 40))
    for max_nn in (30, 100):
        full = reg.compute_fpfh_feature(cloud, max_nn=max_nn, radius=0.1)
        rows = reg.compute_fpfh_feature(cloud, max_nn=max_nn, radius=0.1, indices=torch.from_numpy(sel))
        assert np.array_equal(_bits(rows.cpu().numpy()), _bits(full[torch.from_numpy(sel).cuda()].cpu().numpy()))
        # the oracle on a sub-cloud: brute-force lists (over all 2 M points) of the selected points and their
        # neighbours, whose SPFH rows the selected rows read, plus the points those lists name
        idx, _, cnt = of.lists(pts, max_nn, 0.1, sel.astype(np.int32))
        assert cnt.max() > 64 if max_nn == 100 else (cnt == 30).all()
        need = np.unique(np.concatenate([sel, idx[idx >= 0]]))
        nidx, nd2, ncnt = of.lists(pts, max_nn, 0.1, need.astype(np.int32))
        sub = np.unique(np.concatenate([need, nidx[nidx >= 0]]))
        remap = np.full(len(pts), -1, np.int64)
        remap[sub] = np.arange(len(sub))
        kp = nidx.shape[1]
        sidx = np.full((len(sub), kp), -1, np.int32)
        sd2 = np.zeros((len(sub), kp), np.float32)
        scnt = np.zeros(len(sub), np.int32)
        sidx[remap[need]] = np.where(nidx >= 0, remap[np.maximum(nidx, 0)], -1)
        sd2[remap[need]] = nd2
        scnt[remap[need]] = ncnt
        want = of.fpfh_from_lists(pts[sub], nrm[sub], sidx, sd2, scnt, remap[sel])
        assert np.array_equal(_bits(rows.cpu().numpy()), _bits(want))


def test_permutation_and_duplicates_of_indices():
    pts, nrm = fc.scan(4000, 39)
    perm = np.random.default_rng(7).permutation(len(pts))
    a = reg.compute_fpfh_feature(_cloud(pts, nrm), 60, 0.05).cpu().numpy()
    b = reg.compute_fpfh_feature(_cloud(pts[perm], nrm[perm]), 60, 0.05).cpu().numpy()
    assert np.array_equal(_bits(b), _bits(a[perm]))   # jittered scan: no tied distances
    rows = reg.compute_fpfh_feature(_cloud(pts, nrm), 60, 0.05, indices=[5, 3, 5, 3, 0])
    assert np.array_equal(_bits(rows.cpu().numpy()), _bits(a[[0, 3, 5]]))
    assert tuple(reg.compute_fpfh_feature(_cloud(pts, nrm), 60, 0.05, indices=[]).shape) == (0, 33)


def test_errors():
    pts, nrm = fc.scan(500, 40)
    c = _cloud(pts, nrm)
    for kw, msg in ((dict(max_nn=3), "max_nn must be greater than 3."), (dict(radius=0.0), "radius must be greater than 0."),
                    (dict(max_nn=None, radius=None), "Both max_nn and radius are none."),
                    (dict(max_nn=None, radius=0.05), "max_nn=100, radius"), (dict(max_nn=129), "128")):
        with pytest.raises(RuntimeError, match=msg.replace(".", r"\.").replace("(", r"\(")):
            reg.compute_fpfh_feature(c, **kw)
    with pytest.raises(RuntimeError, match="radius must be finite"):
        reg.compute_fpfh_feature(c, 30, float("inf"))
    with pytest.raises(RuntimeError, match="indices must be integers"):
        reg.compute_fpfh_feature(c, 30, 0.05, indices=torch.tensor([1.7, 2.0]))
    with pytest.raises(RuntimeError, match="has no normal"):
        reg.compute_fpfh_feature(o3d.t.geometry.PointCloud(pts))
    bad = pts.copy()
    bad[7, 1] = np.nan
    with pytest.raises(RuntimeError, match="remove_non_finite_points"):
        reg.compute_fpfh_feature(_cloud(bad, nrm), 30, 0.05)
    badn = nrm.copy()
    badn[3, 0] = np.inf
    with pytest.raises(RuntimeError, match="normal components"):
        reg.compute_fpfh_feature(_cloud(pts, badn), 30, 0.05)
    with pytest.raises(RuntimeError, match="outside"):
        reg.compute_fpfh_feature(c, 30, 0.05, indices=[len(pts)])
    with pytest.raises(RuntimeError, match="Float32"):
        reg.compute_fpfh_feature(_f64_cloud(pts, nrm), 30, 0.05)


def test_empty_cloud():
    empty = o3d.t.geometry.PointCloud(np.zeros((0, 3), np.float32))
    for radius in (None, 0.05):
        got = reg.compute_fpfh_feature(empty, 30, radius)
        assert got.dtype == torch.float32 and tuple(got.shape) == (0, 33) and got.is_cuda


def _f64_cloud(pts, nrm):
    c = _cloud(pts, nrm)
    c.point["positions"] = c.point["positions"].double()
    return c


@pytest.mark.parametrize("dim", [33, 1, 7, 40])
def test_correspondences_equal_oracle(dim):
    rng = np.random.default_rng(dim)
    s = rng.integers(0, 3, (3000, dim)).astype(np.float32) + rng.normal(scale=0.3, size=(3000, dim)).astype(np.float32)
    t = np.concatenate([s[::2] + rng.normal(scale=0.05, size=s[::2].shape).astype(np.float32),
                        rng.integers(0, 3, (700, dim)).astype(np.float32)])
    t[5] = t[9]   # an exact tie between two target rows
    for mutual in (False, True):
        got = reg.correspondences_from_features(torch.from_numpy(s).cuda(), torch.from_numpy(t).cuda(), mutual, 0.1)
        want, _ = of.correspondences_from_features(s, t, mutual, 0.1)
        assert got.dtype == torch.int64 and np.array_equal(got.cpu().numpy(), want)


def test_mutual_filter_fallback(capsys):
    rng = np.random.default_rng(11)
    s = rng.normal(size=(1000, 33)).astype(np.float32)
    t = rng.normal(size=(1000, 33)).astype(np.float32)
    want, _ = of.correspondences_from_features(s, t, True, 0.0)
    k = len(want)
    assert 0 < k < 1000
    S, T = torch.from_numpy(s).cuda(), torch.from_numpy(t).cuda()
    # more than ratio * N mutual pairs: kept (the ratio just below k / N); at k / N exactly: falls back (strict >)
    below = float(np.nextafter(np.float32(k / 1000), np.float32(0)))
    got = reg.correspondences_from_features(S, T, True, below)
    assert np.array_equal(got.cpu().numpy(), want) and "fall back" not in capsys.readouterr().out
    got = reg.correspondences_from_features(S, T, True, float(np.float32(k) / np.float32(1000)))
    assert tuple(got.shape) == (1000, 2) and "Too few correspondences" in capsys.readouterr().out


def test_rotated_copy_end_to_end():
    """A rigidly rotated copy: mutual correspondences must map most points to their own copy.  Rotation changes the
    f32 rounding of every position and normal, so features are equal only to within rounding; on a jittered scan with
    estimated normals a point's nearest feature is its own copy for the large majority of points, and we require at
    least half of the mutual pairs to be exact (a random matching would give about 1 / N)."""
    pts, nrm = fc.scan(6000, 41)
    a = np.deg2rad(30.0)
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    pts2 = (pts.astype(np.float64) @ R.T + [0.3, -0.2, 0.1]).astype(np.float32)
    nrm2 = (nrm.astype(np.float64) @ R.T).astype(np.float32)
    f1 = reg.compute_fpfh_feature(_cloud(pts, nrm), 100, 0.05)
    f2 = reg.compute_fpfh_feature(_cloud(pts2, nrm2), 100, 0.05)
    c = reg.correspondences_from_features(f1, f2, True).cpu().numpy()
    assert len(c) > 0.1 * len(pts)
    assert (c[:, 0] == c[:, 1]).mean() > 0.5

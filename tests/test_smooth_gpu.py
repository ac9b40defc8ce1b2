"""Point-cloud smoothing on the GPU (PointCloud.smooth_laplacian, smooth_taubin, smooth_mls, smooth_bilateral) against
the CPU oracle (oracle/smooth, with brute-force neighbour lists).

Laplacian and Taubin are bit-identical to the oracle.  MLS and bilateral are bit-identical to the oracle's device-math
mode (exp, acos and cos in f64, rounded to f32); against its libm mode, the mode the reference's object code uses, the
bit-identical fraction is printed and every other row is bounded to a few ulp of the cloud's extent."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import oracle
from oracle import knn as ok
from oracle import normals as on
from oracle import smooth as osm
from tests import knn_cases as kc
from tests import normals_cases as nc
from tests.synth import make_icp_pair

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "smooth_kats.json")
MAX_NN = (1, 7, 20, 31)


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


def _lib():
    from open3d_b200 import _lib
    return _lib


def _stream():
    return int(torch.cuda.current_stream().cuda_stream)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _pc(o3d, p, normals=None):
    pc = o3d.t.geometry.PointCloud(p)
    if normals is not None:
        pc.set_point_normals(normals)
    return pc


@pytest.mark.parametrize("name", list(kc.cases()))
def test_laplacian_and_taubin_match_oracle(o3d, name):
    p = kc.cases()[name][0]
    max_nn = MAX_NN[list(kc.cases()).index(name) % len(MAX_NN)]
    pc = _pc(o3d, p)
    for fixed in (False, True):
        got = pc.smooth_laplacian(10, 0.5, max_nn, fixed).point["positions"].cpu().numpy()
        want = osm.smooth_laplacian(p, 10, (0.5,), max_nn, fixed)
        np.testing.assert_array_equal(_bits(got), _bits(want), err_msg=f"laplacian {name} {max_nn} {fixed}")
        got = pc.smooth_taubin(10, 0.5, -0.53, max_nn, fixed).point["positions"].cpu().numpy()
        want = osm.smooth_laplacian(p, 10, (0.5, -0.53), max_nn, fixed)
        np.testing.assert_array_equal(_bits(got), _bits(want), err_msg=f"taubin {name} {max_nn} {fixed}")


def test_every_max_nn_on_the_lattice(o3d):
    """Every shell of the lattice is a tie: the lower-index rule decides which neighbours each pass sees."""
    p = kc.lattice()
    pc = _pc(o3d, p)
    for max_nn in MAX_NN:
        got = pc.smooth_taubin(3, 0.5, -0.53, max_nn).point["positions"].cpu().numpy()
        np.testing.assert_array_equal(_bits(got), _bits(osm.smooth_laplacian(p, 3, (0.5, -0.53), max_nn)))


def test_one_pass_on_a_large_cloud(o3d):
    _, tgt, _, _ = make_icp_pair(2_000_000, seed=1)
    rows = np.sort(np.random.default_rng(5).choice(len(tgt), 2000, replace=False))
    got = _pc(o3d, tgt).smooth_laplacian(1).point["positions"].cpu().numpy()[rows]
    idx, _ = ok.knn(tgt, tgt[rows], 21)
    want = osm.laplacian_pass(tgt, idx, 0.5, rows)
    np.testing.assert_array_equal(_bits(got), _bits(want))


def _libm_bound(name, what, got, libm, extent):
    same = np.all(_bits(got) == _bits(libm), axis=1)
    print(f"\n{what} {name}: {same.mean():.6f} of the rows bit-identical with libm's expf / acosf / cosf")
    assert same.mean() > 0.5, (what, name, same.mean())
    np.testing.assert_allclose(got, libm, rtol=0, atol=1e-4 * extent, err_msg=f"{what} {name}")


@pytest.mark.parametrize("name", list(nc.cases()))
def test_mls_and_bilateral_match_oracle(o3d, name):
    p, radius, max_nn = nc.cases()[name]
    extent = float(np.abs(p).max()) + 1.0
    prior = on.estimate_normals(p, radius, 30)[0]
    for r in (radius, 0.0):
        lists = osm.mls_neighbours(p, r, max_nn)
        out = _pc(o3d, p, prior).smooth_mls(r, max_nn)
        got, gn = out.point["positions"].cpu().numpy(), out.point["normals"].cpu().numpy()
        want, wn = osm.smooth_mls(p, r, max_nn, prior, device_math=True, lists=lists)
        np.testing.assert_array_equal(_bits(got), _bits(want), err_msg=f"mls {name} radius {r}")
        np.testing.assert_array_equal(_bits(gn), _bits(wn), err_msg=f"mls normals {name} radius {r}")
        _libm_bound(name, f"mls radius {r}", got, osm.smooth_mls(p, r, max_nn, prior, False, lists)[0], extent)
    lists = oracle.hybrid_search(p, p, radius, max_nn, bruteforce=True)
    for ss, sr in ((radius, radius), (0.5 * radius, 2 * radius)):
        out = _pc(o3d, p, prior).smooth_bilateral(radius, max_nn, ss, sr)
        got = out.point["positions"].cpu().numpy()
        want = osm.smooth_bilateral(p, prior, radius, max_nn, ss, sr, device_math=True, lists=lists)
        np.testing.assert_array_equal(_bits(got), _bits(want), err_msg=f"bilateral {name} {ss} {sr}")
        np.testing.assert_array_equal(out.point["normals"].cpu().numpy(), prior)
        _libm_bound(name, "bilateral", got, osm.smooth_bilateral(p, prior, radius, max_nn, ss, sr, False, lists),
                    extent)


def test_kats(o3d):
    kats = json.load(open(GOLDEN))
    for case in kats["cases"]:
        nrm = case.get("normals")
        pc = _pc(o3d, np.asarray(case["points"], np.float32), None if nrm is None else np.asarray(nrm, np.float32))
        got = getattr(pc, case["call"])(**case["args"]).point["positions"].cpu().numpy()
        np.testing.assert_allclose(got, case["want"], rtol=0, atol=case["atol"], err_msg=case["name"])
    for case in kats["errors"]:
        pc = _pc(o3d, np.asarray(case["points"], np.float32))
        with pytest.raises(RuntimeError, match="Sigma values must be positive."):
            getattr(pc, case["call"])(**case["args"])


def test_boundaries_and_errors(o3d):
    geo = o3d.t.geometry
    empty = geo.PointCloud(np.zeros((0, 3), np.float32))
    for call in ("smooth_laplacian", "smooth_taubin", "smooth_mls", "smooth_bilateral"):
        assert getattr(empty, call)().point["positions"].shape == (0, 3)
    assert empty.smooth_bilateral(sigma_s=0.0).point["positions"].shape == (0, 3)   # empty returns first
    p = kc.uniform(500)
    pc = _pc(o3d, p)
    for out in (pc.smooth_laplacian(0), pc.smooth_taubin(0), pc.smooth_laplacian(3, max_nn=0),
                pc.smooth_taubin(3, max_nn=-1), pc.smooth_mls(0.0, 0), pc.smooth_mls(-1.0, -1)):
        np.testing.assert_array_equal(out.point["positions"].cpu().numpy(), p)
    with pytest.raises(RuntimeError, match="non-negative"):
        pc.smooth_laplacian(-1)
    with pytest.raises(RuntimeError, match="32"):
        pc.smooth_laplacian(1, max_nn=32)   # k' = 33
    pc.smooth_laplacian(1, max_nn=31)
    with pytest.raises(RuntimeError, match="32"):
        pc.smooth_taubin(1, max_nn=40)
    with pytest.raises(RuntimeError, match="32"):
        pc.smooth_mls(0.1, 33)
    with pytest.raises(RuntimeError, match="32"):
        pc.smooth_mls(0.0, 33)
    few = _pc(o3d, p[:20])
    few.smooth_mls(0.0, 40)   # k' = min(n, max_nn) = 20
    few.smooth_laplacian(1, max_nn=40)   # k' = min(n, max_nn + 1) = 20
    with pytest.raises(RuntimeError, match="fixed-radius"):
        pc.smooth_mls(0.1, 0)
    with pytest.raises(RuntimeError, match="Sigma values must be positive."):
        pc.smooth_bilateral(sigma_r=-1.0)
    with pytest.raises(RuntimeError, match=r"estimate_normals\(max_nn, radius\)"):
        pc.smooth_bilateral()
    f64 = geo.PointCloud()
    f64.point["positions"] = torch.from_numpy(p.astype(np.float64)).cuda()
    for call in ("smooth_laplacian", "smooth_taubin", "smooth_mls", "smooth_bilateral"):
        with pytest.raises(RuntimeError, match="Float32"):
            getattr(f64, call)()


def test_attributes_are_cloned(o3d):
    p, radius, max_nn = nc.cases()["scan"]
    n = len(p)
    prior = on.estimate_normals(p, radius, max_nn)[0]
    pc = _pc(o3d, p, prior)
    pc.set_point_colors(np.abs(p))
    pc.point["labels"] = torch.arange(n, device="cuda")
    before = {k: v.clone() for k, v in pc.point.items()}
    for out in (pc.smooth_laplacian(2), pc.smooth_taubin(2, use_fixed_neighborhoods=True), pc.smooth_mls(radius, max_nn),
                pc.smooth_bilateral(radius, max_nn)):
        assert set(out.point) == set(pc.point)
        for k in ("colors", "labels"):
            assert torch.equal(out.point[k], pc.point[k]) and out.point[k].data_ptr() != pc.point[k].data_ptr()
        assert not torch.equal(out.point["positions"], pc.point["positions"])
    for k, v in before.items():   # the source cloud is untouched
        assert torch.equal(pc.point[k], v)
    bare = _pc(o3d, p).smooth_mls(radius, max_nn)
    assert "normals" not in bare.point


def test_launch_count_is_fixed_per_call(o3d):
    L = _lib()
    counts = {}
    for n in (2000, 50000, 200000):
        p = kc.uniform(n, seed=n)
        prior = np.tile(np.float32([0, 0, 1]), (n, 1))
        pc = _pc(o3d, p, prior)
        calls = {"laplacian": lambda: pc.smooth_laplacian(3),
                 "taubin fixed": lambda: pc.smooth_taubin(3, use_fixed_neighborhoods=True),
                 "mls": lambda: pc.smooth_mls(0.05, 20), "mls knn": lambda: pc.smooth_mls(0.0, 20),
                 "bilateral": lambda: pc.smooth_bilateral(0.05, 20)}
        for name, call in calls.items():
            before = L.launch_count()
            call()
            torch.cuda.synchronize()
            counts.setdefault(name, []).append(L.launch_count() - before)
    for name, c in counts.items():
        assert c[0] >= 1 and len(set(c)) == 1, (name, c)


def test_memory_balances_on_success_and_failure():
    if torch.cuda.get_allocator_backend() == "cudaMallocAsync":
        pytest.skip("torch shares the default memory pool")
    from tests.test_host_ownership_gpu import _Pool
    L = _lib()
    pool = _Pool()
    data = _dev(kc.clusters())
    n = int(data.shape[0])
    bad = data.clone()
    bad[3, 0] = float("nan")
    nrm = torch.zeros_like(data)
    nrm[:, 2] = 1
    out = torch.empty_like(data)
    f = np.array([0.5, -0.53])
    cases = []

    def balanced(name, call, expect=0):
        u0 = pool.used()
        rc = call()
        assert rc == expect, (name, rc, L.last_error())
        cases.append((name, u0, pool.used()))

    for _ in range(2):
        for fixed in (0, 1):
            balanced(f"taubin {fixed}", lambda: L.lib.o3db_smooth_laplacian(data.data_ptr(), n, 2, f.ctypes.data, 2, 20,
                                                                            fixed, out.data_ptr(), _stream()))
            balanced(f"taubin {fixed} with a NaN", lambda: L.lib.o3db_smooth_laplacian(
                bad.data_ptr(), n, 2, f.ctypes.data, 2, 20, fixed, out.data_ptr(), _stream()), L.ERR_INVALID)
        for r in (0.05, 0.0):
            balanced(f"mls {r}", lambda: L.lib.o3db_smooth_mls(data.data_ptr(), n, r, 20, out.data_ptr(), nrm.data_ptr(),
                                                              _stream()))
        balanced("mls knn with a NaN", lambda: L.lib.o3db_smooth_mls(bad.data_ptr(), n, 0.0, 20, out.data_ptr(), None,
                                                                    _stream()), L.ERR_INVALID)
        balanced("bilateral", lambda: L.lib.o3db_smooth_bilateral(data.data_ptr(), nrm.data_ptr(), n, 0.05, 20, 0.05,
                                                                  0.05, out.data_ptr(), _stream()))
    torch.cuda.synchronize()
    for name, u0, u1 in cases:
        assert u1 == u0, (name, u0, u1)

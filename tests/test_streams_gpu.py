"""Every GPU entry point on a non-blocking side stream, and the handles used across streams.

The C ABI promises that a call runs on the `stream` it is given and, when it returns values to the host, synchronises
that stream and never the device (include/open3d_b200.h).  The legacy default stream hides a wrong stream: it waits
for every blocking stream and they wait for it.  So each case here runs on a stream created non-blocking, behind a
~50 ms sleep, with its inputs filled by copies queued after the sleep into tensors that first held a valid decoy of
the same shape (another seed of the same generator).  Library work on any other stream reads the decoy, or reads an
output before it is written, and the result differs from the default-stream run, which is compared bit for bit.
Every decoy is valid data, so a wrong-stream read gives a wrong answer, never an invalid address.

A spy around the ctypes functions records the stream argument of every call: inside a side-stream run each one must
be the side stream, and the calls made there must cover every header entry point with a `void* stream` parameter but
the named exclusions (the header part of that check runs without a GPU).

The harness cannot force a PDL (programmatic dependent launch) overlap window open: it runs the PDL chains on a side
stream behind a caller's kernel, which is where a read before griddepcontrol.wait would see the caller's data late.
"""
import ctypes as C
import gc
import os
import re
import time

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "open3d_b200.h")

# Entry points with a stream parameter that this file does not run on a side stream, and why.
EXCLUDED = {
    "o3db_comm_allreduce_f64": "multi-GPU: needs an NCCL communicator of several ranks (tests/multigpu_check.py); the "
                               "sharded ICP path (a communicator passed to o3db_icp_create) is left out for the same "
                               "reason",
}


def stream_entry_points():
    """{symbol: position of its `void* stream` parameter} for every prototype of the header that has one."""
    with open(HEADER) as f:
        src = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    out = {}
    for name, args in re.findall(r"\b(o3db_\w+)\s*\(([^;{}]*?)\)\s*;", src):
        params = [p.strip() for p in args.split(",")]
        for i, p in enumerate(params):
            if re.fullmatch(r"void\s*\*\s*stream", re.sub(r"\s+", " ", p)):
                out[name] = i
    return out


def test_header_stream_entry_points_are_covered_or_excluded():
    """Runs without a GPU: a new entry point with a stream fails the suite until some code calls it through ctypes
    (`lib.<name>` in the package or in this file) or it has a reasoned entry in EXCLUDED.  That is a text check only:
    that each such call really runs on the side stream is checked on the GPU, by
    test_zz_side_runs_covered_every_entry_point."""
    eps = stream_entry_points()
    assert len(eps) > 70 and eps["o3db_knn_search"] == 7 and eps["o3db_icp_create"] == 8
    assert set(EXCLUDED) <= set(eps), set(EXCLUDED) - set(eps)
    srcs = [__file__] + [os.path.join(dp, f) for dp, _, fs in os.walk(os.path.join(ROOT, "open3d_b200")) for f in fs
                         if f.endswith(".py")]
    text = ""
    for path in srcs:
        with open(path) as f:
            text += f.read()
    # every other one is called through ctypes by the Python layer or by a case of this file
    missing = [n for n in eps if n not in EXCLUDED and not re.search(r"\blib\.%s\b" % n, text)]
    assert not missing, f"entry points with no side-stream case and no exclusion: {missing}"


# ------------------------------------------------------------------------------------------------ GPU harness

class _Spy:
    """Recording wrappers around the o3db_* ctypes functions of the one shared _lib.lib object."""

    def __init__(self, lib, eps):
        self.lib, self.eps, self.orig = lib, eps, {}
        self.side = None            # the side stream's handle while a side-stream run is in progress
        self.side_calls = set()     # symbols called inside side-stream runs
        self.cases_run = set()      # names of the cases that ran on the side stream
        self.wrong = []             # (symbol, stream argument) of side-run calls given another stream
        for name, pos in eps.items():
            fn = getattr(lib, name, None)
            if fn is None:
                continue
            self.orig[name] = fn
            setattr(lib, name, self._wrap(name, pos, fn))

    def _wrap(self, name, pos, fn):
        def call(*args):
            if self.side is not None:
                self.side_calls.add(name)
                got = int(args[pos] or 0)
                if got != self.side:
                    self.wrong.append((name, got))
            return fn(*args)
        return call

    def restore(self):
        for name, fn in self.orig.items():
            setattr(self.lib, name, fn)


@pytest.fixture(scope="module")
def env():
    import open3d_b200
    from open3d_b200 import _lib
    assert torch.cuda.is_available()
    side = torch.cuda.Stream()
    busy = torch.cuda.Stream()
    cuda = C.CDLL("libcuda.so.1")
    for s in (side, busy):
        flags = C.c_uint(0)
        assert cuda.cuStreamGetFlags(C.c_void_p(s.cuda_stream), C.byref(flags)) == 0
        assert flags.value & 1, "the side stream is blocking: it would wait for stream 0 and prove nothing"
    # cycles of torch.cuda._sleep per millisecond
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda._sleep(1000)
    a.record()
    torch.cuda._sleep(20_000_000)
    b.record()
    b.synchronize()
    per_ms = 20_000_000 / a.elapsed_time(b)
    spy = _Spy(_lib.lib, stream_entry_points())
    yield dict(o3d=open3d_b200, L=_lib, side=side, busy=busy, per_ms=per_ms, spy=spy)
    spy.restore()
    side.synchronize()
    busy.synchronize()
    torch.cuda.synchronize()


def _leaves(x):
    """Every array-like leaf of an output tree, as a host numpy array (floats and ints as 0-d arrays)."""
    if isinstance(x, torch.Tensor):
        return [x.detach().cpu().numpy()]
    if isinstance(x, np.ndarray):
        return [x]
    if isinstance(x, (list, tuple)):
        return [a for v in x for a in _leaves(v)]
    if isinstance(x, dict):
        return [a for k in sorted(x) for a in _leaves(x[k])]
    if isinstance(x, (bool, int, float, np.generic)):
        return [np.asarray(x)]
    if x is None:
        return [np.asarray([], np.int8)]
    raise TypeError(type(x))


def _clone(x):
    if isinstance(x, torch.Tensor):
        return x.clone()
    if isinstance(x, (list, tuple)):
        return type(x)(_clone(v) for v in x)
    if isinstance(x, dict):
        return {k: _clone(v) for k, v in x.items()}
    if isinstance(x, np.ndarray):
        return x.copy()
    return x


def _same(a, b):
    la, lb = _leaves(a), _leaves(b)
    if len(la) != len(lb):
        return False
    for x, y in zip(la, lb):
        x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
        if x.shape != y.shape or x.dtype != y.dtype or x.tobytes() != y.tobytes():
            return False
    return True


def _device(inputs):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) else v
            for k, v in inputs.items()}


class Case:
    """make(seed) -> {name: numpy array (uploaded) or anything else (passed as is)};
    run(env, inputs, keep) -> output tree; rng: seed the library's engine before each run."""

    def __init__(self, name, make, run, rng=False, key=None, ulps=0, atol=0.0):
        self.name, self.make, self.run, self.rng, self.key = name, make, run, rng, key or (lambda out: out)
        self.ulps = ulps   # float outputs summed with atomics in no fixed order: this many units in the last place
        self.atol = atol   # float outputs of a computation whose inputs come in no fixed order: absolute tolerance

    def __call__(self, env, inputs, keep):
        if self.rng:
            env["o3d"].utility.random.seed(7)
        return self.key(self.run(env, inputs, keep))


def side_run(env, case, real, decoy_seed=1):
    """The case on the side stream: inputs hold the decoy until copies queued behind a ~50 ms sleep fill them."""
    bufs = _device(case.make(decoy_seed))
    src = _device(real)
    torch.cuda.synchronize()
    side, spy = env["side"], env["spy"]
    keep = []
    spy.cases_run.add(case.name)
    spy.side = int(side.cuda_stream)
    try:
        with torch.cuda.stream(side):
            torch.cuda._sleep(int(50 * env["per_ms"]))
            for k, v in bufs.items():
                if isinstance(v, torch.Tensor):
                    v.copy_(src[k])
            out = _clone(case(env, bufs, keep))
        side.synchronize()
    finally:
        spy.side = None
    return out, keep


def default_run(env, case, inputs):
    keep = []
    out = _clone(case(env, _device(inputs), keep))
    torch.cuda.synchronize()
    return out, keep


# ------------------------------------------------------------------------------------------------ case inputs

def _pc(seed, n=3000):
    from tests.synth import make_colors, make_icp_pair
    src, tgt, nrm, _ = make_icp_pair(n, seed=seed)
    return dict(p=tgt, n=nrm, c=make_colors(tgt, seed).astype(np.float32), s=src)


def _pair(seed, n=3000):
    from tests.synth import make_colors, make_icp_pair
    src, tgt, nrm, _ = make_icp_pair(n, seed=seed)
    rng = np.random.default_rng(seed)
    sn = nrm[rng.permutation(len(nrm))[: len(src)]] if len(nrm) >= len(src) else nrm
    return dict(s=src, t=tgt, tn=nrm, sn=np.ascontiguousarray(sn), sc=make_colors(src, seed).astype(np.float32),
                tc=make_colors(tgt, seed + 5).astype(np.float32))


def _doppler(seed, n=3000):
    from tests.doppler_cases import make_doppler_pair
    s, d, dirs, t, tn, _, _ = make_doppler_pair(n, seed=seed)
    return dict(s=s, d=np.ascontiguousarray(d, np.float32), dirs=np.ascontiguousarray(dirs, np.float32), t=t, tn=tn)


def _depth(seed, color=False):
    from tests.synth import camera_pose, render_depth
    d, c = render_depth(camera_pose(100 + 37 * seed), with_color=True)
    return (d.numpy(), c.numpy()) if color else d.numpy()


def _feats(seed, n=2000, dim=33):
    rng = np.random.default_rng(seed)
    return rng.random((n, dim), np.float32), rng.random((n + 100, dim), np.float32)


K = np.array([[525.0, 0, 319.5], [0, 525.0, 239.5], [0, 0, 1.0]])


def _cloud(o3d, x, normals=None, colors=None):
    pc = o3d.t.geometry.PointCloud(x)
    if normals is not None:
        pc.set_point_normals(normals)
    if colors is not None:
        pc.set_point_colors(colors)
    return pc


def _pts(pc):
    return {k: v for k, v in pc.point.items()}


def _rows_by_voxel(out, voxel):
    """voxel_down_sample's row order is a hash map's and its means f32 atomics': rows sorted by their voxel."""
    pos = out["positions"].cpu().numpy()
    order = np.lexsort(np.floor(pos / voxel).astype(np.int64).T[::-1])
    return {k: v.cpu().numpy()[order] for k, v in out.items()}


def _reg(res):
    return (res.transformation, res.correspondence_set, res.fitness, res.inlier_rmse, res.converged,
            res.num_iterations)


# ------------------------------------------------------------------------------------------------ cases

def _point_cloud_cases():
    cs = []
    add = lambda *a, **k: cs.append(Case(*a, **k))   # noqa: E731

    def vds(e, d, keep):
        out = _cloud(e["o3d"], d["p"], d["n"], d["c"]).voxel_down_sample(0.05)
        return _pts(out)
    # (rows compared in voxel order, and to the f32 atomics' rounding: see _rows_by_voxel)
    add("voxel_down_sample", _pc, vds, key=lambda o: _rows_by_voxel(o, 0.05), ulps=16)

    def vds_raw(e, d, keep):
        L, n = e["L"], d["p"].shape[0]
        po, no, co = (torch.empty_like(d[k]) for k in ("p", "n", "c"))
        cnt = C.c_int64()
        L.check(L.lib.o3db_voxel_down_sample(d["p"].data_ptr(), d["n"].data_ptr(), d["c"].data_ptr(), n, 0.05,
                                             po.data_ptr(), no.data_ptr(), co.data_ptr(), C.byref(cnt),
                                             torch.cuda.current_stream().cuda_stream))
        m = cnt.value
        return {"positions": po[:m], "normals": no[:m], "colors": co[:m]}
    add("voxel_down_sample_raw", _pc, vds_raw, key=lambda o: _rows_by_voxel(o, 0.05), ulps=16)

    for solver in ("reference", "exact"):
        add(f"estimate_color_gradients_{solver}", _pc,
            lambda e, d, keep, s=solver: _cloud(e["o3d"], d["p"], d["n"], d["c"]).estimate_color_gradients(
                30, 0.08, s).point["color_gradients"])

    def grads_default(e, d, keep):
        L, n = e["L"], d["p"].shape[0]
        out = torch.empty_like(d["p"])
        L.check(L.lib.o3db_estimate_color_gradients(d["p"].data_ptr(), d["n"].data_ptr(), d["c"].data_ptr(), n, 0.08,
                                                    30, out.data_ptr(), torch.cuda.current_stream().cuda_stream))
        return out
    add("estimate_color_gradients_c_abi", _pc, grads_default)

    def normals(e, d, keep):
        pc = _cloud(e["o3d"], d["p"])
        pc.estimate_normals(30, 0.08)
        a = pc.point["normals"].clone()
        pc.orient_normals_to_align_with_direction((0.0, 0.3, 1.0))
        b = pc.point["normals"].clone()
        pc.orient_normals_towards_camera_location((0.5, 0.5, -2.0))
        return a, b, pc.point["normals"]
    add("estimate_and_orient_normals", _pc, normals)

    add("remove_radius_outliers", _pc, lambda e, d, k: _cloud(e["o3d"], d["p"]).remove_radius_outliers(6, 0.04)[1])
    add("remove_statistical_outliers", _pc,
        lambda e, d, k: _cloud(e["o3d"], d["p"]).remove_statistical_outliers(20, 1.0)[1])

    def dup_make(seed):
        x = _pc(seed)["p"]
        rng = np.random.default_rng(seed)
        rows = rng.permutation(len(x))
        x[rows[:300]] = x[rows[300:600]]
        x[rows[600:700], 1] = np.nan
        x[rows[700:800], 2] = np.inf
        return dict(p=x)
    add("remove_duplicated_points", dup_make,
        lambda e, d, k: _cloud(e["o3d"], d["p"]).remove_duplicated_points()[1])
    add("remove_non_finite_points", dup_make,
        lambda e, d, k: _cloud(e["o3d"], d["p"]).remove_non_finite_points()[1])

    add("smooth_laplacian", _pc, lambda e, d, k: _cloud(e["o3d"], d["p"]).smooth_laplacian(3, 0.5, 10).point["positions"])
    add("smooth_taubin", _pc, lambda e, d, k: _cloud(e["o3d"], d["p"]).smooth_taubin(2, 0.5, -0.53, 10).point["positions"])
    add("smooth_mls", _pc, lambda e, d, k: _pts(_cloud(e["o3d"], d["p"], d["n"]).smooth_mls(0.06, 20)))
    add("smooth_bilateral", _pc,
        lambda e, d, k: _cloud(e["o3d"], d["p"], d["n"]).smooth_bilateral(0.06, 20, 0.05, 0.05).point["positions"])
    add("cluster_dbscan", _pc, lambda e, d, k: _cloud(e["o3d"], d["p"]).cluster_dbscan(0.025, 5), rng=True)
    add("segment_plane", _pc, lambda e, d, k: _cloud(e["o3d"], d["p"]).segment_plane(0.01, 3, 200), rng=True)
    add("farthest_point_down_sample", _pc,
        lambda e, d, k: _cloud(e["o3d"], d["p"]).farthest_point_down_sample(300, 5).point["positions"])
    add("compute_boundary_points", _pc,
        lambda e, d, k: _cloud(e["o3d"], d["p"], d["n"]).compute_boundary_points(0.06, 30, 90.0)[1])

    def metrics(e, d, k):
        g = e["o3d"].t.geometry
        return _cloud(e["o3d"], d["p"]).compute_metrics(
            _cloud(e["o3d"], d["s"]), [g.Metric.ChamferDistance, g.Metric.HausdorffDistance, g.Metric.FScore],
            g.MetricParameters(fscore_radius=[0.01, 0.02]))
    add("compute_metrics", _pc, metrics)

    def transform(e, d, k):
        pc = _cloud(e["o3d"], d["p"], d["n"])
        T = np.eye(4)
        T[:3, :3] = [[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]
        T[:3, 3] = [0.1, -0.2, 0.3]
        pc.transform(T)
        return _pts(pc)
    add("transform", _pc, transform)

    def knn_lists(e, d, keep):
        L = e["L"]
        nns = e["o3d"].core.nns.NearestNeighborSearch(d["p"])
        nns.knn_index()
        q = d["s"]
        idx = torch.empty((q.shape[0], 40), dtype=torch.int32, device="cuda")
        d2 = torch.empty((q.shape[0], 40), dtype=torch.float32, device="cuda")
        cnt = torch.empty((q.shape[0],), dtype=torch.int32, device="cuda")
        L.check(L.lib.o3db_knn_search_lists(nns._knn.ptr, q.data_ptr(), q.shape[0], 40, 0.05, idx.data_ptr(),
                                            d2.data_ptr(), cnt.data_ptr(), torch.cuda.current_stream().cuda_stream))
        return idx, d2, cnt
    add("knn_search_lists", _pc, knn_lists)

    def spatial_hash(e, d, keep):
        L, n, size = e["L"], d["p"].shape[0], 1024
        index = torch.empty((n,), dtype=torch.int32, device="cuda")
        splits = torch.empty((size + 1,), dtype=torch.int32, device="cuda")
        L.check(L.lib.o3db_build_spatial_hash_table(d["p"].data_ptr(), n, 0.03, size, index.data_ptr(),
                                                    splits.data_ptr(), torch.cuda.current_stream().cuda_stream))
        return index, splits

    def by_bucket(out):   # the order inside a bucket is undefined, as upstream's
        index, splits = out[0].cpu().numpy(), out[1].cpu().numpy()
        bucket = np.repeat(np.arange(len(splits) - 1), np.diff(splits))
        return np.sort(index + bucket.astype(np.int64) * (1 << 32)), splits
    add("build_spatial_hash_table", _pc, spatial_hash, key=by_bucket)
    return cs


def _image_cases():
    cs = []
    add = lambda *a, **k: cs.append(Case(*a, **k))   # noqa: E731
    E = np.eye(4)
    E[:3, 3] = [0.01, -0.02, 0.03]

    add("create_from_depth_image", lambda s: dict(d=_depth(s)),
        lambda e, d, k: _pts(e["o3d"].t.geometry.PointCloud.create_from_depth_image(d["d"], K, E, 1000.0, 3.0, 2)))

    def rgbd(seed):
        dep, col = _depth(seed, color=True)
        return dict(d=dep, c=col)

    def from_rgbd(e, d, k):
        g = e["o3d"].t.geometry
        return _pts(g.PointCloud.create_from_rgbd_image(g.RGBDImage(d["c"], d["d"]), K, E, 1000.0, 3.0, 1))
    add("create_from_rgbd_image", rgbd, from_rgbd)

    def project(e, d, k):
        pc = _cloud(e["o3d"], d["p"], colors=d["c"])
        pc.point["positions"] = pc.point["positions"] + torch.tensor([0.0, 0.0, 1.5], device="cuda")
        a = pc.project_to_depth_image(640, 480, K, None, 1000.0, 4.0)
        b = pc.project_to_rgbd_image(640, 480, K, None, 1000.0, 4.0)
        return a.as_tensor(), b.depth.as_tensor(), b.color.as_tensor()
    add("project_to_images", _pc, project)

    def filters(e, d, k):
        img = e["o3d"].t.geometry.Image(d["d"])
        nan = float("nan")
        depth = img.clip_transform(1000.0, 0.0, 3.0, nan)
        down = depth.pyr_down_depth(0.1, nan)
        v = depth.create_vertex_map(K, nan)
        return depth.as_tensor(), down.as_tensor(), v.as_tensor(), v.create_normal_map(nan).as_tensor(), \
            depth.filter_bilateral(5, 5.0, 10.0).as_tensor()
    add("image_filters", lambda s: dict(d=_depth(s)), filters)
    return cs


def _registration_cases():
    cs = []
    add = lambda *a, **k: cs.append(Case(*a, **k))   # noqa: E731

    def clouds(e, d, est):
        o3d = e["o3d"]
        if est == "doppler":
            s = _cloud(o3d, d["s"])
            s.point["dopplers"], s.point["directions"] = d["d"], d["dirs"]
            return s, _cloud(o3d, d["t"], d["tn"])
        if est == "colored":
            t = _cloud(o3d, d["t"], d["tn"], d["tc"])
            t.estimate_color_gradients(30, 0.08)
            return _cloud(o3d, d["s"], colors=d["sc"]), t
        return _cloud(o3d, d["s"], d["sn"] if est == "symmetric" else None), _cloud(o3d, d["t"], d["tn"])

    def estimator(reg, est):
        return {"plane": reg.TransformationEstimationPointToPlane, "point": reg.TransformationEstimationPointToPoint,
                "symmetric": reg.TransformationEstimationSymmetric, "colored": reg.TransformationEstimationForColoredICP,
                "doppler": reg.TransformationEstimationForDopplerICP}[est]()

    for est in ("plane", "point", "symmetric", "colored", "doppler"):
        make = _doppler if est == "doppler" else _pair

        def one(e, d, k, est=est):
            reg = e["o3d"].t.pipelines.registration
            s, t = clouds(e, d, est)
            return _reg(reg.icp(s, t, 0.05, np.eye(4), estimator(reg, est), reg.ICPConvergenceCriteria(0, 0, 12)))

        def multi(e, d, k, est=est):
            reg = e["o3d"].t.pipelines.registration
            s, t = clouds(e, d, est)
            crit = [reg.ICPConvergenceCriteria(0, 0, n) for n in (6, 4)]
            # voxels far below the 2 cm point spacing: each holds one point, so its mean is exact and the pyramid
            # differs from run to run in row order only (see _rows_by_voxel), which the correspondence set follows
            res = reg.multi_scale_icp(s, t, [2e-4, 1e-4], crit, [0.08, 0.05], np.eye(4), estimator(reg, est))
            return res.transformation, res.fitness, res.inlier_rmse, res.converged, res.num_iterations
        add(f"icp_{est}", make, one)
        # (the pyramid's row order sets the order of the f32 sums: results agree to rounding, not bit for bit)
        add(f"multi_scale_icp_{est}", make, multi, atol=1e-6)

    def one_shots(e, d, keep):
        """The C ABI's one-shot ICP calls (create + iterate + finish + destroy on the caller's stream)."""
        L, st = e["L"], torch.cuda.current_stream().cuda_stream
        opt = L.IcpOptions(0.05, 8, 0.0, 0.0, L.RobustKernel(0, 1.0, 1.0), 0.0)
        T0 = np.eye(4)
        n, m = d["s"].shape[0], d["t"].shape[0]
        outs = []
        for kind in ("plane", "point", "symmetric", "colored"):
            res, corr = L.IcpResult(), torch.empty((n,), dtype=torch.int64, device="cuda")
            per = np.zeros(16)
            if kind == "plane":
                rc = L.lib.o3db_icp_point_to_plane(d["s"].data_ptr(), n, d["t"].data_ptr(), d["tn"].data_ptr(), m,
                                                   L.dptr(T0), C.byref(opt), C.byref(res), corr.data_ptr(),
                                                   L.dptr(per), st)
            elif kind == "point":
                rc = L.lib.o3db_icp_point_to_point(d["s"].data_ptr(), n, d["t"].data_ptr(), m, L.dptr(T0),
                                                   C.byref(opt), C.byref(res), corr.data_ptr(), L.dptr(per), st)
            elif kind == "symmetric":
                rc = L.lib.o3db_icp_symmetric(d["s"].data_ptr(), d["sn"].data_ptr(), n, d["t"].data_ptr(),
                                              d["tn"].data_ptr(), m, L.dptr(T0), C.byref(opt), C.byref(res),
                                              corr.data_ptr(), L.dptr(per), st)
            else:
                g = torch.zeros_like(d["t"])
                L.check(L.lib.o3db_estimate_color_gradients(d["t"].data_ptr(), d["tn"].data_ptr(), d["tc"].data_ptr(),
                                                            m, 0.08, 30, g.data_ptr(), st))
                rc = L.lib.o3db_icp_colored(d["s"].data_ptr(), d["sc"].data_ptr(), n, d["t"].data_ptr(),
                                            d["tn"].data_ptr(), d["tc"].data_ptr(), g.data_ptr(), m, L.dptr(T0),
                                            C.byref(opt), 0.968, C.byref(res), corr.data_ptr(), L.dptr(per), st)
            L.check(rc)
            outs.append((np.array(res.transformation), res.fitness, res.inlier_rmse, res.num_iterations, corr, per))
        h = C.c_void_p()     # a handle reset and run again
        L.check(L.lib.o3db_icp_create(d["s"].data_ptr(), n, d["t"].data_ptr(), d["tn"].data_ptr(), m, L.dptr(T0),
                                      C.byref(opt), None, st, C.byref(h)))
        try:
            L.check(L.lib.o3db_icp_iterate(h, 3, st))
            L.check(L.lib.o3db_icp_reset(h, st))
            L.check(L.lib.o3db_icp_iterate(h, 8, st))
            res, corr, per = L.IcpResult(), torch.empty((n,), dtype=torch.int64, device="cuda"), np.zeros(16)
            L.check(L.lib.o3db_icp_finish(h, C.byref(res), corr.data_ptr(), L.dptr(per), st))
        finally:
            L.lib.o3db_icp_destroy(h)
        outs.append((np.array(res.transformation), res.fitness, corr, per))
        return outs
    add("icp_one_shots", _pair, one_shots)

    def doppler_one_shot(e, d, keep):
        L, st = e["L"], torch.cuda.current_stream().cuda_stream
        opt = L.IcpOptions(0.05, 8, 0.0, 0.0, L.RobustKernel(0, 1.0, 1.0), 0.0)
        reg = e["o3d"].t.pipelines.registration
        params = reg.TransformationEstimationForDopplerICP()._params()
        n, m = d["s"].shape[0], d["t"].shape[0]
        res, corr, per = L.IcpResult(), torch.empty((n,), dtype=torch.int64, device="cuda"), np.zeros(16)
        L.check(L.lib.o3db_icp_doppler(d["s"].data_ptr(), d["d"].data_ptr(), d["dirs"].data_ptr(), n, d["t"].data_ptr(),
                                       d["tn"].data_ptr(), m, L.dptr(np.eye(4)), C.byref(opt), C.byref(params),
                                       C.byref(res), corr.data_ptr(), L.dptr(per), st))
        return np.array(res.transformation), res.fitness, res.inlier_rmse, corr, per
    add("icp_doppler_one_shot", _doppler, doppler_one_shot)

    def poses(e, d, keep):
        """The estimators' single-step poses on a given correspondence set."""
        reg = e["o3d"].t.pipelines.registration
        n = d["s"].shape[0]
        corr = torch.arange(n, dtype=torch.int64, device="cuda")
        corr[::5] = -1
        s = _cloud(e["o3d"], d["s"], d["sn"], d["sc"])
        t = _cloud(e["o3d"], d["t"][:n], d["tn"][:n], d["tc"][:n])
        t.estimate_color_gradients(30, 0.08)
        out = [reg.TransformationEstimationPointToPlane().compute_pose(s, t, corr),
               reg.TransformationEstimationForColoredICP().compute_pose(s, t, corr),
               reg.TransformationEstimationPointToPoint().compute_rt(s, t, corr),
               reg.TransformationEstimationSymmetric().compute_transformation(s, t, corr)]
        ms = s.point["positions"][corr >= 0].mean(0).cpu().numpy()
        mt = t.point["positions"][corr[corr >= 0]].mean(0).cpu().numpy()
        out.append(reg.TransformationEstimationSymmetric().compute_pose(s, t, corr, ms, mt))
        return out
    add("compute_poses", _pair, poses)

    def doppler_pose(e, d, keep):
        reg = e["o3d"].t.pipelines.registration
        n = d["s"].shape[0]
        s = _cloud(e["o3d"], d["s"])
        s.point["dopplers"], s.point["directions"] = d["d"], d["dirs"]
        t = _cloud(e["o3d"], d["t"][:n], d["tn"][:n])
        corr = torch.arange(n, dtype=torch.int64, device="cuda")
        return reg.TransformationEstimationForDopplerICP().compute_pose(s, t, corr, np.eye(4), 0)
    add("compute_pose_doppler", _doppler, doppler_pose)

    def evaluate(e, d, keep):
        reg = e["o3d"].t.pipelines.registration
        s, t = _cloud(e["o3d"], d["s"]), _cloud(e["o3d"], d["t"], d["tn"])
        T = np.eye(4)
        T[:3, 3] = [0.002, -0.001, 0.003]
        L = e["L"]
        info2 = np.zeros(36)
        num = C.c_int64()
        corr = torch.arange(d["s"].shape[0], dtype=torch.int64, device="cuda")
        L.check(L.lib.o3db_compute_information_matrix(d["t"].data_ptr(), corr.data_ptr(), corr.shape[0], L.dptr(info2),
                                                      C.byref(num), torch.cuda.current_stream().cuda_stream))
        return _reg(reg.evaluate_registration(s, t, 0.05, T)), reg.get_information_matrix(s, t, 0.05, T), info2, \
            num.value
    add("evaluate_registration_and_information", _pair, evaluate)

    def fpfh(e, d, keep):
        reg = e["o3d"].t.pipelines.registration
        pc = _cloud(e["o3d"], d["p"], d["n"])
        f = reg.compute_fpfh_feature(pc, 60, 0.1)
        return f, reg.correspondences_from_features(f, f.flip(0), True)
    add("fpfh_and_correspondences", _pc, fpfh)

    def global_make(seed):
        from tests import ransac_cases as rc
        s, t, corr = rc.pair(1500, 400, 0.6, seed)[:3]
        fs, ft = _feats(seed, len(s), 8)
        ft = np.ascontiguousarray(fs[np.arange(len(t)) % len(s)] + 0.01 * np.float32(seed))
        return dict(s=np.ascontiguousarray(s, np.float32), t=np.ascontiguousarray(t, np.float32),
                    corr=np.ascontiguousarray(corr, np.int64), fs=fs, ft=ft)

    def ransac(e, d, keep):
        reg = e["o3d"].t.pipelines.registration
        s, t = _cloud(e["o3d"], d["s"]), _cloud(e["o3d"], d["t"])
        crit = reg.RANSACConvergenceCriteria(2000, 0.999)
        a = reg.registration_ransac_based_on_correspondence(s, t, d["corr"], 0.02, None, 3, None, crit)
        b = reg.registration_ransac_based_on_feature_matching(s, t, d["fs"], d["ft"], True, 0.02, None, 3, None, crit)
        return _reg(a), _reg(b)
    add("registration_ransac", global_make, ransac, rng=True)

    def fgr(e, d, keep):
        reg = e["o3d"].t.pipelines.registration
        s, t = _cloud(e["o3d"], d["s"]), _cloud(e["o3d"], d["t"])
        a = reg.registration_fgr_based_on_correspondence(s, t, d["corr"])
        b = reg.registration_fgr_based_on_feature_matching(s, t, d["fs"], d["ft"])
        return _reg(a), _reg(b)
    add("registration_fgr", global_make, fgr, rng=True)
    return cs


def _odometry_cases():
    cs = []

    def make(seed):
        from tests.synth import camera_pose, render_depth
        a, b = camera_pose(100 + 40 * seed), camera_pose(103 + 40 * seed)
        return dict(t=render_depth(a).numpy(), s=render_depth(b).numpy())

    def multi(e, d, keep):
        odo = e["o3d"].t.pipelines.odometry
        g = e["o3d"].t.geometry
        crit = [odo.OdometryConvergenceCriteria(n) for n in (6, 3, 1)]
        res = odo.rgbd_odometry_multi_scale(g.RGBDImage(None, d["s"]), g.RGBDImage(None, d["t"]), K, np.eye(4),
                                            1000.0, 3.0, crit, odo.Method.PointToPlane)
        return res.transformation, res.inlier_rmse, res.fitness

    def one(e, d, keep):
        odo = e["o3d"].t.pipelines.odometry
        g = e["o3d"].t.geometry
        nan = float("nan")
        maps = []
        for x in (d["s"], d["t"]):
            v = g.Image(x).clip_transform(1000.0, 0.0, 3.0, nan).create_vertex_map(K, nan)
            maps.append(v)
        res = odo.compute_odometry_result_point_to_plane(maps[0], maps[1], maps[1].create_normal_map(nan), K,
                                                         np.eye(4), 0.07, 0.05)
        return res.transformation, res.inlier_rmse, res.fitness
    cs.append(Case("rgbd_odometry_multi_scale", make, multi))
    cs.append(Case("compute_odometry_result_point_to_plane", make, one))
    return cs


VOXEL, RES, TRUNC, SCALE, DMAX = 0.008, 16, 8.0, 1000.0, 3.0


def _frames(seed, n):
    from tests.synth import camera_pose, render_depth
    out = {}
    for i in range(n):
        fid = 100 + i + 300 * seed
        dep, col = render_depth(camera_pose(fid), with_color=True)
        out[f"d{i}"], out[f"c{i}"] = dep.numpy(), col.numpy()
        out[f"E{i}"] = np.linalg.inv(camera_pose(100 + i)).tolist()   # host values: the real frames' poses
    return out


def _volume_cases():
    cs = []
    add = lambda *a, **k: cs.append(Case(*a, **k))   # noqa: E731

    def vbg(e, keep, count=6000):
        g = e["o3d"].t.geometry.VoxelBlockGrid(voxel_size=VOXEL, block_resolution=RES, block_count=count)
        keep.append(g)
        return g

    def state(g):
        idx = g.hashmap().active_buf_indices().long()
        keys = g.hashmap().key_tensor()[idx]
        order = torch.from_numpy(np.lexsort(keys.cpu().numpy().T[::-1]).copy()).cuda()
        idx = idx[order]
        return keys[order], g.attribute("tsdf")[idx], g.attribute("weight").view(torch.int16)[idx], \
            g.attribute("color").view(torch.int16)[idx]

    def integrate(e, d, keep):
        g = vbg(e, keep)
        for i in range(2):
            bc = g.compute_unique_block_coordinates(d[f"d{i}"], K, d[f"E{i}"], SCALE, DMAX, TRUNC)
            g.integrate(bc, d[f"d{i}"], d[f"c{i}"], K, K, d[f"E{i}"], SCALE, DMAX, TRUNC)
        return state(g)
    add("vbg_integrate_device", lambda s: _frames(s, 2), integrate)

    def fused(host):
        def run(e, d, keep):
            g = vbg(e, keep, 64)   # a tiny capacity: the map grows on the device, old buffers go through free_on
            for i in range(3):
                dep, col = d[f"d{i}"], d[f"c{i}"]
                if host:
                    dep, col = dep.cpu().numpy(), col.cpu().numpy()
                g.integrate_frame(dep, col, K, d[f"E{i}"], SCALE, DMAX, TRUNC)
            n = g.hashmap().size()
            frustum = g.last_frustum_block_coordinates().cpu().numpy()   # (in no fixed order, as upstream's)
            return state(g) + (n, frustum[np.lexsort(frustum.T[::-1])])
        return run
    add("vbg_integrate_frame_device_growth", lambda s: _frames(s, 3), fused(False))
    add("vbg_integrate_frame_numpy", lambda s: _frames(s, 3), fused(True))

    def c_abi(e, d, keep):
        """The handle-level calls the Python layer does not reach: sequence, exec stats, estimate_range, hashing,
        the stateless touch / integrate pair, activate / find / reserve."""
        L, st = e["L"], torch.cuda.current_stream().cuda_stream
        g = vbg(e, keep)
        v = g._h
        P = C.c_void_p * 2
        exts = np.ascontiguousarray(np.stack([d["E0"], d["E1"]]).reshape(-1, 16))
        L.check(L.lib.o3db_vbg_integrate_sequence(v, 2, P(d["d0"].data_ptr(), d["d1"].data_ptr()), L.DEPTH_U16,
                                                  P(d["c0"].data_ptr(), d["c1"].data_ptr()), L.COLOR_U8, 480, 640,
                                                  L.dptr(np.ascontiguousarray(K)), L.dptr(exts), SCALE, DMAX, TRUNC,
                                                  0, st))
        ms, launches = np.zeros(1), C.c_int64()
        L.check(L.lib.o3db_vbg_exec_stats(v, L.dptr(ms), C.byref(launches), 1, st))
        keys = g.last_frustum_block_coordinates()
        rng = torch.empty((60, 80, 2), dtype=torch.float32, device="cuda")
        L.check(L.lib.o3db_vbg_estimate_range(v, keys.data_ptr(), keys.shape[0], L.dptr(np.ascontiguousarray(K)),
                                              L.dptr(np.ascontiguousarray(d["E1"])), 480, 640, 8, 0.1, DMAX,
                                              rng.data_ptr(), st))
        hashes = torch.empty((keys.shape[0],), dtype=torch.int64, device="cuda")
        L.check(L.lib.o3db_hash_keys(keys.data_ptr(), keys.shape[0], hashes.data_ptr(), st))
        touch = torch.empty((1 << 16, 3), dtype=torch.int32, device="cuda")
        nt = C.c_int64()
        E0 = np.ascontiguousarray(d["E0"])
        L.check(L.lib.o3db_depth_touch(d["d0"].data_ptr(), L.DEPTH_U16, 480, 640, L.dptr(np.ascontiguousarray(K)),
                                       L.dptr(E0), RES, VOXEL, VOXEL * TRUNC, SCALE, DMAX, 4, touch.data_ptr(),
                                       touch.shape[0], C.byref(nt), st))
        tk = touch[: nt.value]
        order = torch.from_numpy(np.lexsort(tk.cpu().numpy().T[::-1]).copy()).cuda()
        tk = tk[order].contiguous()
        nb = tk.shape[0]
        idx = torch.arange(nb, dtype=torch.int32, device="cuda")
        tsdf = torch.zeros((nb, RES ** 3), dtype=torch.float32, device="cuda")
        wt = torch.zeros((nb, RES ** 3), dtype=torch.uint16, device="cuda")
        col = torch.zeros((nb, RES ** 3, 3), dtype=torch.uint16, device="cuda")
        K9 = np.ascontiguousarray(K)
        L.check(L.lib.o3db_integrate_blocks(d["d0"].data_ptr(), L.DEPTH_U16, d["c0"].data_ptr(), L.COLOR_U8, 480, 640,
                                            idx.data_ptr(), nb, tk.data_ptr(), tsdf.data_ptr(), wt.data_ptr(),
                                            col.data_ptr(), 0, L.dptr(K9), L.dptr(K9), L.dptr(E0), RES, VOXEL,
                                            VOXEL * TRUNC, SCALE, DMAX, st))
        h = g.hashmap()
        h.reserve(h.capacity() + 1000)
        buf, mask = h.activate(tk)
        fbuf, fmask = h.find(tk)
        hashes = np.sort(hashes.cpu().numpy())   # of the frustum keys, which come in no fixed order
        return state(g), launches.value, rng, hashes, tk, tsdf, wt.int(), col.int(), mask, fmask, h.size()
    add("vbg_c_abi", lambda s: _frames(s, 2), c_abi)

    def render(e, d, keep):
        g = vbg(e, keep)
        for i in range(2):
            g.integrate_frame(d[f"d{i}"], d[f"c{i}"], K, d[f"E{i}"], SCALE, DMAX, TRUNC)
        rc = g.ray_cast(None, K, d["E1"], 640, 480, ("depth", "color", "vertex", "normal"), SCALE, 0.1, DMAX, 1.0,
                        TRUNC, 8)
        pc = g.extract_point_cloud(1.0)
        mesh = g.extract_triangle_mesh(1.0)
        return rc, _pts(pc), mesh.vertex, mesh.triangle["indices"]

    def by_position(out):
        """Extraction rows follow the block slots, which the concurrent activation hands out in no fixed order: the
        points sorted by position, the triangles as rows of their vertices' sorted indices, rotated to keep the
        winding."""
        rc, pts, vtx, tri = out
        order = np.lexsort(pts["positions"].cpu().numpy().T[::-1])
        pts = {k: v.cpu().numpy()[order] for k, v in pts.items()}
        vorder = np.lexsort(vtx["positions"].cpu().numpy().T[::-1])
        inv = np.argsort(vorder)
        t = inv[tri.cpu().numpy()]
        t = np.stack([np.roll(r, -int(np.argmin(r))) for r in t]) if len(t) else t
        t = t[np.lexsort(t.T[::-1])] if len(t) else t
        return rc, pts, {k: v.cpu().numpy()[vorder] for k, v in vtx.items()}, t
    add("vbg_ray_cast_and_extract", lambda s: _frames(s, 2), render, key=by_position)
    return cs


def _slam_make(seed):
    from tests.synth import camera_pose, render_depth
    out = {}
    for n in range(7):
        dep, col = render_depth(camera_pose(100 + n + 250 * seed), with_color=True)
        out[f"d{n}"], out[f"c{n}"] = dep.numpy(), col.numpy()
    return out


def _slam_run(e, d, keep):
    """tests/test_odometry_gpu.py::test_dense_slam_loop_vs_oracle's seven-frame loop."""
    from tests.synth import camera_pose
    slam = e["o3d"].t.pipelines.slam
    model = slam.Model(VOXEL, RES, 12000, camera_pose(100))
    keep.append(model)
    pose, poses = camera_pose(100).copy(), []
    raycast_frame = slam.Frame(480, 640, K)
    for n in range(7):
        frame = slam.Frame(480, 640, K)
        frame.set_data("depth", d[f"d{n}"])
        frame.set_data("color", d[f"c{n}"])
        if n > 0:
            res = model.track_frame_to_model(frame, raycast_frame, SCALE, DMAX, 0.07)
            pose = pose @ res.transformation
        poses.append(pose.copy())
        model.update_frame_pose(n, pose)
        model.integrate(frame, SCALE, DMAX, TRUNC)
        model.synthesize_model_frame(raycast_frame, SCALE, 0.1, DMAX, TRUNC, False)
    return np.stack(poses), raycast_frame.get_data("depth")


def _search_cases():
    cs = []
    for dtype in (torch.int32, torch.int64):
        def knn(e, d, keep, dtype=dtype):
            nns = e["o3d"].core.nns.NearestNeighborSearch(d["p"], dtype)
            nns.knn_index()
            a = nns.knn_search(d["s"], 12)
            nns.hybrid_index(0.05)
            return a, nns.hybrid_search(d["s"], 0.05, 12)
        cs.append(Case(f"nns_search_{str(dtype)[6:]}", _pc, knn))
    return cs


CASES = {c.name: c for c in (_point_cloud_cases() + _image_cases() + _registration_cases() + _odometry_cases() +
                             _volume_cases() + _search_cases() + [Case("slam_loop", _slam_make, _slam_run)])}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_side_stream_matches_default_stream(env, name):
    case = CASES[name]
    real = case.make(0)
    ref, keep = default_run(env, case, real)
    dec, keep2 = default_run(env, case, case.make(1))
    assert not _same(ref, dec), f"{name}: the decoy gives the real inputs' result, so it could detect nothing"
    if case.atol:
        assert any(x.dtype.kind == "f" and x.shape == y.shape and np.abs(x - y).max() > case.atol
                   for x, y in zip(_leaves(ref), _leaves(dec))), f"{name}: the decoy is within the tolerance"
    del keep, keep2
    gc.collect()
    spy = env["spy"]
    n_wrong = len(spy.wrong)
    got, keep = side_run(env, case, real)
    assert spy.wrong[n_wrong:] == [], f"{name}: calls inside the side-stream run were given another stream"
    la, lb = _leaves(got), _leaves(ref)
    assert len(la) == len(lb)
    for i, (x, y) in enumerate(zip(la, lb)):
        assert x.shape == y.shape and x.dtype == y.dtype, f"{name}: output {i} {x.shape} {x.dtype} vs {y.shape} {y.dtype}"
        if case.ulps and x.dtype == np.float32:
            np.testing.assert_array_max_ulp(x, y, case.ulps)
            continue
        if case.atol and x.dtype.kind == "f":
            np.testing.assert_allclose(x, y, rtol=0, atol=case.atol, err_msg=f"{name}: output {i}")
            continue
        assert np.ascontiguousarray(x).tobytes() == np.ascontiguousarray(y).tobytes(), \
            f"{name}: output {i} differs on the side stream"
    del keep
    gc.collect()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_calls_never_synchronise_the_device(env, name):
    """A call that returns host values synchronises its own stream only: an event behind a long sleep on another
    non-blocking stream is still pending when the call returns."""
    case, busy, side = CASES[name], env["busy"], env["side"]
    real = case.make(0)
    default_run(env, case, real)                    # warm up: lazy module loading may synchronise on a first launch
    inputs = _device(real)
    gc.collect()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    keep = []
    with torch.cuda.stream(side):
        case(env, inputs, keep)
    side.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    gc.collect()
    torch.cuda.synchronize()
    done = torch.cuda.Event()
    with torch.cuda.stream(busy):
        torch.cuda._sleep(int(max(200.0, 20 * ms) * env["per_ms"]))
        done.record()
    keep2 = []
    with torch.cuda.stream(side):
        case(env, inputs, keep2)
        pending = not done.query()
    side.synchronize()
    busy.synchronize()
    del keep, keep2
    gc.collect()
    assert pending, f"{name} waited for another stream's work: it synchronised the device"


# ------------------------------------------------------------------------------------------------ oracles

@pytest.mark.gpu
def test_side_stream_knn_search_vs_oracle(env):
    from oracle import knn as ok
    d = _pc(0)
    out, _ = side_run(env, CASES["nns_search_int64"], d)
    idx, d2 = ok.knn(d["p"], d["s"], 12)
    assert np.array_equal(out[0][0].cpu().numpy(), idx) and np.array_equal(out[0][1].cpu().numpy(), d2)


@pytest.mark.gpu
def test_side_stream_icp_vs_oracle(env):
    import oracle
    d = _pair(0)
    out, _ = side_run(env, CASES["icp_plane"], d)
    ref = oracle.icp_p2plane(d["s"], d["t"], d["tn"], 0.05, max_iteration=12, relative_fitness=0, relative_rmse=0)
    T, corr, fitness, rmse = out[0], out[1].cpu().numpy(), out[2], out[3]
    np.testing.assert_allclose(T, ref.transformation, atol=2e-5)
    assert abs(fitness - ref.fitness) < 2e-4 and abs(rmse - ref.inlier_rmse) < 2e-6
    assert (corr == ref.correspondences).mean() > 0.999


@pytest.mark.gpu
def test_side_stream_slam_loop_vs_oracle(env):
    from tests.test_odometry_gpu import _oracle_slam
    out, _ = side_run(env, CASES["slam_loop"], _slam_make(0))
    for n, (p, q) in enumerate(zip(out[0], _oracle_slam(list(range(100, 107))))):
        np.testing.assert_allclose(p, q, atol=1e-4, err_msg=f"frame {n}")


# ------------------------------------------------------------------------------------------------ handles

@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
def test_index_built_on_one_stream_searched_on_another(env, dtype):
    """Built on stream A, searched on stream B with no synchronisation by the caller.  The window this checks, the
    tail of create still queued on A (the counting sort and the block flags), is short and the test cannot hold it
    open; that the search waits for it is checked by reading o3db_knn_search / o3db_nns_hybrid_search."""
    import oracle
    from oracle import knn as ok
    o3d, side = env["o3d"], env["side"]
    d = _device(_pc(0))
    a = torch.cuda.Stream()
    torch.cuda.synchronize()
    nns = o3d.core.nns.NearestNeighborSearch(d["p"], dtype)
    with torch.cuda.stream(a):
        nns.knn_index()
        nns.hybrid_index(0.05)
    with torch.cuda.stream(side):
        idx, d2 = nns.knn_search(d["s"], 12)
        hi, hd, hc = nns.hybrid_search(d["s"], 0.05, 12)
    side.synchronize()
    p, s = d["p"].cpu().numpy(), d["s"].cpu().numpy()
    oi, od = ok.knn(p, s, 12)
    assert np.array_equal(idx.cpu().numpy(), oi) and np.array_equal(d2.cpu().numpy(), od)
    wi, wd, wc = oracle.hybrid_search(p, s, 0.05, 12)
    assert np.array_equal(hi.cpu().numpy(), wi) and np.array_equal(hd.cpu().numpy(), wd)
    assert np.array_equal(hc.cpu().numpy(), wc)
    del nns
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_index_freed_while_a_search_on_another_stream_is_queued(env):
    """Each index is destroyed and rebuilt over a permutation of the same points while a search on the side stream
    still waits behind a sleep.  Destroy drains the creation stream (the default stream here) and frees the index's
    buffers on it; only the `used` event of the search, which the creation stream waits on, orders that drain after
    the search.  Without it the drain returns at once, the frees hand the blocks back to the pool in the default
    stream's order, and the rebuild's allocations of the same sizes on that stream take them back and fill them with
    the permuted index (each sorted point carries its dataset index) before the sleep ends: the search then returns
    indices in the permuted numbering.  The old handle is released before its successor is built, so that the
    successor is the only index of that layout the freed blocks can go to: the same count and bounding box give the
    same grid, and every read stays in bounds."""
    from oracle import knn as ok
    import oracle
    o3d, side = env["o3d"], env["side"]
    d = _pc(0)
    p, q = torch.from_numpy(d["p"]).cuda(), torch.from_numpy(d["s"]).cuda()
    perm = torch.from_numpy(np.random.default_rng(3).permutation(len(d["p"]))).cuda()
    p_perm = p[perm].contiguous()
    nns = o3d.core.nns.NearestNeighborSearch(p)
    nns.knn_index()
    nns.hybrid_index(0.05)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(int(100 * env["per_ms"]))
        idx, d2 = nns.knn_search(q, 8)
        hi, hd, hc = nns.hybrid_search(q, 0.05, 8)
    nns.dataset_points = p_perm
    nns._knn = None            # destroys the first KNN index
    nns.knn_index()
    nns._hybrid = None         # and the first hybrid index
    nns.hybrid_index(0.05)
    side.synchronize()
    torch.cuda.synchronize()
    oi, od = ok.knn(d["p"], d["s"], 8)
    assert np.array_equal(idx.cpu().numpy(), oi) and np.array_equal(d2.cpu().numpy(), od)
    wi, wd, wc = oracle.hybrid_search(d["p"], d["s"], 0.05, 8)
    assert np.array_equal(hi.cpu().numpy(), wi) and np.array_equal(hd.cpu().numpy(), wd)
    assert np.array_equal(hc.cpu().numpy(), wc)


def _icp_handle(env, d, stream):
    L = env["L"]
    opt = L.IcpOptions(0.05, 10, 0.0, 0.0, L.RobustKernel(0, 1.0, 1.0), 0.0)
    h = C.c_void_p()
    L.check(L.lib.o3db_icp_create(d["s"].data_ptr(), d["s"].shape[0], d["t"].data_ptr(), d["tn"].data_ptr(),
                                  d["t"].shape[0], L.dptr(np.eye(4)), C.byref(opt), None, stream, C.byref(h)))
    return h


def _icp_finish(env, h, corr, stream):
    """o3db_icp_finish on `stream` into the caller's corr: no other synchronisation, the call synchronises `stream`."""
    L = env["L"]
    res, per = L.IcpResult(), np.zeros(20)
    L.check(L.lib.o3db_icp_finish(h, C.byref(res), corr.data_ptr(), L.dptr(per), stream))
    return np.array(res.transformation), res.fitness, res.inlier_rmse, res.num_iterations, corr.cpu().numpy(), per


def _icp_want(env, d, corr):
    """All on one stream: create, 10 iterations, finish."""
    L = env["L"]
    a = torch.cuda.Stream()
    torch.cuda.synchronize()
    h = _icp_handle(env, d, int(a.cuda_stream))
    L.check(L.lib.o3db_icp_iterate(h, 10, int(a.cuda_stream)))
    want = _icp_finish(env, h, corr, int(a.cuda_stream))
    L.lib.o3db_icp_destroy(h)
    assert want[3] == 10
    return want


@pytest.mark.gpu
def test_icp_handle_iterated_on_another_stream_than_created(env):
    """The point-to-plane handle through the C ABI, created on stream A and at once iterated and finished on stream B,
    gives the all-on-A result bit for bit: only the handle orders B after the tail of create still queued on A (the
    source sort and gather, the initial state).  That window is short and this test cannot hold it open; that the
    iterate waits for A is checked by reading o3db_icp_iterate."""
    L, side = env["L"], env["side"]
    d = _device(_pair(0))
    n = d["s"].shape[0]
    corr = [torch.empty((n,), dtype=torch.int64, device="cuda") for _ in range(2)]
    want = _icp_want(env, d, corr[0])
    a = torch.cuda.Stream()
    torch.cuda.synchronize()
    h = _icp_handle(env, d, int(a.cuda_stream))
    L.check(L.lib.o3db_icp_iterate(h, 10, int(side.cuda_stream)))
    got = _icp_finish(env, h, corr[1], int(side.cuda_stream))
    L.lib.o3db_icp_destroy(h)
    assert _same(got, want)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_icp_handle_finished_on_its_stream_after_iterations_on_another(env):
    """The point-to-plane handle through the C ABI, created on stream A, reset on stream B, iterated on B behind a
    100 ms sleep and finished on A, gives the all-on-A result bit for bit.  Nothing between the iterate and the finish
    synchronises anything, so the finish is queued on A while B still sleeps: without the `used` event that makes A
    wait for the iterations on B, it evaluates the state the reset left (no iteration, the initial transformation) and
    reports that.  (The synchronisations of A after create and of B after the reset only keep those steps out of the
    ordering under test.)"""
    L, side = env["L"], env["side"]
    d = _device(_pair(0))
    n = d["s"].shape[0]
    corr = [torch.empty((n,), dtype=torch.int64, device="cuda") for _ in range(2)]
    want = _icp_want(env, d, corr[0])
    a = torch.cuda.Stream()
    A, B = int(a.cuda_stream), int(side.cuda_stream)
    torch.cuda.synchronize()
    h = _icp_handle(env, d, A)
    a.synchronize()
    L.check(L.lib.o3db_icp_reset(h, B))
    side.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(int(100 * env["per_ms"]))
    L.check(L.lib.o3db_icp_iterate(h, 10, B))
    got = _icp_finish(env, h, corr[1], A)
    side.synchronize()          # (so that destroy below never frees what B still reads, fixed or not)
    L.lib.o3db_icp_destroy(h)
    assert got[3] == 10, f"the finish on A ran after {got[3]} iterations: it did not wait for the iterations on B"
    assert _same(got, want)
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_zz_side_runs_covered_every_entry_point(env):
    """Runs after the cases above (file order): every header entry point with a stream, but the exclusions, was
    called inside a side-stream run, and always with the side stream.  Skipped when this session did not run every
    case on the side stream (a -k selection, deselection, another order), since the coverage is then unknown."""
    spy = env["spy"]
    assert spy.wrong == []
    not_run = sorted(set(CASES) - spy.cases_run)
    if not_run:
        pytest.skip(f"{len(not_run)} side-stream cases did not run in this session, e.g. {not_run[0]}")
    missing = sorted(set(spy.eps) - set(EXCLUDED) - spy.side_calls)
    assert not missing, f"never called on the side stream: {missing}"

"""Sum replay of the fused ICP iteration: a 32-query chunk whose points the pending update leaves bit-for-bit where
they were adds the 32 sums it stored in the previous iteration instead of computing them again.

The evaluation pass (o3db_icp_finish) moves the points and invalidates those lines, so `iterate(k); finish;
iterate(24 - k); finish` recomputes every chunk in iteration k + 1, where `iterate(24); finish` replays the unmoved
ones.  Both must give the same bits.  The clouds have more than three chunk rows and a partial last row, as in
test_icp_sweep_gpu.py, and 24 iterations leave them well aligned, so that most chunks replay.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.synth import make_colors, make_icp_pair

pytestmark = pytest.mark.gpu

THREADS = 768   # kIcpThreads: one block per SM
ITERS = 24


def _cloud_points():
    row = torch.cuda.get_device_properties(0).multi_processor_count * THREADS
    return 3 * row + row // 3


@pytest.fixture(scope="module")
def L():
    import open3d_b200  # noqa: F401
    from open3d_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


def _create(L, kind, stream):
    """A handle on the bench's kind of pair: point-to-plane (L2 or Tukey) or ColoredICP."""
    src, tgt, nrm, T_gt = make_icp_pair(_cloud_points(), seed=5)
    n = len(src)
    keep = [torch.from_numpy(a).cuda() for a in (src, tgt, nrm)]
    opt = L.IcpOptions()
    opt.max_correspondence_distance, opt.max_iteration = 0.05, ITERS
    opt.relative_fitness = opt.relative_rmse = 0.0
    opt.kernel = L.RobustKernel(5, 0.05, 1.0) if kind == "tukey" else L.RobustKernel(0, 1.0, 1.0)
    h = C.c_void_p()
    if kind == "colored":
        rng = np.random.default_rng(3)
        world = (src.astype(np.float64) @ T_gt[:3, :3].T + T_gt[:3, 3]).astype(np.float32)
        extra = [make_colors(world, 1), make_colors(tgt, 1), rng.normal(0, 0.05, tgt.shape).astype(np.float32)]
        sc, tc, grad = [torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in extra]
        keep += [sc, tc, grad]
        L.check(L.lib.o3db_icp_create_colored(keep[0].data_ptr(), sc.data_ptr(), n, keep[1].data_ptr(),
                                              keep[2].data_ptr(), tc.data_ptr(), grad.data_ptr(), len(tgt),
                                              L.dptr(np.eye(4)), C.byref(opt), 0.968, None, stream, C.byref(h)))
    else:
        L.check(L.lib.o3db_icp_create(keep[0].data_ptr(), n, keep[1].data_ptr(), keep[2].data_ptr(), len(tgt),
                                      L.dptr(np.eye(4)), C.byref(opt), None, stream, C.byref(h)))
    return h, n, keep


def _finish(L, h, n, stream):
    res = L.IcpResult()
    corr = torch.full((n,), -7, dtype=torch.int64, device="cuda")
    per = np.zeros((ITERS, 2))
    L.check(L.lib.o3db_icp_finish(h, C.byref(res), corr.data_ptr(), L.dptr(per), stream))
    torch.cuda.synchronize()
    return np.array(res.transformation), res.fitness, res.inlier_rmse, res.num_iterations, corr.cpu().numpy(), per


def _register(L, h, n, batches, stream):
    """o3db_icp_reset, then o3db_icp_iterate followed by o3db_icp_finish for each entry of `batches`."""
    L.check(L.lib.o3db_icp_reset(h, stream))
    for k in batches:
        L.check(L.lib.o3db_icp_iterate(h, k, stream))
        out = _finish(L, h, n, stream)
    return out


def _assert_same_bits(a, b):
    assert a[0].tobytes() == b[0].tobytes()
    assert a[1] == b[1] and a[2] == b[2] and a[3] == b[3]
    assert np.array_equal(a[4], b[4])
    assert a[5].tobytes() == b[5].tobytes()


@pytest.mark.parametrize("kind", ["p2plane", "colored", "tukey"])
def test_replayed_sums_equal_recomputed_sums(L, kind):
    stream = int(torch.cuda.current_stream().cuda_stream)
    h, n, _keep = _create(L, kind, stream)
    try:
        straight = _register(L, h, n, [ITERS], stream)
        split = {k: _register(L, h, n, [k, ITERS - k], stream) for k in (6, 12, 18)}
    finally:
        L.lib.o3db_icp_destroy(h)
    assert straight[3] == ITERS and straight[1] > 0.9
    for k, other in split.items():
        _assert_same_bits(straight, other)


def test_reset_invalidates_cached_sums(L):
    """A registration left unfinished keeps its cached lines valid; o3db_icp_reset gathers the source again, so the
    next registration must recompute every chunk in its first iteration (the identity update moves no point)."""
    stream = int(torch.cuda.current_stream().cuda_stream)
    h, n, _keep = _create(L, "p2plane", stream)
    try:
        first = _register(L, h, n, [ITERS], stream)
        L.check(L.lib.o3db_icp_reset(h, stream))
        L.check(L.lib.o3db_icp_iterate(h, ITERS, stream))
        second = _register(L, h, n, [ITERS], stream)
    finally:
        L.lib.o3db_icp_destroy(h)
    assert first[3] == ITERS and first[1] > 0.9
    _assert_same_bits(first, second)

"""The fused ICP iteration walks each warp's chunks forward after an even number of iterations and backward after an
odd one.  A warp owns one chunk per row of grid-size x 768 points (101 376 on a 132-SM H100), so the order only
matters on clouds of several rows; these tests use more than three rows and a partial last row, which some warps
reach and others do not.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.synth import make_icp_pair
from tests.test_icp_gpu import test_icp_loop_vs_oracle as _loop_vs_oracle

pytestmark = pytest.mark.gpu

THREADS = 768   # kIcpThreads: one block per SM


def _row():
    return torch.cuda.get_device_properties(0).multi_processor_count * THREADS


def _cloud_points():
    """A point count of more than three rows that is not a whole number of rows."""
    row = _row()
    return 3 * row + row // 3


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


@pytest.mark.parametrize("iters", [5, 6])
def test_icp_loop_vs_oracle_several_rows(o3d, iters):
    """The bars of test_icp_loop_vs_oracle, on a cloud where warps walk several chunks in both directions; an odd
    count ends on a backward iteration, so the evaluation pass walks forward, an even count the other way round."""
    n = _cloud_points()
    src = make_icp_pair(n, seed=1)[0]
    row = _row()
    assert len(src) > 3 * row and len(src) % row != 0
    _loop_vs_oracle(o3d, n, iters)


def _register(L, h, batches, n, stream):
    """o3db_icp_reset, then one o3db_icp_iterate per entry of `batches` and o3db_icp_finish."""
    L.check(L.lib.o3db_icp_reset(h, stream))
    for k in batches:
        L.check(L.lib.o3db_icp_iterate(h, k, stream))
    res = L.IcpResult()
    corr = torch.full((n,), -7, dtype=torch.int64, device="cuda")
    per = np.zeros((sum(batches), 2))
    L.check(L.lib.o3db_icp_finish(h, C.byref(res), corr.data_ptr(), L.dptr(per), stream))
    torch.cuda.synchronize()
    return np.array(res.transformation), res.fitness, res.inlier_rmse, res.num_iterations, corr.cpu().numpy(), per


@pytest.mark.parametrize("iters", [7, 8])
def test_icp_iterate_batching_gives_identical_bits(o3d, iters):
    """The sweep direction comes from device state, so one launch per o3db_icp_iterate call and all launches in one
    call give the same bits, and o3db_icp_reset starts the sequence over."""
    from open3d_b200 import _lib as L
    stream = int(torch.cuda.current_stream().cuda_stream)
    src, tgt, nrm, _ = make_icp_pair(_cloud_points(), seed=4)
    n = len(src)
    d = [torch.from_numpy(a).cuda() for a in (src, tgt, nrm)]
    opt = L.IcpOptions()
    opt.max_correspondence_distance, opt.max_iteration = 0.05, iters
    opt.relative_fitness = opt.relative_rmse = 0.0
    opt.kernel = L.RobustKernel(0, 1.0, 1.0)
    h = C.c_void_p()
    L.check(L.lib.o3db_icp_create(d[0].data_ptr(), n, d[1].data_ptr(), d[2].data_ptr(), len(tgt),
                                  L.dptr(np.eye(4)), C.byref(opt), None, stream, C.byref(h)))
    try:
        one_by_one = _register(L, h, [1] * iters, n, stream)
        at_once = _register(L, h, [iters], n, stream)
        split = _register(L, h, [3, iters - 3], n, stream)
    finally:
        L.lib.o3db_icp_destroy(h)
    assert one_by_one[3] == iters and one_by_one[1] > 0.9
    for other in (at_once, split):
        assert one_by_one[0].tobytes() == other[0].tobytes()
        assert one_by_one[1] == other[1] and one_by_one[2] == other[2] and one_by_one[3] == other[3]
        assert np.array_equal(one_by_one[4], other[4])
        assert one_by_one[5].tobytes() == other[5].tobytes()

"""torchrun --nproc-per-node N tests/multigpu_p2p_check.py
N-rank check of the source-sharded point-to-point ICP: the raw moments about the shared pivot add over the ranks like
the point-to-plane sums do, so the sharded result must equal the single-GPU result on the whole source, and every rank
must hold the identical transformation."""
import ctypes as C
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from open3d_b200 import _lib as L  # noqa: E402
from open3d_b200.distributed import Communicator, shard_range  # noqa: E402
from tests.synth import make_icp_pair  # noqa: E402


def run(src, tgt, iters, comm):
    stream = int(torch.cuda.current_stream().cuda_stream)
    d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (src, tgt)]
    opt = L.IcpOptions()
    opt.max_correspondence_distance, opt.max_iteration = 0.05, iters
    opt.relative_fitness = opt.relative_rmse = 0.0
    opt.kernel = L.RobustKernel(0, 1.0, 1.0)
    h = C.c_void_p()
    L.check(L.lib.o3db_icp_create_point_to_point(d[0].data_ptr(), len(src), d[1].data_ptr(), len(tgt), L.dptr(np.eye(4)),
                                                 C.byref(opt), comm.handle if comm else None, stream, C.byref(h)))
    L.check(L.lib.o3db_icp_iterate(h, iters, stream))
    res = L.IcpResult()
    per = np.zeros((iters, 2))
    L.check(L.lib.o3db_icp_finish(h, C.byref(res), None, L.dptr(per), stream))
    L.lib.o3db_icp_destroy(h)
    return np.array(res.transformation).reshape(4, 4), res.fitness, res.inlier_rmse, per


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
    comm = Communicator(rank, world)
    src, tgt, _, _ = make_icp_pair(400_000, seed=5)
    b, e = shard_range(len(src), rank, world)
    T, fit, rmse, per = run(src[b:e], tgt, 10, comm)
    t = torch.from_numpy(T).cuda()
    ref = t.clone()
    dist.broadcast(ref, src=0)
    assert torch.equal(t, ref), "ranks disagree on the transformation"
    if rank == 0:
        T1, fit1, rmse1, per1 = run(src, tgt, 10, None)
        np.testing.assert_allclose(T, T1, atol=1e-9)
        np.testing.assert_allclose(per, per1, atol=1e-9)
        assert abs(fit - fit1) < 1e-12 and abs(rmse - rmse1) < 1e-9
        print(f"multigpu_p2p_check ok: world={world} fitness={fit:.6f} rmse={rmse:.6f} "
              f"|T - T_single|max={np.abs(T - T1).max():.2e}")
    comm.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

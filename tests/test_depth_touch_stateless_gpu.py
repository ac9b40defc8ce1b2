"""The stateless o3db_depth_touch, which the reference-facing forwarders call (integration/o3d_forwarders.cpp), against
the CPU oracle on the frames test_tsdf_gpu.py sends through the grid's GetUniqueBlockCoordinates: the same block set,
bit for bit, without the reference build."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from tests.synth import PRIMESENSE_K, camera_pose, render_depth

pytestmark = pytest.mark.gpu

VOXEL, RES, TRUNC_MULT = 0.008, 16, 8.0
SCALE, DMAX = 1000.0, 3.0


def _sorted_keys(k):
    k = np.asarray(k, np.int32).reshape(-1, 3)
    return k[np.lexsort((k[:, 2], k[:, 1], k[:, 0]))]


@pytest.mark.parametrize("frame_id,f32", [(0, False), (137, False), (500, True)])
def test_stateless_depth_touch_block_set_bit_exact(frame_id, f32):
    from open3d_b200 import _lib as L
    T = camera_pose(frame_id)
    E = np.ascontiguousarray(oracle.inverse_transformation(T), np.float64)
    depth = render_depth(T).numpy()
    if f32:
        depth = depth.astype(np.float32)
    K9 = np.ascontiguousarray(PRIMESENSE_K, np.float64)
    d = torch.from_numpy(depth).cuda()
    out = torch.empty((1 << 16, 3), dtype=torch.int32, device="cuda")
    n = C.c_int64()
    stream = int(torch.cuda.current_stream().cuda_stream)
    L.check(L.lib.o3db_depth_touch(d.data_ptr(), L.DEPTH_F32 if f32 else L.DEPTH_U16, 480, 640, L.dptr(K9), L.dptr(E),
                                   RES, VOXEL, VOXEL * TRUNC_MULT, SCALE, DMAX, 4, out.data_ptr(), out.shape[0],
                                   C.byref(n), stream))
    torch.cuda.synchronize()
    got = out[:n.value].cpu().numpy()
    want = oracle.depth_touch(depth, PRIMESENSE_K, E, RES, VOXEL, VOXEL * TRUNC_MULT, SCALE, DMAX, 4)
    assert len(got) == len(want) > 100
    assert len(np.unique(got, axis=0)) == len(got)          # unique
    assert np.array_equal(_sorted_keys(got), want)          # identical set, bit for bit

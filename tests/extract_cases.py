"""Hand-built voxel block volumes for the point-cloud extraction tests (CPU and GPU): each one isolates an edge of
ExtractPointCloud (t/geometry/kernel/VoxelBlockGridImpl.h:1122-1381) that a volume fused from depth frames reaches
only by chance.  Buffers use the slam::Model layout: keys [n,3] int32, tsdf [n,R^3] f32, weight [n,R^3] u16,
colour [n,R^3,3] u16, voxel (x, y, z) of a block at (z*R + y)*R + x."""
import numpy as np

KINDS = ("plane_face", "plane_no_neighbour", "zero_tsdf", "weight_at_threshold", "subnormal")
THRESHOLD = 3.0


def _grid(R):
    z, y, x = np.meshgrid(np.arange(R), np.arange(R), np.arange(R), indexing="ij")
    return x.reshape(-1), y.reshape(-1), z.reshape(-1)


def edge_volume(kind, R=8, with_color=True, seed=0):
    """-> dict(keys, tsdf, weight, color or None) for one of KINDS at block resolution R."""
    rng = np.random.default_rng(seed)
    if kind == "plane_no_neighbour":
        keys = np.array([[0, 0, 0], [0, 1, 0]], np.int32)
    else:
        keys = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.int32)
    n = len(keys)
    x, y, z = _grid(R)
    tsdf = np.empty((n, R ** 3), np.float32)
    weight = np.full((n, R ** 3), 5, np.uint16)
    for b, k in enumerate(keys):
        gx, gy, gz = x + k[0] * R, y + k[1] * R, z + k[2] * R
        if kind in ("plane_face", "plane_no_neighbour"):
            # a tilted plane: inside block 0 and, for y = R-1, between its voxel R-1 and voxel 0 of block 1
            d = (R - 0.55) + 0.45 * (gy - R + 1) - 0.05 * gz - gx
        else:
            d = (R / 2 + 0.3) + 0.11 * gy + 0.09 * gz - gx
        tsdf[b] = np.clip(d * 0.1, -1.0, 1.0).astype(np.float32)
    if kind == "zero_tsdf":
        # exact zeros (both signs) on a crossing: tsdf_i * tsdf_o == 0 is not < 0, so no point from these pairs
        sel = (x == R // 2) & (y % 2 == 0)
        tsdf[0, sel] = 0.0
        tsdf[1, sel & (z % 3 == 0)] = -0.0
    if kind == "weight_at_threshold":
        # weight == threshold is excluded (weight_o <= threshold, weight_i > threshold)
        weight[0, (x + y + z) % 3 == 0] = int(THRESHOLD)
        weight[2, (x + 2 * y) % 4 == 1] = int(THRESHOLD)
        weight[1, y % 5 == 0] = int(THRESHOLD) + 1
    if kind == "subnormal":
        # tsdf_o subnormal: the product, the ratio and the interpolated normal stay subnormal; a flush to zero
        # drops these points or changes their bits
        tsdf[:] = 0.3
        o = (2 * R + 2) * R + 2 if R > 3 else 0
        tsdf[0, o] = np.float32(-1e-40)
        tsdf[1, R ** 3 // 2] = np.float32(-3e-39)
    color = None
    if with_color:
        color = rng.integers(0, 65536, size=(n, R ** 3, 3)).astype(np.uint16)
    return dict(keys=keys, tsdf=tsdf, weight=weight, color=color)

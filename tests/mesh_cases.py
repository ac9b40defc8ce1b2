"""Hand-built voxel block volumes for the triangle-mesh extraction tests (CPU and GPU), in the layout of
tests/extract_cases.py.  Each isolates an edge of ExtractTriangleMesh (VoxelBlockGridImpl.h:1385-1780) that a fused
volume reaches only by chance."""
import numpy as np

from tests.extract_cases import _grid, edge_volume

THRESHOLD = 3.0
# blocks around block (0, 0, 0): the surface crosses each of its faces, with every -/+ neighbour present or absent
NEIGHBOURS = {
    "all": [[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [1, 1, 0], [1, 0, 1],
            [0, 1, 1], [1, 1, 1], [-1, -1, 0], [-1, 0, -1], [0, -1, -1]],
    "plus_only": [[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 1]],
    "minus_only": [[0, 0, 0], [-1, 0, 0], [0, -1, 0], [0, 0, -1]],
    "alone": [[0, 0, 0]],
}
KINDS = ("random_signs", "sphere_all", "sphere_plus_only", "sphere_minus_only", "sphere_alone", "zero_and_minus_zero",
         "subnormal", "weight_at_threshold")


def mesh_volume(kind, R=8, with_color=True, seed=0):
    """-> dict(keys, tsdf, weight, color or None) for one of KINDS at block resolution R."""
    rng = np.random.default_rng(seed)
    if kind == "random_signs":
        # 8 blocks of random signs and magnitudes: every one of the 256 cases occurs (asserted by the tests)
        keys = np.array([[x, y, z] for z in (0, 1) for y in (0, 1) for x in (0, 1)], np.int32)
        tsdf = (rng.choice([-1.0, 1.0], size=(len(keys), R ** 3)) * rng.uniform(0.05, 1.0, (len(keys), R ** 3)))
        tsdf = tsdf.astype(np.float32)
        weight = rng.integers(4, 60, size=(len(keys), R ** 3)).astype(np.uint16)
    elif kind.startswith("sphere_"):
        keys = np.array(NEIGHBOURS[kind[len("sphere_"):]], np.int32)
        x, y, z = _grid(R)
        tsdf = np.empty((len(keys), R ** 3), np.float32)
        for b, k in enumerate(keys):
            g = np.stack([x + k[0] * R, y + k[1] * R, z + k[2] * R], 1).astype(np.float64) + 0.5
            c = np.array([R * 0.45, R * 0.55, R * 0.5])
            tsdf[b] = np.clip((np.linalg.norm(g - c, axis=1) - R * 0.62) * 0.2, -1, 1)
        weight = np.full((len(keys), R ** 3), 7, np.uint16)
    else:
        base = {"zero_and_minus_zero": "zero_tsdf", "subnormal": "subnormal",
                "weight_at_threshold": "weight_at_threshold"}[kind]
        v = edge_volume(base, R, with_color, seed)
        tsdf, weight, keys = v["tsdf"], v["weight"], v["keys"]
        if kind == "zero_and_minus_zero":
            # a corner at exactly 0 next to a negative one: a vertex at ratio 0 (the point cloud has no point there)
            x, y, z = _grid(R)
            tsdf[2, (x == R // 2 + 1) & (z % 2 == 1)] = -0.0
            tsdf[0, (x + y + z) % 7 == 0] = 0.0
        if kind == "subnormal":
            tsdf[2, 5 % R ** 3] = np.float32(1e-41)
    color = rng.integers(0, 65536, size=(len(keys), R ** 3, 3)).astype(np.uint16) if with_color else None
    return dict(keys=keys, tsdf=tsdf, weight=weight, color=color)


CORNERS = ((0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1))


def cube_cases(keys, tsdf, weight, R, threshold=THRESHOLD):
    """[size, R^3] case of the cube at each voxel (bit k: corner k has tsdf < 0), -1 where the cube does not
    contribute (a corner missing or of weight <= threshold); computed directly in numpy."""
    keys = np.asarray(keys).reshape(-1, 3)
    size = len(keys)
    slot = {tuple(k): i for i, k in enumerate(keys.tolist())}
    nb = np.array([[slot.get((k[0] + d % 3 - 1, k[1] + (d % 9) // 3 - 1, k[2] + d // 9 - 1), -1) for d in range(27)]
                   for k in keys.tolist()], np.int64).reshape(size, 27)
    x, y, z = _grid(R)
    t, w = np.asarray(tsdf).reshape(-1), np.asarray(weight).reshape(-1).astype(np.float32)
    case = np.zeros((size, R ** 3), np.int64)
    ok = np.ones((size, R ** 3), bool)
    for ci, (dx, dy, dz) in enumerate(CORNERS):
        gx, gy, gz = x + dx, y + dy, z + dz
        bx, by, bz = gx // R, gy // R, gz // R
        s = nb[:, 13 + bx + 3 * by + 9 * bz]
        lin = s * R ** 3 + ((gz - bz * R) * R + gy - by * R) * R + gx - bx * R
        valid = s >= 0
        lin = np.where(valid, lin, 0)
        ok &= valid & ~(w[lin] <= np.float32(threshold))
        case |= (t[lin] < 0).astype(np.int64) << ci
    return np.where(ok, case, -1)


def case_histogram(v, R, threshold=THRESHOLD):
    """Counts of each contributing cube case in the volume."""
    c = cube_cases(v["keys"], v["tsdf"], v["weight"], R, threshold)
    return np.bincount(c[c >= 0], minlength=256)

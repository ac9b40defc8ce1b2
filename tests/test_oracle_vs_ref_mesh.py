"""The oracle's triangle-mesh extraction and case table against the reference's OWN ExtractTriangleMeshCPU<float,
uint16_t, uint16_t> and tri_table (compiled unmodified into oracle/_ref/libo3dref_mesh.so by oracle/ref_shim_mesh), and
the oracle's mesh of a fused room against the room's analytic geometry.  CPU only.

Each case's surface is fixed by the face rule (mesh_oracle.c); only the diagonals that split its polygons may differ
from upstream's table, so triangles are compared as the oriented boundary cycles of each cube's patches."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle.mesh as mesh_oracle
from tests.mesh_cases import KINDS, THRESHOLD, case_histogram, cube_cases, mesh_volume
from tests.synth import ROOM_MAX, ROOM_MIN, SPHERE_C, SPHERE_R
from tests.test_oracle_vs_ref_extract import VOXEL, fuse_room

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libo3dref_mesh.so")
needs_ref = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref not built (needs the reference sources)")
vp = C.c_void_p


@pytest.fixture(scope="module")
def ref():
    L = C.CDLL(REF)
    L.ref_extract_triangle_mesh.restype = C.c_int64
    L.ref_extract_triangle_mesh.argtypes = [vp, C.c_int64, vp, vp, vp, C.c_int, C.c_float, C.c_float, C.c_int,
                                            C.c_int64, C.c_int64, vp, vp, vp, vp, C.POINTER(C.c_int64)]
    L.ref_mc_table_row.argtypes = [C.c_int, vp, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    return L


def reference_mesh(ref, keys, size, tsdf, weight, color, R, threshold, threads=1):
    keys, tsdf, weight = (np.ascontiguousarray(a) for a in (keys, tsdf, weight))
    color = None if color is None else np.ascontiguousarray(color)
    args = (keys.ctypes.data, size, tsdf.ctypes.data, weight.ctypes.data, None if color is None else color.ctypes.data,
            R, VOXEL, threshold, threads)
    nt = C.c_int64(0)
    nv = ref.ref_extract_triangle_mesh(*args, 0, 0, None, None, None, None, C.byref(nt))
    out = {"positions": np.zeros((nv, 3), np.float32), "normals": np.zeros((nv, 3), np.float32),
           "indices": np.zeros((nt.value, 3), np.int32)}
    if color is not None:
        out["colors"] = np.zeros((nv, 3), np.float32)
    ref.ref_extract_triangle_mesh(*args, nv, nt.value, out["positions"].ctypes.data, out["normals"].ctypes.data,
                                  out["colors"].ctypes.data if color is not None else None, out["indices"].ctypes.data,
                                  C.byref(nt))
    return out


def boundary_cycles(tris):
    """The oriented boundary cycles of a set of triangles, each rotated to start at its smallest entry."""
    directed = {(t[i], t[(i + 1) % 3]) for t in tris for i in range(3)}
    assert len(directed) == 3 * len(tris), "a directed edge is used twice"
    nxt = {}
    for a, b in directed:
        if (b, a) not in directed:
            assert a not in nxt, "a vertex starts two boundary edges"
            nxt[a] = b
    out, seen = set(), set()
    for a in sorted(nxt):
        if a in seen:
            continue
        cyc, e = [], a
        while e not in seen:
            seen.add(e)
            cyc.append(e)
            e = nxt[e]
        assert e == a
        k = cyc.index(min(cyc))
        out.add(tuple(cyc[k:] + cyc[:k]))
    return out


def ref_table_row(ref, c):
    row = np.zeros(16, np.int32)
    mask, count = C.c_int32(0), C.c_int32(0)
    ref.ref_mc_table_row(c, row.ctypes.data, C.byref(mask), C.byref(count))
    tris = [tuple(row[3 * i:3 * i + 3]) for i in range(5) if row[3 * i] != -1]
    return tris, int(mask.value), int(count.value)


@needs_ref
def test_case_table_is_the_reference_surface(ref):
    patches = 0
    for c in range(256):
        want, want_mask, want_count = ref_table_row(ref, c)
        got, got_mask = mesh_oracle.table_row(c)
        got = [tuple(t) for t in got.tolist()]
        assert len(got) == want_count == len(want), c
        assert got_mask == want_mask, c
        assert boundary_cycles(got) == boundary_cycles(want), c
        # every patch is an oriented disc: one boundary cycle, V - E + F = 1
        comp = list(range(len(got)))
        for i in range(len(got)):
            for j in range(i):
                if len(set(got[i]) & set(got[j])) == 2:
                    a, b = comp[i], comp[j]
                    comp = [b if x == a else x for x in comp]
        for p in set(comp):
            tris = [t for t, q in zip(got, comp) if q == p]
            verts = {v for t in tris for v in t}
            edges = {frozenset((t[i], t[(i + 1) % 3])) for t in tris for i in range(3)}
            assert len(boundary_cycles(tris)) == 1 and len(verts) - len(edges) + len(tris) == 1, (c, tris)
            patches += 1
    assert patches == 358


def assert_same_mesh(got, want, keys, tsdf, weight, R, threshold):
    """Vertex arrays bit for bit in the same order; triangles per cube as the same oriented boundary cycles."""
    assert set(got) == set(want)
    for name in ("positions", "normals", "colors"):
        if name in want:
            assert got[name].shape == want[name].shape, name
            assert np.array_equal(got[name].view(np.uint32), want[name].view(np.uint32)), name
    gi, wi = got["indices"], want["indices"]
    assert gi.shape == wi.shape
    cases = cube_cases(keys, tsdf, weight, R, threshold).reshape(-1)
    ntri = np.array([len(mesh_oracle.table_row(c)[0]) for c in range(256)])
    counts = np.where(cases >= 0, ntri[np.maximum(cases, 0)], 0)
    assert counts.sum() == len(gi)
    ends = np.cumsum(counts)
    for v in np.nonzero(counts)[0]:
        lo, hi = ends[v] - counts[v], ends[v]
        assert boundary_cycles([tuple(t) for t in gi[lo:hi].tolist()]) == \
            boundary_cycles([tuple(t) for t in wi[lo:hi].tolist()]), v


@needs_ref
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("R", [8, 4, 1])
@pytest.mark.parametrize("with_color", [True, False])
def test_hand_built_mesh_is_the_reference_mesh(ref, kind, R, with_color):
    v = mesh_volume(kind, R, with_color)
    size = len(v["keys"])
    got = mesh_oracle.extract_triangle_mesh(v["keys"], size, v["tsdf"], v["weight"], v["color"], R, VOXEL, THRESHOLD)
    want = reference_mesh(ref, v["keys"], size, v["tsdf"], v["weight"], v["color"], R, THRESHOLD)
    assert_same_mesh(got, want, v["keys"], v["tsdf"], v["weight"], R, THRESHOLD)
    if kind == "random_signs" and R == 8:
        assert (case_histogram(v, R) > 0).all()


@pytest.fixture(scope="module")
def rooms():
    return {(R, c): fuse_room((200, 203, 206, 209), R, c) for R in (16, 8) for c in (True, False)}


@needs_ref
@pytest.mark.parametrize("R", [16, 8])
@pytest.mark.parametrize("with_color", [True, False])
@pytest.mark.parametrize("threshold", [0.0, 3.0])
def test_room_mesh_is_the_reference_mesh(ref, rooms, R, with_color, threshold):
    keys, size, tsdf, wt, col = rooms[(R, with_color)]
    got = mesh_oracle.extract_triangle_mesh(keys, size, tsdf, wt, col, R, VOXEL, threshold)
    want = reference_mesh(ref, keys, size, tsdf, wt, col, R, threshold)
    assert len(got["indices"]) > 20000
    assert_same_mesh(got, want, keys, tsdf, wt, R, threshold)


def test_room_mesh_geometry(rooms):
    """The oracle's mesh of a fused room lies on the analytic surfaces, is an oriented manifold and faces free space."""
    keys, size, tsdf, wt, col = rooms[(16, True)]
    m = mesh_oracle.extract_triangle_mesh(keys, size, tsdf, wt, col, 16, VOXEL, 3.0)
    p, nrm, tri = m["positions"].astype(np.float64), m["normals"].astype(np.float64), m["indices"]
    assert len(tri) > 20000 and tri.min() >= 0 and tri.max() < len(p)
    lo, hi = np.asarray(ROOM_MIN), np.asarray(ROOM_MAX)
    d_wall = np.minimum(np.abs(p - lo), np.abs(p - hi)).min(axis=1)
    d_sphere = np.abs(np.linalg.norm(p - np.asarray(SPHERE_C), axis=1) - SPHERE_R)
    assert np.minimum(d_wall, d_sphere).max() < VOXEL
    # each undirected edge in at most two triangles; a shared edge in opposite directions
    directed = np.concatenate([tri[:, [0, 1]], tri[:, [1, 2]], tri[:, [2, 0]]])
    assert len(np.unique(directed, axis=0)) == len(directed)
    und = np.sort(directed, axis=1)
    _, counts = np.unique(und, axis=0, return_counts=True)
    assert counts.max() <= 2
    # the winding's normal agrees in sign with the vertices' interpolated TSDF gradients
    a, b, c = p[tri[:, 0]], p[tri[:, 1]], p[tri[:, 2]]
    face = np.cross(b - a, c - a)
    dots = np.einsum("ij,ij->i", face, nrm[tri].sum(axis=1))
    assert (dots > 0).mean() > 0.999, (dots <= 0).sum()

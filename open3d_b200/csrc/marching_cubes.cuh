// marching_cubes.cuh — the marching-cubes case table of the triangle-mesh extraction (extract.cu), generated at
// compile time from the rule that fixes upstream's surface (DESIGN.md §4.27).
//
// Corner k of the cube at voxel o sits at o + kCorner[k] (the standard marching-cubes numbering that
// t/geometry/kernel/GeometryMacros.h uses); edge e joins corners kEdge[e][0] and kEdge[e][1], the first being the
// lower end, so the edge is the axis-edge_axis(e) edge owned by voxel o + kCorner[kEdge[e][0]].  Case bit k is set
// when corner k has tsdf < 0.
//
// For case c the generator
//   1. cuts each of the 6 faces: an edge whose corners differ in their bit carries a vertex; a face with two such
//      edges gets the one segment between them, a face with four (diagonal corners share their bit) gets two
//      segments, each cutting off one of the face's two set corners;
//   2. orients every segment along m x n, where m points from the segment towards the face's set corners it cuts
//      off and n is the face's outward normal.  Every patch's normal then points towards the set (negative)
//      corners, which is the orientation of upstream's table; the kernel writes each triangle reversed, as upstream
//      does;
//   3. chains the segments into cycles (every crossed edge has one segment in and one out), taken in order of their
//      lowest edge, each starting at its lowest edge;
//   4. caps each cycle a0 a1 ... a(k-1) with the fan (a0, ai, ai+1), i = 1 .. k-2.
// The edge mask and the triangle count of a case follow from the same code.
#pragma once

#include <cstdint>

namespace o3db {
namespace mc {

constexpr int kCorner[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0}, {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
constexpr int kEdge[12][2] = {{0, 1}, {1, 2}, {3, 2}, {0, 3}, {4, 5}, {5, 6}, {7, 6}, {4, 7}, {0, 4}, {1, 5}, {2, 6}, {3, 7}};
constexpr int kMaxTri = 5;   // the most triangles any case gets

// corner index of the cube corner at offset (x, y, z) in {0, 1}^3, and the offset of corner k along axis d
constexpr int corner_at(int x, int y, int z) { return 4 * z + (y ? (x ? 2 : 3) : (x ? 1 : 0)); }
constexpr int corner_offset(int k, int d) { return d == 0 ? ((k ^ (k >> 1)) & 1) : (k >> d) & 1; }

constexpr int edge_axis(int e) {
    return kCorner[kEdge[e][1]][0] != kCorner[kEdge[e][0]][0] ? 0 : kCorner[kEdge[e][1]][1] != kCorner[kEdge[e][0]][1] ? 1 : 2;
}

constexpr int edge_between(int a, int b) {
    for (int e = 0; e < 12; ++e)
        if ((kEdge[e][0] == a && kEdge[e][1] == b) || (kEdge[e][0] == b && kEdge[e][1] == a)) return e;
    return -1;
}

struct Table {
    uint8_t ntri[256];          // triangles of the case
    uint16_t edges[256];        // bit e: edge e carries a vertex
    int8_t tri[256][3 * kMaxTri];   // edge indices, three per triangle, before the kernel's reversal
    uint8_t owner[12];          // edge e: offset of its owning voxel (bits 0-2: x, y, z) | its axis << 3
};

constexpr Table make_table() {
    Table t{};
    for (int e = 0; e < 12; ++e) {
        const int* p = kCorner[kEdge[e][0]];
        t.owner[e] = (uint8_t)(p[0] | p[1] << 1 | p[2] << 2 | edge_axis(e) << 3);
    }
    for (int c = 0; c < 256; ++c) {
        int next[12] = {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1};
        unsigned edges = 0;
        for (int e = 0; e < 12; ++e)
            if (((c >> kEdge[e][0]) ^ (c >> kEdge[e][1])) & 1) edges |= 1u << e;
        // 1-2: the oriented segments of the 6 faces; positions are doubled so that edge midpoints are integers
        for (int f = 0; f < 6; ++f) {
            const int ax = f >> 1, side = f & 1, u = (ax + 1) % 3, v = (ax + 2) % 3;
            int corner[4] = {0, 0, 0, 0};   // the face's corners in cyclic order
            const int uv[4][2] = {{0, 0}, {1, 0}, {1, 1}, {0, 1}};
            for (int k = 0; k < 4; ++k) {
                int p[3] = {0, 0, 0};
                p[ax] = side;
                p[u] = uv[k][0];
                p[v] = uv[k][1];
                corner[k] = corner_at(p[0], p[1], p[2]);
            }
            int fe[4] = {0, 0, 0, 0};   // fe[k]: the edge from corner k to corner k+1
            int nset = 0, ncut = 0;
            for (int k = 0; k < 4; ++k) {
                fe[k] = edge_between(corner[k], corner[(k + 1) & 3]);
                nset += (c >> corner[k]) & 1;
                ncut += (edges >> fe[k]) & 1;
            }
            int seg[2][2] = {{-1, -1}, {-1, -1}}, m[2][3] = {{0, 0, 0}, {0, 0, 0}};
            int nseg = 0;
            if (ncut == 2) {
                for (int k = 0; k < 4; ++k)
                    if ((edges >> fe[k]) & 1) seg[0][seg[0][0] < 0 ? 0 : 1] = fe[k];
                // from the centroid of the clear corners towards that of the set corners (both scaled)
                for (int k = 0; k < 4; ++k)
                    for (int d = 0; d < 3; ++d)
                        m[0][d] += 2 * kCorner[corner[k]][d] * (((c >> corner[k]) & 1) ? 4 - nset : -nset);
                nseg = 1;
            } else if (ncut == 4) {
                for (int k = 0; k < 4; ++k) {
                    if (!((c >> corner[k]) & 1)) continue;
                    const int a = fe[(k + 3) & 3], b = fe[k];   // the two face edges at set corner k
                    seg[nseg][0] = a;
                    seg[nseg][1] = b;
                    for (int d = 0; d < 3; ++d)
                        m[nseg][d] = 4 * kCorner[corner[k]][d] - (kCorner[kEdge[a][0]][d] + kCorner[kEdge[a][1]][d]) -
                                     (kCorner[kEdge[b][0]][d] + kCorner[kEdge[b][1]][d]);
                    ++nseg;
                }
            }
            for (int s = 0; s < nseg; ++s) {
                int a = seg[s][0], b = seg[s][1], d[3] = {0, 0, 0};
                for (int k = 0; k < 3; ++k)
                    d[k] = kCorner[kEdge[b][0]][k] + kCorner[kEdge[b][1]][k] - kCorner[kEdge[a][0]][k] - kCorner[kEdge[a][1]][k];
                // (m x d) . n with n = +-e_ax: keep a -> b when it is negative (m x n along d)
                const int mxd = m[s][u] * d[v] - m[s][v] * d[u];
                const int dot = side ? mxd : -mxd;
                if (dot > 0) {
                    const int tmp = a;
                    a = b;
                    b = tmp;
                }
                next[a] = b;
            }
        }
        // 3-4: cycles from their lowest edge, each capped by a fan
        unsigned seen = 0;
        int n = 0;
        for (int e0 = 0; e0 < 12; ++e0) {
            if (!((edges >> e0) & 1) || ((seen >> e0) & 1)) continue;
            int cyc[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0}, len = 0;
            for (int e = e0; e >= 0 && !((seen >> e) & 1); e = next[e]) {
                seen |= 1u << e;
                cyc[len++] = e;
            }
            for (int i = 1; i + 1 < len; ++i) {
                t.tri[c][3 * n] = (int8_t)cyc[0];
                t.tri[c][3 * n + 1] = (int8_t)cyc[i];
                t.tri[c][3 * n + 2] = (int8_t)cyc[i + 1];
                ++n;
            }
        }
        t.ntri[c] = (uint8_t)n;
        t.edges[c] = (uint16_t)edges;
    }
    return t;
}

}  // namespace mc
}  // namespace o3db

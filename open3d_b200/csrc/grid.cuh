// grid.cuh — dense uniform search grid over the target cloud and the exact
// 1-NN-within-radius scan used by both the stand-alone hybrid search and the
// fused ICP iteration kernel.
//
// Replaces the reference's hashed CSR table (core/nns/FixedRadiusSearchImpl.cuh:
// 63-134 build, :514-631 query).  Results (index, dist^2, count) are identical
// to an exhaustive search; the table layout is private to this library.
//
// Layout in HBM (built once per target / scale):
//   pts4      float4[M]   target points sorted by cell key, .w = original index bits
//   nrm4      float4[M]   target normals in the same order (optional)
//   cell_start u32[ncell+1] CSR offsets, key = (iz*ny + iy)*nx + ix (x fastest, so
//              every (iy,iz) row of cells is ONE contiguous run of pts4)
#pragma once

#include "common.cuh"

namespace o3db {

// All fields are in GRID axis order: grid-x is the fastest-varying axis of the CSR table.
// ax[k] names the real coordinate (0 = x, 1 = y, 2 = z) that grid axis k follows; the host
// makes the axis with the smallest extent the fastest one, so that for surface-like clouds a
// whole "column" of cells along the thin direction is one short contiguous run.
struct Grid {
    float ox, oy, oz;   // origin = bbox min
    float inv_c, c;     // cell size and reciprocal (grid-y, grid-z)
    float inv_cx, cx;   // cell size along grid-x, the thin axis: kThinFactor x coarser — slab scans cross
                        // all grid-x cells anyway, and the CSR table shrinks by that factor (L2 residency)
    float tol;          // pruning slack covering binning round-off (see DESIGN.md)
    int nx, ny, nz;
    float bmin[3], bmax[3];
    int ax[3];
};

__device__ __forceinline__ float pick_axis(int a, float x, float y, float z) { return a == 0 ? x : (a == 1 ? y : z); }
// real (x,y,z) -> grid-ordered (gx,gy,gz)
__device__ __forceinline__ void to_grid(const Grid& g, float x, float y, float z, float& gx, float& gy, float& gz) {
    gx = pick_axis(g.ax[0], x, y, z);
    gy = pick_axis(g.ax[1], x, y, z);
    gz = pick_axis(g.ax[2], x, y, z);
}

// Monotone binning: x <= y  =>  cell1(x) <= cell1(y)  (sub, mul by a positive
// constant, floor and clamp are all monotone under round-to-nearest).  Coverage
// of the radius search relies only on this property, never on exact cell bounds.
__device__ __forceinline__ int cell1(float x, float o, float inv_c, int n) {
    int i = __float2int_rd((x - o) * inv_c);
    return min(max(i, 0), n - 1);
}

__device__ __forceinline__ unsigned cell_key(const Grid& g, float rx, float ry, float rz) {
    float x, y, z;
    to_grid(g, rx, ry, rz, x, y, z);
    const int ix = cell1(x, g.ox, g.inv_cx, g.nx);
    const int iy = cell1(y, g.oy, g.inv_c, g.ny);
    const int iz = cell1(z, g.oz, g.inv_c, g.nz);
    return (unsigned)((iz * g.ny + iy) * g.nx + ix);
}

// Lower / upper end of the interval that must be binned to cover |t - q| <= r
// given that dist^2 was accepted in f32: r' = r (1 + 1e-6) plus 2 ulp of |q|.
__device__ __forceinline__ float lo_bound(float q, float rr) { return (q - rr) - fabsf(q) * 2.4e-7f; }
__device__ __forceinline__ float hi_bound(float q, float rr) { return (q + rr) + fabsf(q) * 2.4e-7f; }

static constexpr unsigned kSlabMax = 32;   // longest slab scanned whole (see nn_search_two_pass)

struct Best {
    float d;    // best dist^2 so far (starts at the threshold: accepts d <= thr)
    int j;      // position in the sorted arrays, -1 = none
    int idx;    // original index of the best point (tie-break: lower wins)
    float x, y, z;
};

// Scans pts[s, e): 4 independent 128-bit loads in flight per step (the tail re-reads the last
// candidate, which cannot change the result).
__device__ __forceinline__ void scan_range(const float4* __restrict__ pts, unsigned s, unsigned e,
                                           float qx, float qy, float qz, Best& b) {
    for (unsigned j = s; j < e; j += 4) {
        float4 t[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) t[k] = __ldg(&pts[min(j + k, e - 1)]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float dx = t[k].x - qx, dy = t[k].y - qy, dz = t[k].z - qz;
            // canonical arithmetic (bit-identical to oracle/icp_oracle.c dist2_f32)
            const float d = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
            const int idx = __float_as_int(t[k].w);
            if (d < b.d || (d == b.d && idx < b.idx)) {
                b.d = d;
                b.j = (int)min(j + k, e - 1);
                b.idx = idx;
                b.x = t[k].x;
                b.y = t[k].y;
                b.z = t[k].z;
            }
        }
    }
}

// ONE loop over the concatenation of up to NS slabs [s[k], s[k] + n[k]): a warp then runs
// max_lane(sum n)/4 trips instead of sum_slabs(max_lane(n_slab)/4) — the lanes' slabs fill differently, and
// padding every slab separately to the warp's worst lane left two thirds of the candidate slots idle (ncu,
// DESIGN.md §4.1).  The running best is one 64-bit key (dist^2 bits : index) so that "closer, ties to the
// lower index" is a single unsigned comparison; non-negative floats order like their bit patterns.
// `best` / `bj` come in initialised ("nothing": thr:INT_MAX / 0xffffffff, or a seed candidate) and are only
// replaced by keys <= best.
static constexpr unsigned kNoPoint = 0xffffffffu;
// TRACK2: also keep d2nd = the smallest dist^2 among the scanned candidates that did NOT end up best (the
// caller derives from it how far every point other than the winner is: see nn_search_seeded_fast).
template <int NS, bool TRACK2>
__device__ __forceinline__ void scan_slabs_flat(const float4* __restrict__ pts, const unsigned (&s)[NS],
                                                const unsigned (&n)[NS], float qx, float qy, float qz,
                                                unsigned long long& best, unsigned& bj, float& d2nd) {
    unsigned pre[NS], off[NS];   // slab k covers virtual indices [pre[k], pre[k] + n[k]); global = off[k] + virtual
    unsigned total = 0;
#pragma unroll
    for (int k = 0; k < NS; ++k) {
        pre[k] = total;
        off[k] = s[k] - total;
        total += n[k];
    }
    for (unsigned v = 0; v < total; v += 4) {
        unsigned jj[4];
        float4 t[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const unsigned w = min(v + k, total - 1);   // the tail re-reads the last candidate (cannot change the result)
            unsigned o = off[0];
#pragma unroll
            for (int q = 1; q < NS; ++q) o = w >= pre[q] ? off[q] : o;
            jj[k] = o + w;
            t[k] = __ldg(&pts[jj[k]]);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float dx = t[k].x - qx, dy = t[k].y - qy, dz = t[k].z - qz;
            const float d = fmaf(dz, dz, fmaf(dy, dy, dx * dx));   // canonical (see scan_range)
            const unsigned long long key =
                    ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)__float_as_int(t[k].w);
            if (TRACK2) {
                // (a re-read of the current best — the loop's tail padding — must not count as a second point)
                if (key < best) {
                    d2nd = fminf(d2nd, __uint_as_float((unsigned)(best >> 32)));
                    best = key;
                    bj = jj[k];
                } else if (key != best) {
                    d2nd = fminf(d2nd, d);
                }
            } else if (key <= best) {   // d >= 0, so the bit patterns order like the values; NaN sorts last
                best = key;
                bj = jj[k];
            }
        }
    }
}

// Every point whose (grid-y, grid-z) cell is touched by the box [q - rad, q + rad], over ALL grid-x cells,
// as at most NS slabs in one flat loop.  For every grid-z of the box, the cells [all grid-x] x [y0..y1] are
// ONE contiguous run of the table (x fastest, then y); grid-x is the cloud's thin direction, so for
// surface-like data a run holds just the handful of points of a few cell columns, for two CSR loads.
// All CSR loads are issued together, then all candidates four at a time: two dependent round trips whatever
// the box size.  Returns false — nothing scanned, best / bj untouched — when the box spans more than NS
// grid-z rows or a slab is long (volumetric data): the caller then prunes row by row (nn_search_from).
template <int NS, bool TRACK2 = false>
__device__ __forceinline__ bool scan_box_flat(const Grid& g, const float4* __restrict__ pts,
                                              const unsigned* __restrict__ cs, float gy, float gz, float qx,
                                              float qy, float qz, float rad, unsigned long long& best,
                                              unsigned& bj, float* d2nd = nullptr) {
    const int y0 = cell1(lo_bound(gy, rad), g.oy, g.inv_c, g.ny), y1 = cell1(hi_bound(gy, rad), g.oy, g.inv_c, g.ny);
    const int z0 = cell1(lo_bound(gz, rad), g.oz, g.inv_c, g.nz), z1 = cell1(hi_bound(gz, rad), g.oz, g.inv_c, g.nz);
    if (z1 - z0 >= NS) return false;
    unsigned s[NS], n[NS];
    unsigned longest = 0;
#pragma unroll
    for (int dz = 0; dz < NS; ++dz) {
        unsigned b0 = 0, b1 = 0;
        if (z0 + dz <= z1) {
            const int plane = (z0 + dz) * g.ny;
            b0 = __ldg(&cs[(plane + y0) * g.nx]);
            b1 = __ldg(&cs[(plane + y1 + 1) * g.nx]);
        }
        s[dz] = b0;
        n[dz] = b1 - b0;
        longest = max(longest, n[dz]);
    }
    if (longest > kSlabMax) return false;
    float dummy = 0.f;
    scan_slabs_flat<NS, TRACK2>(pts, s, n, qx, qy, qz, best, bj, TRACK2 ? *d2nd : dummy);
    return true;
}

// One (iy, iz) row of cells: visit only the x cells that can still hold a point at
// distance <= best, given that every point of the row is at least sqrt(gap2) away in (y, z).
// skip_cx >= 0: that cell was scanned already.
__device__ __forceinline__ void scan_row(const Grid& g, const float4* __restrict__ pts,
                                         const unsigned* __restrict__ cs, int row, int x0, int x1, int skip_cx,
                                         float gap2, float gqx, float qx, float qy, float qz, Best& b) {
    // admissible |dx|: dx^2 <= best - gap2 (1e-6 best covers the rounding of the subtraction)
    const float ex = sqrtf(fmaf(b.d, 1e-6f, b.d - gap2)) * 1.00001f;
    const int xa = max(x0, cell1(lo_bound(gqx, ex), g.ox, g.inv_cx, g.nx));
    const int xb = min(x1, cell1(hi_bound(gqx, ex), g.ox, g.inv_cx, g.nx));
    if (skip_cx < xa || skip_cx > xb) {
        if (xa <= xb) scan_range(pts, cs[row + xa], cs[row + xb + 1], qx, qy, qz, b);
    } else {
        if (xa < skip_cx) scan_range(pts, cs[row + xa], cs[row + skip_cx], qx, qy, qz, b);
        if (skip_cx < xb) scan_range(pts, cs[row + skip_cx + 1], cs[row + xb + 1], qx, qy, qz, b);
    }
}

// Exact nearest neighbour of (qx,qy,qz) among points with dist^2 <= thr.
// rr = radius * (1 + 1e-6).  Visiting order: the query's own cell, the rest of its row, then the
// other rows of the neighbourhood; a row (and the x cells inside it) is skipped as soon as its
// distance lower bound exceeds the best distance found so far.  PRUNE = false visits everything
// (used to validate the pruning).
// nn_search_from: `b` is pre-initialised — either "nothing yet" (d = thr, j = -1, idx = INT_MAX) or an
// actual candidate (a seed): every point that beats b lies within rr of the query, so rr may be the
// seed's distance instead of the search radius.
template <bool PRUNE>
__device__ __forceinline__ void nn_search_from(const Grid& g, const float4* __restrict__ pts,
                                               const unsigned* __restrict__ cs, float qx, float qy,
                                               float qz, float rr, Best& b) {
    float gx, gy, gz;                       // the query in grid axis order (cells / gaps only)
    to_grid(g, qx, qy, qz, gx, gy, gz);
    const float lx = lo_bound(gx, rr), hx = hi_bound(gx, rr);
    const float ly = lo_bound(gy, rr), hy = hi_bound(gy, rr);
    const float lz = lo_bound(gz, rr), hz = hi_bound(gz, rr);
    // entirely outside the bounding box (or NaN): no candidate can pass
    if (hx < g.bmin[0] || lx > g.bmax[0] || hy < g.bmin[1] || ly > g.bmax[1] || hz < g.bmin[2] ||
        lz > g.bmax[2] || !(qx == qx) || !(qy == qy) || !(qz == qz))
        return;
    const int x0 = cell1(lx, g.ox, g.inv_cx, g.nx), x1 = cell1(hx, g.ox, g.inv_cx, g.nx);
    const int y0 = cell1(ly, g.oy, g.inv_c, g.ny), y1 = cell1(hy, g.oy, g.inv_c, g.ny);
    const int z0 = cell1(lz, g.oz, g.inv_c, g.nz), z1 = cell1(hz, g.oz, g.inv_c, g.nz);
    const int cx = cell1(gx, g.ox, g.inv_cx, g.nx);
    const int cy = cell1(gy, g.oy, g.inv_c, g.ny), cz = cell1(gz, g.oz, g.inv_c, g.nz);
    if (!PRUNE) {
        for (int iz = z0; iz <= z1; ++iz)
            for (int iy = y0; iy <= y1; ++iy) {
                const int row = (iz * g.ny + iy) * g.nx;
                scan_range(pts, cs[row + x0], cs[row + x1 + 1], qx, qy, qz, b);
            }
        return;
    }
    {
        const int row = (cz * g.ny + cy) * g.nx;
        scan_range(pts, cs[row + cx], cs[row + cx + 1], qx, qy, qz, b);   // own cell
        scan_row(g, pts, cs, row, x0, x1, cx, 0.f, gx, qx, qy, qz, b);     // rest of the own row
    }
    for (int iz = z0; iz <= z1; ++iz) {
        float dz = 0.f;
        if (iz > cz) dz = (g.oz + (float)iz * g.c) - gz - g.tol;
        else if (iz < cz) dz = gz - (g.oz + (float)(iz + 1) * g.c) - g.tol;
        dz = fmaxf(dz, 0.f);
        dz *= dz;
        if (dz > b.d) continue;
        for (int iy = y0; iy <= y1; ++iy) {
            if (iy == cy && iz == cz) continue;
            float dy = 0.f;
            if (iy > cy) dy = (g.oy + (float)iy * g.c) - gy - g.tol;
            else if (iy < cy) dy = gy - (g.oy + (float)(iy + 1) * g.c) - g.tol;
            dy = fmaxf(dy, 0.f);
            const float gap2 = fmaf(dy, dy, dz);
            if (gap2 > b.d) continue;  // strict: keeps exact ties reachable
            scan_row(g, pts, cs, (iz * g.ny + iy) * g.nx, x0, x1, -1, gap2, gx, qx, qy, qz, b);
        }
    }
}

template <bool PRUNE>
__device__ __forceinline__ void nn_search(const Grid& g, const float4* __restrict__ pts,
                                          const unsigned* __restrict__ cs, float qx, float qy,
                                          float qz, float rr, float thr, Best& b) {
    b.d = thr;
    b.j = -1;
    b.idx = 0x7fffffff;
    b.x = b.y = b.z = 0.f;
    nn_search_from<PRUNE>(g, pts, cs, qx, qy, qz, rr, b);
}

// --------------------------------------------------------- searches of the fused ICP kernels
//
// Fast path (inline, scan_box_flat<3> from a seed) and slow path (nn_search_slow, deliberately NOT inlined:
// it runs for a handful of queries per iteration once the clouds are roughly aligned, and keeping its loops
// out of the iteration kernel's main body keeps that body's register allocation tight).
//
// Seeds (temporal coherence): `seed_j` is the sorted position of the point that won this query in the
// previous iteration.  The seed is an ACTUAL candidate, so the exact nearest neighbour is either the seed or a
// point with key (dist^2 : index) <= the seed's — and every such point lies within sqrt(dist^2_seed) of the
// query per axis.  Scanning all cells that the box [q - rad, q + rad] touches (rad = that distance, inflated
// by 1e-5 for the f32 rounding of the distance arithmetic; binning slack as in lo_bound / hi_bound) is
// therefore exhaustive: same result, bit for bit, as the unseeded search, from ~4 candidates instead of ~16.

// canonical dist^2 (bit-identical to oracle/icp_oracle.c dist2_f32)
__device__ __forceinline__ float dist2_canonical(const float4 t, float qx, float qy, float qz) {
    const float dx = t.x - qx, dy = t.y - qy, dz = t.z - qz;
    return fmaf(dz, dz, fmaf(dy, dy, dx * dx));
}

// Seeded fast path.  ts = pts[seed_j] and sd = its canonical dist^2 <= thr (the caller has both: the staged
// kernel fetched the seed one chunk ahead and needs the distance for its certificate).  The box [q - rad,
// q + rad], rad = sqrt(sd) (hardware reciprocal square root, 2 ulp, with a 1e-4 margin), is scanned from
// "nothing yet": it contains the seed, hence the exact winner and every point tying with it.
// A seed farther than r1 (right after a large update: the old winner is a motion's length away while the true
// neighbour is millimetres away) would bound a box larger than the unseeded search's pass 1, often taller than 3
// cell rows; the box is then pass 1's, [q - r1, q + r1], and its best point is the exact winner when it lies within
// r1 (r1_accept2 = (r1 (1 - 1e-4))^2, as in nn_search_slow): every point outside the box is farther than r1.
// Fewer candidates is what saves time in these iterations, whose scans are bound by the instructions every candidate
// costs (DESIGN.md §4.1); and the query leaves with a clearance, where nn_search_slow leaves none.
// On return `handled` = false when the fast path does not apply (box taller than 3 cell rows, long slabs, or the
// best point of pass 1's box not within r1: the caller then calls nn_search_slow); otherwise the winner's sorted
// position is returned and `clearance` = a lower bound on the distance from the query to EVERY target point other
// than the winner: min(sqrt(d2nd), rad) — a point that was not scanned lies outside the box, i.e. farther than rad
// along grid-y or grid-z (binning is monotone; lo_bound / hi_bound only widen the box).
__device__ __forceinline__ unsigned nn_search_seeded_fast(const Grid& g, const float4* __restrict__ pts,
                                                          const unsigned* __restrict__ cs, float qx, float qy,
                                                          float qz, float r1, float r1_accept2, float rr, float thr,
                                                          float sd, bool& handled, float& clearance) {
    const float rs = sd > 0.f ? fminf(rr, sd * rsqrtf(sd) * 1.0001f) : 0.f;
    const bool far = rs > r1;
    const float rad = far ? r1 : rs;
    float gx, gy, gz;
    to_grid(g, qx, qy, qz, gx, gy, gz);
    unsigned long long best = ((unsigned long long)__float_as_uint(thr) << 32) | 0x7fffffffull;
    unsigned bj = kNoPoint;
    float d2nd = __int_as_float(0x7f7fffff);
    handled = scan_box_flat<3, true>(g, pts, cs, gy, gz, qx, qy, qz, rad, best, bj, &d2nd) &&
              (!far || (bj != kNoPoint && __uint_as_float((unsigned)(best >> 32)) <= r1_accept2));
    // rounded down: 2 ulp of the reciprocal square root and the f32 rounding of d2nd are inside the 1e-5
    clearance = fminf(rad, d2nd * rsqrtf(fmaxf(d2nd, 1e-37f)) * 0.99999f);
    return bj;
}

// Everything else: no seed (first iteration, previously unmatched points), far seed, volumetric data.
//   no seed:   pass 1 scans the box [q - r1, q + r1] (r1 = max(cell size, r / 2)); if the best point
//              found is within r1 it is the exact nearest neighbour (nothing closer can lie outside the
//              box); r1_accept2 = (r1 (1 - 1e-4))^2;
//   then:      the full-radius box (or the seed-bounded one) as one flat 5-slab scan;
//   otherwise: the pruned row-by-row search.
// Returns the winner's sorted position or kNoPoint.
__device__ __noinline__ unsigned nn_search_slow(const Grid* gp, const float4* __restrict__ pts,
                                                const unsigned* __restrict__ cs, float qx, float qy, float qz,
                                                float r1, float r1_accept2, float rr, float thr, int seed_j) {
    const Grid& g = *gp;
    unsigned long long best = ((unsigned long long)__float_as_uint(thr) << 32) | 0x7fffffffull;
    unsigned bj = kNoPoint;
    unsigned long long seed_key = ~0ull;
    float rad = rr;
    if (seed_j >= 0) {
        const float4 ts = __ldg(&pts[seed_j]);
        const float sd = dist2_canonical(ts, qx, qy, qz);
        if (sd <= thr) {
            seed_key = ((unsigned long long)__float_as_uint(sd) << 32) | (unsigned)__float_as_int(ts.w);
            rad = fminf(rr, sqrtf(sd) * 1.00001f);
        }
    }
    float gx, gy, gz;
    to_grid(g, qx, qy, qz, gx, gy, gz);
    if (seed_key == ~0ull) {
        // entirely outside the bounding box (or NaN): no candidate can pass
        if (hi_bound(gx, rr) < g.bmin[0] || lo_bound(gx, rr) > g.bmax[0] || hi_bound(gy, rr) < g.bmin[1] ||
            lo_bound(gy, rr) > g.bmax[1] || hi_bound(gz, rr) < g.bmin[2] || lo_bound(gz, rr) > g.bmax[2] ||
            !(qx == qx) || !(qy == qy) || !(qz == qz))
            return kNoPoint;
    }
    // A seed farther than r1 bounds a box larger than pass 1's (typical right after a large first update:
    // the old winner is a motion's length away while the true neighbour is millimetres away): pass 1 first.
    if (r1 < rad && scan_box_flat<5>(g, pts, cs, gy, gz, qx, qy, qz, r1, best, bj) && bj != kNoPoint &&
        __uint_as_float((unsigned)(best >> 32)) <= r1_accept2)
        return bj;
    if (seed_key < best) {   // the seed is an actual candidate: it bounds whatever comes next
        best = seed_key;
        bj = (unsigned)seed_j;
    }
    // every point that can still win lies within the distance of the best candidate known so far
    if (bj != kNoPoint) rad = fminf(rad, sqrtf(__uint_as_float((unsigned)(best >> 32))) * 1.00001f);
    if (scan_box_flat<5>(g, pts, cs, gy, gz, qx, qy, qz, rad, best, bj)) return bj;
    if (scan_box_flat<9>(g, pts, cs, gy, gz, qx, qy, qz, rad, best, bj)) return bj;   // cells finer than r / 2
    Best b;
    b.d = __uint_as_float((unsigned)(best >> 32));
    b.idx = (int)(unsigned)(best & 0xffffffffull);
    b.j = bj == kNoPoint ? -1 : (int)bj;
    b.x = b.y = b.z = 0.f;
    nn_search_from<true>(g, pts, cs, qx, qy, qz, rad, b);
    return b.j < 0 ? kNoPoint : (unsigned)b.j;
}

}  // namespace o3db

// remove_oracle.c — TEST INFRASTRUCTURE: the CPU oracle of t::geometry::PointCloud's clean-up filters
// (t/geometry/PointCloud.cpp:650-676, 716-760), restated in C.
//
// Radius count: the number of points q with dist(p, q) <= thr, p itself included, thr = (float)r * (float)r, with one
// of two predicates on d = p - q in f32:
//   mode 0 "cuda"   dist = fmaf(d2, d2, fmaf(d1, d1, fmaf(d0, d0, 0))): upstream's NeighborTest<L2, float>
//                   (core/nns/FixedRadiusSearchImpl.cuh:41-59) as nvcc contracts it for sm_90a;
//   mode 1 "plain"  dist = ((0 + d0 d0) + d1 d1) + d2 d2, each op rounded: MiniVec::dot (utility/MiniVec.h:47-51)
//                   without contraction, as upstream's CPU search computes it through Eigen.
// Either by brute force over all pairs, or over a grid of cells of at least 1.0001 (1 + 1e-5) r, from the 27 cells
// around the query (every accepted point lies within r (1 + 4 2^-24) per axis); the tests check that the two agree.
// Duplicates: the first occurrence of each bit pattern of the three coordinates.  Non-finite: upstream's four flag rules.
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static inline int neighbour(const float* p, const float* q, float thr, int mode) {
    const float d0 = p[0] - q[0], d1 = p[1] - q[1], d2 = p[2] - q[2];
    float dist;
    if (mode == 0) {
        dist = fmaf(d2, d2, fmaf(d1, d1, fmaf(d0, d0, 0.f)));
    } else {
        float t = 0.f + d0 * d0;
        t = t + d1 * d1;
        dist = t + d2 * d2;
    }
    return dist <= thr;
}

// counts[i] = the number of neighbours of point i, itself included, stopping at cap (cap <= 0: no cap)
void orc_radius_counts_brute(const float* pts, int64_t n, double radius, int mode, int64_t cap, int64_t* counts) {
    const float r = (float)radius, thr = r * r;
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t i = 0; i < n; ++i) {
        int64_t c = 0;
        for (int64_t j = 0; j < n && (cap <= 0 || c < cap); ++j) c += neighbour(pts + 3 * j, pts + 3 * i, thr, mode);
        counts[i] = c;
    }
}

typedef struct {
    int64_t key;
    int64_t idx;
} KeyIdx;

static int cmp_keyidx(const void* a, const void* b) {
    const KeyIdx *x = a, *y = b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    return x->idx < y->idx ? -1 : (x->idx > y->idx);
}

// the same counts over a grid; returns -1 on a non-finite coordinate or out of memory
int orc_radius_counts_grid(const float* pts, int64_t n, double radius, int mode, int64_t cap, int64_t* counts) {
    if (n == 0) return 0;
    double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int64_t i = 0; i < 3 * n; ++i) {
        if (!isfinite(pts[i])) return -1;
        mn[i % 3] = fmin(mn[i % 3], pts[i]);
        mx[i % 3] = fmax(mx[i % 3], pts[i]);
    }
    double c = radius * (1.0 + 1e-5) * 1.0001;
    int64_t dim[3];
    for (;;) {
        double cells = 1;
        for (int a = 0; a < 3; ++a) {
            dim[a] = (int64_t)floor((mx[a] - mn[a]) / c) + 1;
            cells *= (double)dim[a];
        }
        if (cells < 4e18) break;
        c *= 2;
    }
    KeyIdx* s = malloc((size_t)n * sizeof(KeyIdx));
    if (!s) return -1;
#define CELL(i, a) ((int64_t)floor(((double)pts[3 * (i) + (a)] - mn[a]) / c))
    for (int64_t i = 0; i < n; ++i) {
        s[i].key = (CELL(i, 2) * dim[1] + CELL(i, 1)) * dim[0] + CELL(i, 0);
        s[i].idx = i;
    }
    qsort(s, (size_t)n, sizeof(KeyIdx), cmp_keyidx);
    const float r = (float)radius, thr = r * r;
#pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < n; ++i) {
        const int64_t cx = CELL(i, 0), cy = CELL(i, 1), cz = CELL(i, 2);
        int64_t cnt = 0;
        for (int64_t z = cz - 1; z <= cz + 1; ++z)
            for (int64_t y = cy - 1; y <= cy + 1; ++y)
                for (int64_t x = cx - 1; x <= cx + 1; ++x) {
                    if (x < 0 || y < 0 || z < 0 || x >= dim[0] || y >= dim[1] || z >= dim[2]) continue;
                    const int64_t key = (z * dim[1] + y) * dim[0] + x;
                    int64_t lo = 0, hi = n;   // first entry with s.key >= key
                    while (lo < hi) {
                        const int64_t m = (lo + hi) / 2;
                        if (s[m].key < key) lo = m + 1;
                        else hi = m;
                    }
                    for (int64_t k = lo; k < n && s[k].key == key && (cap <= 0 || cnt < cap); ++k)
                        cnt += neighbour(pts + 3 * s[k].idx, pts + 3 * i, thr, mode);
                }
        counts[i] = cap > 0 && cnt > cap ? cap : cnt;
    }
#undef CELL
    free(s);
    return 0;
}

typedef struct {
    uint32_t k[3];
    int64_t idx;
} BitsIdx;

static int cmp_bitsidx(const void* a, const void* b) {
    const BitsIdx *x = a, *y = b;
    for (int t = 0; t < 3; ++t)
        if (x->k[t] != y->k[t]) return x->k[t] < y->k[t] ? -1 : 1;
    return x->idx < y->idx ? -1 : (x->idx > y->idx);
}

// mask[i] = 1 for the lowest index of every bit pattern; returns -1 when out of memory
int orc_remove_duplicated_points(const float* pts, int64_t n, uint8_t* mask) {
    BitsIdx* s = malloc((size_t)(n > 0 ? n : 1) * sizeof(BitsIdx));
    if (!s) return -1;
    for (int64_t i = 0; i < n; ++i) {
        memcpy(s[i].k, pts + 3 * i, 3 * sizeof(uint32_t));
        s[i].idx = i;
        mask[i] = 0;
    }
    qsort(s, (size_t)n, sizeof(BitsIdx), cmp_bitsidx);
    for (int64_t i = 0; i < n; ++i)
        if (i == 0 || memcmp(s[i].k, s[i - 1].k, sizeof(s[i].k)) != 0) mask[s[i].idx] = 1;
    free(s);
    return 0;
}

// PointCloud.cpp:716-738: IsFinite, IsNan().LogicalNot() or IsInf().LogicalNot(), All over the row; or all true
void orc_remove_non_finite_points(const float* pts, int64_t n, int remove_nan, int remove_inf, uint8_t* mask) {
    for (int64_t i = 0; i < n; ++i) {
        int keep = 1;
        for (int a = 0; a < 3; ++a) {
            const float v = pts[3 * i + a];
            if (remove_nan && remove_inf) keep &= isfinite(v) != 0;
            else if (remove_nan) keep &= !isnan(v);
            else if (remove_inf) keep &= !isinf(v);
        }
        mask[i] = (uint8_t)keep;
    }
}

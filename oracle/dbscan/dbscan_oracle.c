/* dbscan_oracle.c — CPU oracle of DBSCAN clustering (o3db_cluster_dbscan), restating upstream's
 * geometry::PointCloud::ClusterDBSCAN (geometry/PointCloudCluster.cpp:21-97) as DESIGN.md §4.19 writes it out.
 *
 * TEST INFRASTRUCTURE ONLY.
 *   neighbours  j of i iff d2 < eps * eps, d2 = ((0 + dx dx) + dy dy) + dz dz in f64, dx = x_i - x_j (nanoflann's
 *               L2 metric and radius test); found either by a uniform grid of cells of at least eps (OpenMP) or by a
 *               brute force over every point;
 *   core        at least min_points neighbours, the point itself included;
 *   labels      upstream's sequential labelling: in index order, an unlabelled core point starts a cluster, and a
 *               work list spreads it over its neighbours, expanding from core points only; a label >= 0 is never
 *               overwritten.
 * The points must be finite (the device rejects other clouds).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static inline int is_neighbour(const float* q, const float* p, double eps2) {
    const double dx = (double)q[0] - (double)p[0];
    const double dy = (double)q[1] - (double)p[1];
    const double dz = (double)q[2] - (double)p[2];
    double d2 = 0.0;
    d2 += dx * dx;
    d2 += dy * dy;
    d2 += dz * dz;
    return d2 < eps2;
}

/* ------------------------------------------------------------------ neighbour search */

#define AXIS_BITS 21
#define AXIS_CELLS (1 << (AXIS_BITS - 1))   /* cells per axis at most */

typedef struct {
    uint64_t key;
    int64_t idx;
} Entry;

typedef struct {
    const float* pts;
    int64_t n;
    double eps2;
    int brute;
    /* grid */
    double mn[3], c;
    Entry* sorted;        /* points by cell key */
} Search;

static int cmp_entry(const void* a, const void* b) {
    const Entry* x = (const Entry*)a;
    const Entry* y = (const Entry*)b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    return x->idx < y->idx ? -1 : (x->idx > y->idx);
}

static inline int64_t cell_of(const Search* s, const float* p, int a) {
    return (int64_t)floor(((double)p[a] - s->mn[a]) / s->c);
}

static inline uint64_t key_of(int64_t ix, int64_t iy, int64_t iz) {
    return ((uint64_t)ix << (2 * AXIS_BITS)) | ((uint64_t)iy << AXIS_BITS) | (uint64_t)iz;
}

/* Cells of at least eps (1 + 1e-6), and at most AXIS_CELLS per axis, so that a neighbour's cell differs from the
 * query's by at most one along every axis: |dx| < eps (1 + 1e-15), and the cell index of a coordinate is computed to
 * well within 1e-6 of a cell. */
static int search_init(Search* s, const float* pts, int64_t n, double eps, int brute) {
    memset(s, 0, sizeof(*s));
    s->pts = pts;
    s->n = n;
    s->eps2 = eps * eps;
    s->brute = brute;
    if (brute || n == 0) return 0;
    double mx[3];
    for (int a = 0; a < 3; ++a) s->mn[a] = mx[a] = pts[a];
    for (int64_t i = 0; i < n; ++i)
        for (int a = 0; a < 3; ++a) {
            const double v = pts[3 * i + a];
            if (v < s->mn[a]) s->mn[a] = v;
            if (v > mx[a]) mx[a] = v;
        }
    s->c = eps * (1.0 + 1e-6);
    for (int a = 0; a < 3; ++a)
        if ((mx[a] - s->mn[a]) / s->c > AXIS_CELLS - 2) s->c = (mx[a] - s->mn[a]) / (AXIS_CELLS - 2);
    s->sorted = (Entry*)malloc((size_t)n * sizeof(Entry));
    if (!s->sorted) return -1;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        const float* p = pts + 3 * i;
        s->sorted[i].key = key_of(cell_of(s, p, 0), cell_of(s, p, 1), cell_of(s, p, 2));
        s->sorted[i].idx = i;
    }
    qsort(s->sorted, (size_t)n, sizeof(Entry), cmp_entry);
    return 0;
}

static int64_t lower_bound(const Search* s, uint64_t key) {
    int64_t lo = 0, hi = s->n;
    while (lo < hi) {
        const int64_t mid = lo + (hi - lo) / 2;
        if (s->sorted[mid].key < key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

/* Calls visit(j, ctx) for every neighbour j of point i, in no particular order; stops when visit returns 0. */
typedef int (*VisitFn)(int64_t j, void* ctx);

static void for_each_neighbour(const Search* s, int64_t i, VisitFn visit, void* ctx) {
    const float* q = s->pts + 3 * i;
    if (s->brute) {
        for (int64_t j = 0; j < s->n; ++j)
            if (is_neighbour(q, s->pts + 3 * j, s->eps2) && !visit(j, ctx)) return;
        return;
    }
    const int64_t cx = cell_of(s, q, 0), cy = cell_of(s, q, 1), cz = cell_of(s, q, 2);
    for (int64_t ix = cx - 1; ix <= cx + 1; ++ix)
        for (int64_t iy = cy - 1; iy <= cy + 1; ++iy)
            for (int64_t iz = cz - 1; iz <= cz + 1; ++iz) {
                if (ix < 0 || iy < 0 || iz < 0) continue;
                const uint64_t key = key_of(ix, iy, iz);
                for (int64_t k = lower_bound(s, key); k < s->n && s->sorted[k].key == key; ++k) {
                    const int64_t j = s->sorted[k].idx;
                    if (is_neighbour(q, s->pts + 3 * j, s->eps2) && !visit(j, ctx)) return;
                }
            }
}

static int count_visit(int64_t j, void* ctx) {
    (void)j;
    ++*(int64_t*)ctx;
    return 1;
}

/* core[i] = point i has at least min_points neighbours, itself included (PointCloudCluster.cpp:57) */
static void core_flags(const Search* s, int64_t min_points, uint8_t* core) {
#pragma omp parallel for schedule(dynamic, 256)
    for (int64_t i = 0; i < s->n; ++i) {
        int64_t count = 0;
        for_each_neighbour(s, i, count_visit, &count);
        core[i] = count >= min_points;
    }
}

/* ------------------------------------------------------------------ labelling */

typedef struct {
    int64_t* data;
    int64_t size, cap;
    int failed;
} Stack;

static void push(Stack* st, int64_t v) {
    if (st->size == st->cap) {
        const int64_t cap = st->cap ? 2 * st->cap : 1024;
        int64_t* d = (int64_t*)realloc(st->data, (size_t)cap * sizeof(int64_t));
        if (!d) {
            st->failed = 1;
            return;
        }
        st->data = d;
        st->cap = cap;
    }
    st->data[st->size++] = v;
}

typedef struct {
    Stack* st;
    const int32_t* labels;
} PushCtx;

/* push every neighbour; with labels, only those not yet labelled >= 0 */
static int push_visit(int64_t j, void* ctx) {
    PushCtx* c = (PushCtx*)ctx;
    if (!c->labels || c->labels[j] < 0) push(c->st, j);
    return !c->st->failed;
}

/* labels [n]: upstream's labels; core (NULL or [n]): 1 for core points.  Returns the number of clusters, or -1 when
 * memory ran out. */
int64_t orc_dbscan(const float* pts, int64_t n, double eps, int64_t min_points, int brute, int32_t* labels,
                   uint8_t* core_out) {
    Search s;
    if (search_init(&s, pts, n, eps, brute)) return -1;
    uint8_t* core = (uint8_t*)malloc((size_t)(n > 0 ? n : 1));
    if (!core) {
        free(s.sorted);
        return -1;
    }
    core_flags(&s, min_points, core);
    for (int64_t i = 0; i < n; ++i) labels[i] = -2;   /* undefined */
    int32_t cluster = 0;
    Stack st = {0};
    for (int64_t idx = 0; idx < n && !st.failed; ++idx) {
        if (labels[idx] != -2) continue;
        if (!core[idx]) {
            labels[idx] = -1;
            continue;
        }
        labels[idx] = cluster;
        st.size = 0;
        PushCtx all = {&st, NULL};
        for_each_neighbour(&s, idx, push_visit, &all);
        while (st.size > 0 && !st.failed) {
            const int64_t nb = st.data[--st.size];
            if (nb == idx || labels[nb] >= 0) continue;
            labels[nb] = cluster;
            if (core[nb]) {
                PushCtx unlabelled = {&st, labels};
                for_each_neighbour(&s, nb, push_visit, &unlabelled);
            }
        }
        ++cluster;
    }
    const int failed = st.failed;
    if (core_out) memcpy(core_out, core, (size_t)n);
    free(st.data);
    free(core);
    free(s.sorted);
    return failed ? -1 : cluster;
}

/* core flags only: 1 where point i has at least min_points neighbours */
int orc_dbscan_core(const float* pts, int64_t n, double eps, int64_t min_points, int brute, uint8_t* core) {
    Search s;
    if (search_init(&s, pts, n, eps, brute)) return -1;
    core_flags(&s, min_points, core);
    free(s.sorted);
    return 0;
}

/* boundary_oracle.c — CPU restatement of t::geometry::PointCloud::ComputeBoundaryPoints (t/geometry/PointCloud.cpp:
 * 803-853, t/geometry/kernel/PointCloudImpl.h:354-506), Float32 clouds.
 *
 * TEST INFRASTRUCTURE ONLY, like the rest of oracle/: the product never links or calls it.
 *
 * Precision follows the reference's CPU build (g++ -ffp-contract=off):
 *   frame (GetCoordinateSystemOnPlane, :354-379): f32, the branch test fabsf(..) < 1e-6 in f64, 1.0 / sqrtf(..) in f64
 *     rounded to f32, then u = cross_3x1(n, v);
 *   angles (:478-491): atan2(dot_3x1(v, d), dot_3x1(u, d)) with d = p_j - p_i, over the neighbours after the first;
 *   sort: upstream's heap sort (:381-422), ascending;
 *   test (IsBoundaryPoints, :424-440): the largest consecutive gap by std::max from 0, the wrap gap
 *     2*M_PI - a[m-1] + a[0] in f64 rounded to f32, then max_gap > angle_threshold * M_PI / 180.0 in f64.
 * atan2 has two modes:
 *   ORC_ATAN2_LIBM  libm's atan2f, as the reference's object code calls it; checked bit for bit against the reference's
 *                   own code, compiled from its headers into oracle/_ref/libo3dref_boundary.so
 *                   (tests/test_oracle_vs_ref_boundary.py);
 *   ORC_ATAN2_F64   (float)atan2((double)y, (double)x), the device's evaluation.
 * The neighbour lists come from the oracle's hybrid search (oracle/icp_oracle.c), which orders them as the product does.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

enum { ORC_ATAN2_LIBM = 0, ORC_ATAN2_F64 = 1 };

void orc_boundary_frame_f32(const float n[3], float u[3], float v[3]) {
    if (!(fabsf(n[0] - n[2]) < 1e-6) || !(fabsf(n[1] - n[2]) < 1e-6)) {
        const float inv = 1.0 / sqrtf(n[0] * n[0] + n[1] * n[1]);
        v[0] = -1 * n[1] * inv;
        v[1] = n[0] * inv;
        v[2] = 0;
    } else {
        const float inv = 1.0 / sqrtf(n[1] * n[1] + n[2] * n[2]);
        v[0] = 0;
        v[1] = -1 * n[2] * inv;
        v[2] = n[1] * inv;
    }
    u[0] = n[1] * v[2] - n[2] * v[1];
    u[1] = n[2] * v[0] - n[0] * v[2];
    u[2] = n[0] * v[1] - n[1] * v[0];
}

static void heapify(float* a, int n, int root) {
    int largest = root;
    for (;;) {
        const int l = 2 * largest + 1, r = 2 * largest + 2;
        int next = largest;
        if (l < n && a[l] > a[next]) next = l;
        if (r < n && a[r] > a[next]) next = r;
        if (next == largest) break;
        const float t = a[largest];
        a[largest] = a[next];
        a[next] = t;
        largest = next;
    }
}

static void heap_sort(float* a, int n) {
    for (int i = n / 2 - 1; i >= 0; i--) heapify(a, n, i);
    for (int i = n - 1; i > 0; i--) {
        const float t = a[0];
        a[0] = a[i];
        a[i] = t;
        heapify(a, i, 0);
    }
}

/* IsBoundaryPoints over sorted angles[0..m), m >= 1; *max_gap receives max_diff */
int orc_is_boundary_f32(const float* angles, int m, double angle_threshold, float* max_gap) {
    float diff, max_diff = 0;
    for (int i = 0; i < m - 1; i++) {
        diff = angles[i + 1] - angles[i];
        max_diff = max_diff < diff ? diff : max_diff;   /* std::max(max_diff, diff) */
    }
    diff = 2 * M_PI - angles[m - 1] + angles[0];
    max_diff = max_diff < diff ? diff : max_diff;
    if (max_gap) *max_gap = max_diff;
    return max_diff > angle_threshold * M_PI / 180.0;
}

/* the whole function: indices [n, nn_size] and counts [n] of the hybrid search; mask [n] and max_gap [n] (may be
 * NULL) are written for every point, 0 where the point has no neighbour besides its list's first entry */
void orc_compute_boundary_points_f32(const float* pts, const float* nrm, int64_t n, const int32_t* idx, int nn_size,
                                     const int32_t* cnt, double angle_threshold, int mode, uint8_t* mask,
                                     float* max_gap) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        float u[3], v[3], ang[32];
        orc_boundary_frame_f32(nrm + 3 * i, u, v);
        const int m = cnt[i] - 1;
        mask[i] = 0;
        if (max_gap) max_gap[i] = 0.0f;
        if (m <= 0) continue;
        const float* q = pts + 3 * i;
        for (int k = 0; k < m; ++k) {
            const float* r = pts + 3 * (int64_t)idx[i * nn_size + k + 1];
            const float d[3] = {r[0] - q[0], r[1] - q[1], r[2] - q[2]};
            const float y = v[0] * d[0] + v[1] * d[1] + v[2] * d[2];
            const float x = u[0] * d[0] + u[1] * d[1] + u[2] * d[2];
            ang[k] = mode == ORC_ATAN2_LIBM ? atan2f(y, x) : (float)atan2((double)y, (double)x);
        }
        heap_sort(ang, m);
        mask[i] = (uint8_t)orc_is_boundary_f32(ang, m, angle_threshold, max_gap ? max_gap + i : NULL);
    }
}

// pointcloud.cu — t::geometry::PointCloud::VoxelDownSample for sm_90a (SURVEY.md 8f #1: the
// pyramid build that sits directly in front of the ICP loop, Registration.cpp:237-240, 266-269).
//
// Reference (t/geometry/PointCloud.cpp:496-560): voxel = floor(p / voxel_size) (f32), a HashSet
// insert + find to map points to dense voxel ids, then one IndexAdd_ pass per attribute and a
// division by the per-voxel count.  Here: one kernel hashes every point's voxel key into a
// lock-free table (the first point of a voxel claims a dense id), one kernel accumulates all
// attributes with f32 atomics (the reference's IndexAdd_ is f32 too), one divides.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "hash.cuh"
#include "svd3.cuh"
#include "eigen3x3.cuh"

namespace o3db {

static constexpr int kVT = 256;

static constexpr int kMaxAttrs = 4;

struct VdsArgs {
    const float* pos;
    const float* attr[kMaxAttrs];   // extra [n,3] f32 point attributes (normals, colors, color_gradients, ...)
    float* attr_out[kMaxAttrs];
    int nattr;
    int n;
    float voxel_size;
    int* keys;          // [n,3] voxel key of every point
    Table tab;          // committed keys = vkeys
    int* vkeys;         // [n,3] key of every voxel id
    int* counter;       // number of voxels
    int* vid;           // [n] voxel id of the point (filled by the winners in pass 1, by all in pass 2)
    float* pos_out;
    float* cnt;         // [n] points per voxel (f32, as voxel_num_points upstream)
};

// pass 1: voxel keys + claim.  A winner takes the next dense id and publishes it at once.
__global__ void vds_claim_kernel(VdsArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    // PointCloud.cpp:506-507: (positions / voxel_size).Floor().To(Int64) — Float32 division
    const int kx = (int)floorf(__fdiv_rn(a.pos[3 * i], a.voxel_size));
    const int ky = (int)floorf(__fdiv_rn(a.pos[3 * i + 1], a.voxel_size));
    const int kz = (int)floorf(__fdiv_rn(a.pos[3 * i + 2], a.voxel_size));
    a.keys[3 * i] = kx;
    a.keys[3 * i + 1] = ky;
    a.keys[3 * i + 2] = kz;
    __threadfence();   // the key must be visible before a marker can point at it
    unsigned bucket = 0;
    const int r = probe<true>(a.tab, a.keys, i, kx, ky, kz, &bucket);
    int id = -1;
    if (r == kResInserted) {
        id = atomicAdd(a.counter, 1);
        a.vkeys[3 * id] = kx;
        a.vkeys[3 * id + 1] = ky;
        a.vkeys[3 * id + 2] = kz;
        __threadfence();
        atomicExch(&a.tab.table[bucket], id);   // provisional marker -> committed id
    } else if (r >= 0) {
        id = r;
    }
    a.vid[i] = id;   // -1: the voxel was still provisional when this point looked; resolved in pass 2
}

// pass 2: every point adds its attributes to its voxel (IndexAdd_, PointCloud.cpp:536-552).
__global__ void vds_accumulate_kernel(VdsArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    int id = a.vid[i];
    if (id < 0) {
        unsigned bucket;
        id = probe<false>(a.tab, a.keys, 0, a.keys[3 * i], a.keys[3 * i + 1], a.keys[3 * i + 2], &bucket);
    }
    if (id < 0) return;   // cannot happen: every key was inserted in pass 1
    atomicAdd(&a.cnt[id], 1.0f);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        atomicAdd(&a.pos_out[3 * (size_t)id + c], a.pos[3 * (size_t)i + c]);
#pragma unroll
        for (int k = 0; k < kMaxAttrs; ++k)
            if (k < a.nattr) atomicAdd(&a.attr_out[k][3 * (size_t)id + c], a.attr[k][3 * (size_t)i + c]);
    }
}

// pass 3: voxel_attr /= voxel_num_points (PointCloud.cpp:549)
__global__ void vds_divide_kernel(VdsArgs a) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= *a.counter) return;
    const float c = a.cnt[v];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        a.pos_out[3 * (size_t)v + k] = a.pos_out[3 * (size_t)v + k] / c;
#pragma unroll
        for (int t = 0; t < kMaxAttrs; ++t)
            if (t < a.nattr) a.attr_out[t][3 * (size_t)v + k] = a.attr_out[t][3 * (size_t)v + k] / c;
    }
}

}  // namespace o3db

using namespace o3db;

extern "C" int o3db_voxel_down_sample_attrs(const float* positions_dev, const float* const* attrs_dev, int num_attrs,
                                            int64_t n, double voxel_size, float* positions_out_dev,
                                            float* const* attrs_out_dev, int64_t* num_out_host, void* stream) {
    O3DB_REQUIRE(voxel_size > 0, "voxel_size must be positive.");   // PointCloud.cpp:498-500
    O3DB_REQUIRE(n >= 0 && n < INT_MAX / 4, "o3db_voxel_down_sample: bad point count");
    O3DB_REQUIRE(num_out_host != nullptr, "o3db_voxel_down_sample: num_out_host is null");
    O3DB_REQUIRE(num_attrs >= 0 && num_attrs <= kMaxAttrs, "o3db_voxel_down_sample: at most %d extra attributes",
                 kMaxAttrs);
    *num_out_host = 0;
    if (n == 0) return O3DB_OK;
    O3DB_REQUIRE(positions_dev && positions_out_dev, "o3db_voxel_down_sample: null positions");
    O3DB_REQUIRE(num_attrs == 0 || (attrs_dev && attrs_out_dev), "o3db_voxel_down_sample: null attribute list");
    for (int k = 0; k < num_attrs; ++k)
        O3DB_REQUIRE(attrs_dev[k] && attrs_out_dev[k], "o3db_voxel_down_sample: attribute in/out buffers must come in pairs");
    configure_memory_pool();
    cudaStream_t st = (cudaStream_t)stream;
    unsigned nb = 16;
    while ((int64_t)nb < 2 * n) nb <<= 1;
    const size_t b_keys = (size_t)n * 3 * sizeof(int), b_tab = (size_t)nb * sizeof(int), b_vid = (size_t)n * sizeof(int),
                 b_cnt = (size_t)n * sizeof(float);
    DevPtr<char> scratch;
    if (int rc = dev_alloc(scratch, 2 * b_keys + b_tab + b_vid + b_cnt + 64, st)) return rc;
    char* base = scratch.get();
    VdsArgs a{};
    a.pos = positions_dev;
    a.nattr = num_attrs;
    for (int k = 0; k < kMaxAttrs; ++k) {
        a.attr[k] = k < num_attrs ? attrs_dev[k] : nullptr;
        a.attr_out[k] = k < num_attrs ? attrs_out_dev[k] : nullptr;
    }
    a.n = (int)n;
    a.voxel_size = (float)voxel_size;   // scalar operand takes the tensor's dtype (Float32)
    a.keys = (int*)base;
    a.vkeys = (int*)(base + b_keys);
    int* table = (int*)(base + 2 * b_keys);
    a.vid = (int*)(base + 2 * b_keys + b_tab);
    a.cnt = (float*)(base + 2 * b_keys + b_tab + b_vid);
    a.counter = (int*)(base + 2 * b_keys + b_tab + b_vid + b_cnt);
    a.tab = Table{table, nb - 1, a.vkeys};
    a.pos_out = positions_out_dev;
    O3DB_CUDA_CHECK(cudaMemsetAsync(table, 0xff, b_tab, st));
    O3DB_CUDA_CHECK(cudaMemsetAsync(a.cnt, 0, b_cnt + 64, st));   // counts + counter
    O3DB_CUDA_CHECK(cudaMemsetAsync(positions_out_dev, 0, (size_t)n * 3 * sizeof(float), st));
    for (int k = 0; k < num_attrs; ++k)
        O3DB_CUDA_CHECK(cudaMemsetAsync(attrs_out_dev[k], 0, (size_t)n * 3 * sizeof(float), st));
    const unsigned grid = (unsigned)ceil_div(n, kVT);
    vds_claim_kernel<<<grid, kVT, 0, st>>>(a);
    O3DB_LAUNCH_CHECK();
    vds_accumulate_kernel<<<grid, kVT, 0, st>>>(a);
    O3DB_LAUNCH_CHECK();
    vds_divide_kernel<<<grid, kVT, 0, st>>>(a);
    O3DB_LAUNCH_CHECK();
    int m = 0;
    O3DB_CUDA_CHECK(cudaMemcpyAsync(&m, a.counter, sizeof(int), cudaMemcpyDeviceToHost, st));
    O3DB_CUDA_CHECK(cudaStreamSynchronize(st));
    *num_out_host = m;
    return O3DB_OK;
}

extern "C" int o3db_voxel_down_sample(const float* positions_dev, const float* normals_dev, const float* colors_dev,
                                      int64_t n, double voxel_size, float* positions_out_dev, float* normals_out_dev,
                                      float* colors_out_dev, int64_t* num_out_host, void* stream) {
    O3DB_REQUIRE((normals_dev == nullptr) == (normals_out_dev == nullptr) &&
                         (colors_dev == nullptr) == (colors_out_dev == nullptr),
                 "o3db_voxel_down_sample: attribute in/out buffers must come in pairs");
    const float* in[2];
    float* out[2];
    int k = 0;
    if (normals_dev) {
        in[k] = normals_dev;
        out[k++] = normals_out_dev;
    }
    if (colors_dev) {
        in[k] = colors_dev;
        out[k++] = colors_out_dev;
    }
    return o3db_voxel_down_sample_attrs(positions_dev, in, k, n, voxel_size, positions_out_dev, out, num_out_host, stream);
}

// ---------------------------------------------------------------- colour gradients
//
// t::geometry::PointCloud::EstimateColorGradients (PointCloud.cpp:723-767) with the hybrid search
// (PointCloudImpl.h:1066-1165, EstimateColorGradientsUsingHybridSearchCUDA): per point, a 3x3
// least-squares fit of the intensity over the neighbours projected on the tangent plane, plus the
// orthogonality row ((k-1) n) . g = 0.  The normal equations are accumulated in f32 in the
// reference's operation order (no FMA contraction: the system's condition number is ~1e5, so a
// last-bit change of AtA moves the solution by 1e-2).  The 3x3 solve is selectable:
//   O3DB_GRADIENT_SOLVER_REFERENCE (default) — the reference's own solve_svd3x3<float> semantics
//     (core/linalg/kernel/SVD3x3.h: 4-sweep fast SVD), restated in svd3.cuh; results are bit-identical
//     to the reference's CPU kernel on identical inputs;
//   O3DB_GRADIENT_SOLVER_EXACT — the exact pseudo-inverse of the same f32 system (f64 cyclic Jacobi;
//     eigenvalues below 1e-10 dropped as SVD3x3.h:2184-2187 drops singular values).  The fast SVD is
//     off by a median 12 % on these systems (tests/test_oracle_vs_ref.py pins the gap).

namespace o3db {

__device__ inline void solve_sym3x3_pinv(const double Ain[9], const double b[3], double x[3]) {
    double A[3][3], V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) A[i][j] = 0.5 * (Ain[3 * i + j] + Ain[3 * j + i]);
    for (int sweep = 0; sweep < 64; ++sweep) {
        const double off = fabs(A[0][1]) + fabs(A[0][2]) + fabs(A[1][2]);
        if (off < 1e-300) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                if (fabs(A[p][q]) < 1e-300) continue;
                const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
                for (int k = 0; k < 3; ++k) {
                    const double akp = A[k][p], akq = A[k][q];
                    A[k][p] = c * akp - sn * akq;
                    A[k][q] = sn * akp + c * akq;
                }
                for (int k = 0; k < 3; ++k) {
                    const double apk = A[p][k], aqk = A[q][k];
                    A[p][k] = c * apk - sn * aqk;
                    A[q][k] = sn * apk + c * aqk;
                }
                for (int k = 0; k < 3; ++k) {
                    const double vkp = V[k][p], vkq = V[k][q];
                    V[k][p] = c * vkp - sn * vkq;
                    V[k][q] = sn * vkp + c * vkq;
                }
            }
    }
    x[0] = x[1] = x[2] = 0.0;
    for (int i = 0; i < 3; ++i) {
        const double lam = A[i][i];
        if (fabs(lam) < 1e-10) continue;
        const double proj = (V[0][i] * b[0] + V[1][i] * b[1] + V[2][i] * b[2]) / lam;
        for (int k = 0; k < 3; ++k) x[k] += V[k][i] * proj;
    }
}

#define MUL(a, b) __fmul_rn(a, b)
#define ADD(a, b) __fadd_rn(a, b)
#define SUB(a, b) __fsub_rn(a, b)

__device__ __forceinline__ float intensity3(const float* c) { return (float)((ADD(ADD(c[0], c[1]), c[2])) / 3.0); }

template <int SOLVER>
__global__ void color_gradient_kernel(const float* __restrict__ pts, const float* __restrict__ nrm,
                                      const float* __restrict__ col, const int32_t* __restrict__ idx,
                                      const int32_t* __restrict__ cnt, int64_t n, int max_nn,
                                      float* __restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t o = 3 * i;
    const int count = cnt[i];
    if (count < 4) {   // PointCloudImpl.h:1086-1090
        out[o] = out[o + 1] = out[o + 2] = 0.f;
        return;
    }
    const float vt[3] = {pts[o], pts[o + 1], pts[o + 2]};
    const float nt[3] = {nrm[o], nrm[o + 1], nrm[o + 2]};
    const float it = intensity3(col + o);
    float AtA[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, Atb[3] = {0, 0, 0};
    const float s = ADD(ADD(MUL(vt[0], nt[0]), MUL(vt[1], nt[1])), MUL(vt[2], nt[2]));
    const int32_t* my = idx + i * max_nn;
    int k = 1;   // neighbour 0 is the point itself
    for (; k < count; ++k) {
        const int64_t a = 3 * (int64_t)my[k];
        const float va[3] = {pts[a], pts[a + 1], pts[a + 2]};
        const float d = SUB(ADD(ADD(MUL(va[0], nt[0]), MUL(va[1], nt[1])), MUL(va[2], nt[2])), s);
        const float vp[3] = {SUB(va[0], MUL(d, nt[0])), SUB(va[1], MUL(d, nt[1])), SUB(va[2], MUL(d, nt[2]))};
        const float ia = intensity3(col + a);
        const float A[3] = {SUB(vp[0], vt[0]), SUB(vp[1], vt[1]), SUB(vp[2], vt[2])};
        AtA[0] = ADD(AtA[0], MUL(A[0], A[0]));
        AtA[1] = ADD(AtA[1], MUL(A[1], A[0]));
        AtA[2] = ADD(AtA[2], MUL(A[2], A[0]));
        AtA[4] = ADD(AtA[4], MUL(A[1], A[1]));
        AtA[5] = ADD(AtA[5], MUL(A[2], A[1]));
        AtA[8] = ADD(AtA[8], MUL(A[2], A[2]));
        const float b = SUB(ia, it);
        Atb[0] = ADD(Atb[0], MUL(A[0], b));
        Atb[1] = ADD(Atb[1], MUL(A[1], b));
        Atb[2] = ADD(Atb[2], MUL(A[2], b));
    }
    // orthogonality constraint, weight (k - 1) (PointCloudImpl.h:1141-1151)
    const float w = (float)(k - 1);
    const float A[3] = {MUL(w, nt[0]), MUL(w, nt[1]), MUL(w, nt[2])};
    AtA[0] = ADD(AtA[0], MUL(A[0], A[0]));
    AtA[1] = ADD(AtA[1], MUL(A[0], A[1]));
    AtA[2] = ADD(AtA[2], MUL(A[0], A[2]));
    AtA[4] = ADD(AtA[4], MUL(A[1], A[1]));
    AtA[5] = ADD(AtA[5], MUL(A[1], A[2]));
    AtA[8] = ADD(AtA[8], MUL(A[2], A[2]));
    AtA[3] = AtA[1];
    AtA[6] = AtA[2];
    AtA[7] = AtA[5];
    if (SOLVER == O3DB_GRADIENT_SOLVER_REFERENCE) {   // PointCloudImpl.h:1163
        float x[3];
        svd3::solve(AtA, Atb, x);
        out[o] = x[0];
        out[o + 1] = x[1];
        out[o + 2] = x[2];
        return;
    }
    double Ad[9], bd[3], xd[3];
    for (int q = 0; q < 9; ++q) Ad[q] = (double)AtA[q];
    for (int q = 0; q < 3; ++q) bd[q] = (double)Atb[q];
    solve_sym3x3_pinv(Ad, bd, xd);
    out[o] = (float)xd[0];
    out[o + 1] = (float)xd[1];
    out[o + 2] = (float)xd[2];
}

#undef MUL
#undef ADD
#undef SUB

}  // namespace o3db

extern "C" int o3db_estimate_color_gradients(const float* positions_dev, const float* normals_dev,
                                             const float* colors_dev, int64_t n, double radius, int max_nn,
                                             float* color_gradients_dev, void* stream) {
    return o3db_estimate_color_gradients_solver(positions_dev, normals_dev, colors_dev, n, radius, max_nn,
                                                O3DB_GRADIENT_SOLVER_REFERENCE, color_gradients_dev, stream);
}

extern "C" int o3db_estimate_color_gradients_solver(const float* positions_dev, const float* normals_dev,
                                                    const float* colors_dev, int64_t n, double radius, int max_nn,
                                                    int solver, float* color_gradients_dev, void* stream) {
    using namespace o3db;
    O3DB_REQUIRE(solver == O3DB_GRADIENT_SOLVER_REFERENCE || solver == O3DB_GRADIENT_SOLVER_EXACT,
                 "o3db_estimate_color_gradients: unknown solver");
    O3DB_REQUIRE(n >= 0 && n < INT_MAX, "o3db_estimate_color_gradients: bad point count");
    if (n == 0) return O3DB_OK;
    O3DB_REQUIRE(positions_dev && color_gradients_dev, "o3db_estimate_color_gradients: null positions / output");
    O3DB_REQUIRE(colors_dev != nullptr, "PointCloud must have colors attribute.");     // PointCloud.cpp:727-729
    O3DB_REQUIRE(normals_dev != nullptr, "PointCloud must have normals attribute.");   // PointCloud.cpp:730-733
    O3DB_REQUIRE(radius > 0, "o3db_estimate_color_gradients: the hybrid search needs a positive radius");
    O3DB_REQUIRE(max_nn >= 1 && max_nn <= 32, "o3db_estimate_color_gradients: max_nn must be in 1..32");
    cudaStream_t st = (cudaStream_t)stream;
    o3db_nns* raw = nullptr;
    int rc = o3db_nns_create(positions_dev, n, radius, stream, &raw);
    if (rc) return rc;
    const std::unique_ptr<o3db_nns, HandleDestroy<o3db_nns_destroy>> index(raw);
    DevPtr<int32_t> idx, cnt;
    rc = dev_alloc(idx, (size_t)n * max_nn, st);
    if (rc) return rc;
    rc = dev_alloc(cnt, (size_t)n, st);
    if (rc) return rc;
    rc = o3db_nns_hybrid_search(index.get(), positions_dev, n, radius, max_nn, idx.get(), nullptr, cnt.get(), stream);
    if (rc) return rc;
    const unsigned nb = (unsigned)((n + kVT - 1) / kVT);
    if (solver == O3DB_GRADIENT_SOLVER_REFERENCE)
        color_gradient_kernel<O3DB_GRADIENT_SOLVER_REFERENCE><<<nb, kVT, 0, st>>>(positions_dev, normals_dev, colors_dev, idx.get(),
                                                                                 cnt.get(), n, max_nn, color_gradients_dev);
    else
        color_gradient_kernel<O3DB_GRADIENT_SOLVER_EXACT><<<nb, kVT, 0, st>>>(positions_dev, normals_dev, colors_dev, idx.get(),
                                                                             cnt.get(), n, max_nn, color_gradients_dev);
    O3DB_LAUNCH_CHECK();
    cudaStreamSynchronize(st);   // the index is destroyed on return; its buffers must outlive the kernels
    return O3DB_OK;
}

// ---------------------------------------------------------------- normals
//
// t::geometry::PointCloud::EstimateNormals with the hybrid search (PointCloud.cpp:856-984): the hybrid search of the
// cloud on itself, then one kernel that does per point what upstream does in two passes over a transient
// "covariances" attribute:
//   EstimatePointWiseRobustNormalizedCovarianceKernel (PointCloudImpl.h:512-586) — centroid and six cumulants in f64
//     in neighbour-list order, Bessel's correction, stored f32; fewer than 3 neighbours give the identity.  With the
//     same neighbour lists and no FMA contraction (__dadd_rn / __dmul_rn) this is bit-identical to the reference;
//   EstimatePointWiseNormalsWithFastEigen3x3<float> (:746-1009) — f32, in the reference CPU build's operation order,
//     with q, p and the angle in f64 where upstream's double literals put them; acos and cos are evaluated in f64
//     and rounded to f32 (a correctly rounded acosf / cosf; the reference calls libm's, which are not);
//   the orientation of EstimateNormalsFromCovariances (:1011-1065).
// One thread per point; the neighbour rows are read twice (centroid, cumulants), the second time from L1.

namespace o3db {

#define MUL(a, b) __fmul_rn(a, b)
#define ADD(a, b) __fadd_rn(a, b)
#define SUB(a, b) __fsub_rn(a, b)
#define DIV(a, b) __fdiv_rn(a, b)

__global__ void __launch_bounds__(kVT) normals_kernel(const float* __restrict__ pts, const int32_t* __restrict__ idx,
                                                      const int32_t* __restrict__ cnt, int64_t n, int max_nn,
                                                      int has_normals, float* __restrict__ nrm,
                                                      float* __restrict__ cov_out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int count = cnt[i];
    float C[9] = {1.0f, 0.0f, 0.0f, 0.0f, 1.0f, 0.0f, 0.0f, 0.0f, 1.0f};
    if (count >= 3) {
        const int32_t* my = idx + i * max_nn;
        double c0 = 0.0, c1 = 0.0, c2 = 0.0;
        for (int k = 0; k < count; ++k) {
            const int64_t a = 3 * (int64_t)my[k];
            c0 = __dadd_rn(c0, (double)pts[a]);
            c1 = __dadd_rn(c1, (double)pts[a + 1]);
            c2 = __dadd_rn(c2, (double)pts[a + 2]);
        }
        c0 = __ddiv_rn(c0, (double)count);
        c1 = __ddiv_rn(c1, (double)count);
        c2 = __ddiv_rn(c2, (double)count);
        double sxx = 0.0, syy = 0.0, szz = 0.0, sxy = 0.0, sxz = 0.0, syz = 0.0;
        for (int k = 0; k < count; ++k) {
            const int64_t a = 3 * (int64_t)my[k];
            const double x = __dsub_rn((double)pts[a], c0), y = __dsub_rn((double)pts[a + 1], c1),
                         z = __dsub_rn((double)pts[a + 2], c2);
            sxx = __dadd_rn(sxx, __dmul_rn(x, x));
            syy = __dadd_rn(syy, __dmul_rn(y, y));
            szz = __dadd_rn(szz, __dmul_rn(z, z));
            sxy = __dadd_rn(sxy, __dmul_rn(x, y));
            sxz = __dadd_rn(sxz, __dmul_rn(x, z));
            syz = __dadd_rn(syz, __dmul_rn(y, z));
        }
        const double f = (double)(count - 1);   // Bessel's correction
        C[0] = (float)__ddiv_rn(sxx, f);
        C[4] = (float)__ddiv_rn(syy, f);
        C[8] = (float)__ddiv_rn(szz, f);
        C[1] = C[3] = (float)__ddiv_rn(sxy, f);
        C[2] = C[6] = (float)__ddiv_rn(sxz, f);
        C[5] = C[7] = (float)__ddiv_rn(syz, f);
    }
    if (cov_out) {
#pragma unroll
        for (int k = 0; k < 9; ++k) cov_out[9 * i + k] = C[k];
    }
    float v[3];
    normal_from_covariance(C, v);
    const int64_t o = 3 * i;
    if (has_normals) {   // flip where the new normal points against the prior one; a zero normal stays zero
        if (dot3_rn(nrm + o, v) < 0.0f) {
            v[0] = -v[0];
            v[1] = -v[1];
            v[2] = -v[2];
        }
    } else if (dot3_rn(v, v) == 0.0f) {
        v[0] = 0.0f;
        v[1] = 0.0f;
        v[2] = 1.0f;
    }
    nrm[o] = v[0];
    nrm[o + 1] = v[1];
    nrm[o + 2] = v[2];
}

// OrientNormalsToAlignWithDirection (PointCloudImpl.h:261-294)
__global__ void __launch_bounds__(kVT) orient_direction_kernel(float* __restrict__ nrm, int64_t n, float dx, float dy,
                                                               float dz) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float* v = nrm + 3 * i;
    const float d[3] = {dx, dy, dz};
    const float x = v[0], y = v[1], z = v[2];
    if (__fsqrt_rn(dot3_rn(v, v)) == 0.0f) {
        v[0] = dx;
        v[1] = dy;
        v[2] = dz;
    } else if (dot3_rn(v, d) < 0.0f) {
        v[0] = -x;
        v[1] = -y;
        v[2] = -z;
    }
}

// OrientNormalsTowardsCameraLocation (PointCloudImpl.h:296-351)
__global__ void __launch_bounds__(kVT) orient_camera_kernel(const float* __restrict__ pts, float* __restrict__ nrm,
                                                            int64_t n, float cx, float cy, float cz) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float* v = nrm + 3 * i;
    const float* p = pts + 3 * i;
    const float r[3] = {SUB(cx, p[0]), SUB(cy, p[1]), SUB(cz, p[2])};
    if (__fsqrt_rn(dot3_rn(v, v)) == 0.0f) {
        const float norm_new = __fsqrt_rn(dot3_rn(r, r));
        if (norm_new == 0.0f) {
            v[0] = 0.0f;
            v[1] = 0.0f;
            v[2] = 1.0f;
        } else {
            v[0] = DIV(r[0], norm_new);
            v[1] = DIV(r[1], norm_new);
            v[2] = DIV(r[2], norm_new);
        }
    } else if (dot3_rn(v, r) < 0.0f) {
        v[0] = -v[0];
        v[1] = -v[1];
        v[2] = -v[2];
    }
}

#undef MUL
#undef ADD
#undef SUB
#undef DIV

}  // namespace o3db

extern "C" int o3db_estimate_normals(const float* positions_dev, int64_t n, double radius, int max_nn, int has_normals,
                                     float* normals_dev, float* covariances_dev, void* stream) {
    using namespace o3db;
    O3DB_REQUIRE(n >= 0 && n < INT_MAX / 3, "o3db_estimate_normals: bad point count");
    if (n == 0) return O3DB_OK;
    O3DB_REQUIRE(positions_dev && normals_dev, "o3db_estimate_normals: null positions / normals");
    O3DB_REQUIRE(radius > 0, "o3db_estimate_normals: the hybrid search needs a positive radius");
    O3DB_REQUIRE(max_nn >= 1 && max_nn <= 32, "o3db_estimate_normals: max_nn must be in 1..32");
    cudaStream_t st = (cudaStream_t)stream;
    o3db_nns* raw = nullptr;
    int rc = o3db_nns_create(positions_dev, n, radius, stream, &raw);
    if (rc) return rc;
    const std::unique_ptr<o3db_nns, HandleDestroy<o3db_nns_destroy>> index(raw);
    DevPtr<int32_t> idx, cnt;
    rc = dev_alloc(idx, (size_t)n * max_nn, st);
    if (rc) return rc;
    rc = dev_alloc(cnt, (size_t)n, st);
    if (rc) return rc;
    rc = o3db_nns_hybrid_search(index.get(), positions_dev, n, radius, max_nn, idx.get(), nullptr, cnt.get(), stream);
    if (rc) return rc;
    const unsigned nb = (unsigned)((n + kVT - 1) / kVT);
    normals_kernel<<<nb, kVT, 0, st>>>(positions_dev, idx.get(), cnt.get(), n, max_nn, has_normals ? 1 : 0, normals_dev,
                                       covariances_dev);
    O3DB_LAUNCH_CHECK();
    cudaStreamSynchronize(st);   // the index is destroyed on return; its buffers must outlive the kernels
    return O3DB_OK;
}

extern "C" int o3db_orient_normals_to_align_with_direction(float* normals_dev, int64_t n, const float direction_host[3],
                                                           void* stream) {
    using namespace o3db;
    O3DB_REQUIRE(n >= 0 && n < INT_MAX / 3, "o3db_orient_normals_to_align_with_direction: bad point count");
    O3DB_REQUIRE(direction_host != nullptr, "o3db_orient_normals_to_align_with_direction: null direction");
    if (n == 0) return O3DB_OK;
    O3DB_REQUIRE(normals_dev != nullptr, "No normals in the PointCloud. Call EstimateNormals() first.");
    cudaStream_t st = (cudaStream_t)stream;
    orient_direction_kernel<<<(unsigned)ceil_div(n, kVT), kVT, 0, st>>>(normals_dev, n, direction_host[0],
                                                                        direction_host[1], direction_host[2]);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

extern "C" int o3db_orient_normals_towards_camera_location(const float* positions_dev, float* normals_dev, int64_t n,
                                                           const float camera_host[3], void* stream) {
    using namespace o3db;
    O3DB_REQUIRE(n >= 0 && n < INT_MAX / 3, "o3db_orient_normals_towards_camera_location: bad point count");
    O3DB_REQUIRE(camera_host != nullptr, "o3db_orient_normals_towards_camera_location: null camera location");
    if (n == 0) return O3DB_OK;
    O3DB_REQUIRE(positions_dev != nullptr, "o3db_orient_normals_towards_camera_location: null positions");
    O3DB_REQUIRE(normals_dev != nullptr, "No normals in the PointCloud. Call EstimateNormals() first.");
    cudaStream_t st = (cudaStream_t)stream;
    orient_camera_kernel<<<(unsigned)ceil_div(n, kVT), kVT, 0, st>>>(positions_dev, normals_dev, n, camera_host[0],
                                                                     camera_host[1], camera_host[2]);
    O3DB_LAUNCH_CHECK();
    return O3DB_OK;
}

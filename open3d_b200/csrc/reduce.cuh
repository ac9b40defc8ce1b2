// reduce.cuh — the 29(+1)-scalar Gauss-Newton reduction shared by the ICP kernels (icp.cu) and RGB-D
// odometry (odometry.cu): per-thread f32 partials -> f64 warp tree -> per-warp shared-memory slots ->
// per-block partials -> last block (atomic ticket) sums in block order, with reduce_sums the whole loop of the
// stand-alone reductions; plus the f64 6x6 solve and pose -> transformation that the reference runs on the host
// (kernel/TransformationConverter.cpp), and the on-device Gauss-Newton step built from them
// (gauss_newton_step_warp, left_multiply_warp) that the fused ICP and odometry loops run on one warp; and the
// point-to-point estimator's terms in the same slots with its f64 Kabsch step (kabsch_step_warp).
#pragma once

#include <utility>

#include "common.cuh"

namespace o3db {

static constexpr int kThreads = 256;
static constexpr int kNumSums = 30;   // 29 reference slots + sum of dist^2
static constexpr int kSumStride = 32;
static constexpr int kFlushEvery = 32;   // f32 terms per thread before the f64 tree (error <= kFlushEvery * 2^-24 of sum|term|)

// ------------------------------------------------- 29(+1)-scalar reduction

// Per-thread f32 partials (at most kFlushEvery terms each) -> f64 warp tree ->
// per-warp f64 slots in shared memory.  Deterministic for a fixed launch shape.
__device__ __forceinline__ void flush_acc(float (&acc)[kNumSums], double (*s_warp)[kSumStride]) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kNumSums; ++k) {
        const double v = warp_sum((double)acc[k]);
        if (lane == 0) s_warp[w][k] += v;
        acc[k] = 0.f;
    }
}

// Transposed warp reduction (the fused ICP kernels): every lane brings one query's 30 terms, lane l leaves
// with the sum over the warp of term l.  Five exchange steps; in step `half` a lane keeps one half of its
// remaining terms and trades the other half with lane ^ half, so a term costs one shuffle in total
// (16 + 8 + 4 + 2 + 1 = 31 shuffles for 32 slots) instead of five, and the running totals of a warp live in
// ONE register per lane instead of 30: the search keeps the register file.  The association is a fixed
// binary tree over the lanes: deterministic.
// Every index into v[] is a template argument, not a loop counter, so the array stays in registers whatever the
// unroller decides.  Written as nested loops over `half`, the sm_90a build kept v[] (and the callers' term arrays) in
// local memory: 176 B of stack per thread, stored and reloaded through L1 / L2 for every 32-query chunk, which made the
// ICP iteration 3.3x slower on an H100 (tests/test_local_memory.py guards against it).
template <int HALF, int... K>
__device__ __forceinline__ void warp_transpose_step(float (&v)[32], bool up, std::integer_sequence<int, K...>) {
    ((v[K] = (up ? v[K + HALF] : v[K]) + __shfl_xor_sync(0xffffffffu, up ? v[K] : v[K + HALF], HALF)), ...);
}
template <int HALF>
__device__ __forceinline__ void warp_transpose_steps(float (&v)[32], unsigned lane) {
    // step HALF: lane keeps v[k + HALF] (upper lane) or v[k] (lower lane) and adds what lane ^ HALF sends, k < HALF
    warp_transpose_step<HALF>(v, (lane & HALF) != 0, std::make_integer_sequence<int, HALF>{});
    if constexpr (HALF > 1) warp_transpose_steps<HALF / 2>(v, lane);
}
__device__ __forceinline__ float warp_transpose_sum32(float (&v)[32]) {
    warp_transpose_steps<16>(v, threadIdx.x & 31u);
    return v[0];
}

// Block epilogue: per-warp slots -> block partial -> (last block) grand total in
// block-index order.  Returns true in the last block, with s_final[] filled.
template <int THREADS = kThreads>
__device__ __forceinline__ bool block_reduce_to_global(double (*s_warp)[kSumStride], double* __restrict__ partials,
                                                       unsigned* ticket, double* s_final) {
    __shared__ bool s_last;
    __syncthreads();
    if (threadIdx.x < kNumSums) {
        double v = 0;
#pragma unroll
        for (int w = 0; w < THREADS / 32; ++w) v += s_warp[w][threadIdx.x];
        partials[(size_t)blockIdx.x * kSumStride + threadIdx.x] = v;
    }
    __threadfence();   // release of the block partial before the ticket
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!s_last) return false;
    __threadfence();   // acquire of everybody's partials after it
    // Grand total by the WHOLE block (round 1 had 30 threads walk all per-block partials one dependent
    // L2 round trip at a time: ~130k cycles for 444 blocks, a third of the kernel): warp w sums the blocks
    // b = w, w + 8, ... for all 30 columns (lane = column, 256-byte coalesced rows, 8 loads in flight),
    // then thread k adds the 8 per-warp totals in warp order.  The association is fixed by the launch
    // shape, so the result is still deterministic for a given grid.
    __shared__ double s_part[THREADS / 32][kSumStride];
    {
        const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        constexpr int kW = THREADS / 32, kU = 8;
        double v = 0;
        for (unsigned b = w; b < gridDim.x; b += kU * kW) {   // kU loads in flight, also in the last (partial) batch
            double t[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const unsigned bb = b + u * kW;
                t[u] = bb < gridDim.x ? __ldcg(&partials[(size_t)bb * kSumStride + lane]) : 0.0;
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) v += t[u];
        }
        s_part[w][lane] = v;
    }
    __syncthreads();
    if (threadIdx.x < kNumSums) {
        double v = 0;
#pragma unroll
        for (int w = 0; w < THREADS / 32; ++w) v += s_part[w][threadIdx.x];
        s_final[threadIdx.x] = v;
    }
    if (threadIdx.x == 0) *ticket = 0;
    __syncthreads();
    return true;
}

// The whole reduction of a kThreads-thread block over elements [0, n): a grid-stride loop in which each thread calls
// body(i, acc) for its element i < n of every kThreads-wide stride, body adding that element's terms to the f32
// partials acc; flush_acc into s_warp (zeroed here) every kFlushEvery strides and once at the end; then
// block_reduce_to_global.  All threads of the block must call it.  Returns true in the last block, with s_final[] filled.
template <typename Body>
__device__ __forceinline__ bool reduce_sums(int64_t n, double (*s_warp)[kSumStride], double* __restrict__ partials,
                                            unsigned* ticket, double* s_final, Body&& body) {
    for (int k = threadIdx.x; k < (kThreads / 32) * kSumStride; k += kThreads) (&s_warp[0][0])[k] = 0.0;
    __syncthreads();
    float acc[kNumSums];
#pragma unroll
    for (int k = 0; k < kNumSums; ++k) acc[k] = 0.f;
    int since = 0;
    for (int64_t base = (int64_t)blockIdx.x * kThreads; base < n; base += (int64_t)gridDim.x * kThreads) {
        const int64_t i = base + threadIdx.x;
        if (i < n) body(i, acc);
        if (++since == kFlushEvery) {
            flush_acc(acc, s_warp);
            since = 0;
        }
    }
    flush_acc(acc, s_warp);
    return block_reduce_to_global(s_warp, partials, ticket, s_final);
}

// --------------------------------------------------------- 6x6 solve (f64)

// TransformationConverter.cpp:189-226: LU with partial pivoting (LAPACK dgesv semantics).
__device__ __host__ inline bool solve6x6(const double* A, double* x) {
    double M[6][7];
    for (int j = 0; j < 6; ++j) {
        const int base = (j * (j + 1)) / 2;
        for (int k = 0; k <= j; ++k) {
            M[j][k] = A[base + k];
            M[k][j] = A[base + k];
        }
        M[j][6] = -A[21 + j];
    }
    for (int c = 0; c < 6; ++c) {
        int piv = c;
        double best = fabs(M[c][c]);
        for (int r = c + 1; r < 6; ++r)
            if (fabs(M[r][c]) > best) {
                best = fabs(M[r][c]);
                piv = r;
            }
        if (!(best > 0.0)) return false;
        if (piv != c)
            for (int k = 0; k < 7; ++k) {
                const double t = M[c][k];
                M[c][k] = M[piv][k];
                M[piv][k] = t;
            }
        for (int r = c + 1; r < 6; ++r) {
            const double f = M[r][c] / M[c][c];
            for (int k = c; k < 7; ++k) M[r][k] -= f * M[c][k];
        }
    }
    for (int r = 5; r >= 0; --r) {
        double s = M[r][6];
        for (int k = r + 1; k < 6; ++k) s -= M[r][k] * x[k];
        x[r] = s / M[r][r];
    }
    return true;
}

// The same factorisation by one warp (the fused loops run it in the serial tail of every iteration, where
// a single thread walking a 6 x 7 array in local memory cost ~5 us): lane c < 7 owns column c of the augmented
// matrix in registers; per elimination step the pivot choice and the five multipliers are computed by the
// owner of the pivot column and broadcast, every lane updates its own column.  Same operations on the same
// operands as solve6x6 up to the back substitution, which runs column-oriented (as LAPACK's dtrsv does) from
// shared memory on lane 0.  Must be called by all 32 lanes of a warp; `Ms` is 42 doubles of shared memory.
// Returns false (on every lane) for a singular system.
__device__ __forceinline__ bool solve6x6_warp(const double* __restrict__ A, double* __restrict__ Ms, double* x) {
    const int lane = threadIdx.x & 31;
    const int c_own = lane < 7 ? lane : 6;
    double col[6];
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        const int hi = r > c_own ? r : c_own, lo = r > c_own ? c_own : r;
        col[r] = c_own == 6 ? -A[21 + r] : A[(hi * (hi + 1)) / 2 + lo];
    }
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 6; ++c) {
        int piv = c;
        double best = fabs(col[c]);
#pragma unroll
        for (int r = c + 1; r < 6; ++r)
            if (fabs(col[r]) > best) {
                best = fabs(col[r]);
                piv = r;
            }
        piv = __shfl_sync(0xffffffffu, piv, c);
        best = __shfl_sync(0xffffffffu, best, c);
        if (!(best > 0.0)) ok = false;
#pragma unroll
        for (int r = c + 1; r < 6; ++r)
            if (piv == r) {
                const double t = col[c];
                col[c] = col[r];
                col[r] = t;
            }
#pragma unroll
        for (int r = c + 1; r < 6; ++r) {
            const double f = __shfl_sync(0xffffffffu, col[r] / col[c], c);
            col[r] -= f * col[c];
        }
    }
    if (lane < 7) {
#pragma unroll
        for (int r = 0; r < 6; ++r) Ms[r * 7 + lane] = col[r];
    }
    __syncwarp();
    if (lane == 0 && ok) {
        double b[6];
#pragma unroll
        for (int r = 0; r < 6; ++r) b[r] = Ms[r * 7 + 6];
#pragma unroll
        for (int k = 5; k >= 0; --k) {
            const double xk = b[k] / Ms[k * 7 + k];
            x[k] = xk;
#pragma unroll
            for (int r = 0; r < k; ++r) b[r] -= Ms[r * 7 + k] * xk;
        }
    }
    __syncwarp();
    return ok;
}

// TransformationConverterImpl.h:22-42 + TransformationConverter.cpp:81-104.  The trigonometric values come in as
// arguments so that a warp can evaluate the six sin / cos calls on six lanes (odometry.cu) and still run the very
// same expressions as the single-thread path.
__device__ __host__ inline void pose_to_T_trig(const double* p, double ca, double sa, double cb, double sb, double cg,
                                               double sg, double* T) {
    T[0] = cg * cb;
    T[1] = -1 * sg * ca + cg * sb * sa;
    T[2] = sg * sa + cg * sb * ca;
    T[3] = p[3];
    T[4] = sg * cb;
    T[5] = cg * ca + sg * sb * sa;
    T[6] = -1 * cg * sa + sg * sb * ca;
    T[7] = p[4];
    T[8] = -1 * sb;
    T[9] = cb * sa;
    T[10] = cb * ca;
    T[11] = p[5];
    T[12] = T[13] = T[14] = 0.0;
    T[15] = 1.0;
}

__device__ __host__ inline void pose_to_T(const double* p, double* T) {
    pose_to_T_trig(p, cos(p[0]), sin(p[0]), cos(p[1]), sin(p[1]), cos(p[2]), sin(p[2]), T);
}

// -------------------------------------------------- Gauss-Newton step on one warp

// The on-device part of one Gauss-Newton step, by ONE warp (all 32 lanes must call it): the 29 f64 sums ->
// solve6x6_warp -> the six cos / sin of the pose on six lanes -> the update U = pose_to_T_trig on lane 0.
// `scratch` is 64 doubles of shared memory: the pose in [0, 6), cos a, cos b, cos g, sin a, sin b, sin g in [8, 14),
// the solve's matrix in [16, 58), and U in [16, 32) (the matrix is dead by then), where the caller reads it.
// Returns false on every lane for a singular system, and then leaves U unwritten.
__device__ __forceinline__ bool gauss_newton_step_warp(const double* sums, double* scratch) {
    const int lane = threadIdx.x & 31;
    double* pose = scratch;
    double* trig = scratch + 8;
    if (!solve6x6_warp(sums, scratch + 16, pose)) return false;
    if (lane < 3) trig[lane] = cos(pose[lane]);
    else if (lane < 6) trig[lane] = sin(pose[lane - 3]);
    __syncwarp();
    if (lane == 0) pose_to_T_trig(pose, trig[0], trig[3], trig[1], trig[4], trig[2], trig[5], scratch + 16);
    __syncwarp();
    return true;
}

// -------------------------------------------------- Kabsch step on one warp (point-to-point)

// Point-to-point slot layout of the 32-wide sum array, about a fixed pivot c (s' = s - c, t' = t - c in f32):
//   [3 j + k] sum of t'_j s'_k (j, k < 3),  [9 + k] sum of s'_k,  [12 + k] sum of t'_k,  [28] count,  [29] sum of d^2.
// Raw moments about a fixed point are linear over chunks, shards and ranks, unlike the reference's two-pass centred
// sums (RegistrationCPU.cpp:497-617), which they reproduce: Sxy = M / n - mean(t') mean(s')^T.
static constexpr int kP2pSourceSum = 9, kP2pTargetSum = 12, kCountSlot = 28;

template <int NACC>
__device__ __forceinline__ void accumulate_p2point(float (&acc)[NACC], const float (&s)[3], const float (&t)[3]) {
#pragma unroll
    for (int j = 0; j < 3; ++j) {
#pragma unroll
        for (int k = 0; k < 3; ++k) acc[3 * j + k] += t[j] * s[k];
        acc[kP2pSourceSum + j] += s[j];
        acc[kP2pTargetSum + j] += t[j];
    }
    acc[kCountSlot] += 1.0f;
}

// One Jacobi rotation of columns P and Q of G (and of V) that makes the two columns of G orthogonal; returns whether
// it had anything to do.  The indices are template arguments so that both matrices stay in registers.
template <int P, int Q>
__device__ __forceinline__ bool jacobi_orthogonalize_columns(double (&G)[3][3], double (&V)[3][3]) {
    double alpha = 0, beta = 0, gamma = 0;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        alpha += G[r][P] * G[r][P];
        beta += G[r][Q] * G[r][Q];
        gamma += G[r][P] * G[r][Q];
    }
    if (!(gamma * gamma > 1e-32 * alpha * beta)) return false;   // orthogonal to f64 precision (or a zero column)
    const double zeta = (beta - alpha) / (2.0 * gamma);
    const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
    const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const double gp = G[r][P], gq = G[r][Q], vp = V[r][P], vq = V[r][Q];
        G[r][P] = c * gp - s * gq;
        G[r][Q] = s * gp + c * gq;
        V[r][P] = c * vp - s * vq;
        V[r][Q] = s * vp + c * vq;
    }
    return true;
}

// The rotation of ComputeRtPointToPointCPU (RegistrationCPU.cpp:619-653): R = U diag(1, 1, sign(det U det V)) V^T for
// the SVD H = U S V^T of the 3 x 3 row-major H, in f64.  One-sided (Hestenes) Jacobi: plane rotations from the right
// make the columns of G = H V orthogonal, so that G = U S.  With i, j the two columns of largest norm,
//   R = u_i v_i^T + u_j v_j^T + (u_i x u_j)(v_i x v_j)^T,
// which is the formula above whatever the sign of the third singular pair (the two signs cancel against the
// determinants), so neither the smallest singular value nor its vectors are ever divided by: a planar cloud (rank 2)
// and a reflection (det H < 0) need no special case.  For rank <= 1 (all matches collinear or coincident) the
// rotation is not unique, upstream's is whatever LAPACK returns, and this one completes the basis with the coordinate
// axis least aligned with u_i: a proper rotation with finite entries.
__device__ inline void kabsch_rotation(const double* H, double* R) {
    double G[3][3], V[3][3];
    double scale = 0;
#pragma unroll
    for (int k = 0; k < 9; ++k) scale = fmax(scale, fabs(H[k]));
    const double inv = scale > 0 ? 1.0 / scale : 0.0;   // (the rotation does not depend on the scale of H)
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            G[r][c] = H[3 * r + c] * inv;
            V[r][c] = r == c ? 1.0 : 0.0;
        }
    for (int sweep = 0; sweep < 40; ++sweep) {   // (converges quadratically: 5-8 sweeps in practice)
        bool any = jacobi_orthogonalize_columns<0, 1>(G, V);
        any |= jacobi_orthogonalize_columns<0, 2>(G, V);
        any |= jacobi_orthogonalize_columns<1, 2>(G, V);
        if (!any) break;
    }
    double n2[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) n2[c] = G[0][c] * G[0][c] + G[1][c] * G[1][c] + G[2][c] * G[2][c];
    // k = the column of smallest norm, (i, j, k) a cyclic shift of (0, 1, 2), then i = the larger of the two
    const int k = (n2[0] <= n2[1] && n2[0] <= n2[2]) ? 0 : (n2[1] <= n2[2] ? 1 : 2);
    double gi[3], gj[3], vi[3], vj[3], ni, nj;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        gi[r] = k == 0 ? G[r][1] : (k == 1 ? G[r][2] : G[r][0]);
        gj[r] = k == 0 ? G[r][2] : (k == 1 ? G[r][0] : G[r][1]);
        vi[r] = k == 0 ? V[r][1] : (k == 1 ? V[r][2] : V[r][0]);
        vj[r] = k == 0 ? V[r][2] : (k == 1 ? V[r][0] : V[r][1]);
    }
    ni = k == 0 ? n2[1] : (k == 1 ? n2[2] : n2[0]);
    nj = k == 0 ? n2[2] : (k == 1 ? n2[0] : n2[1]);
    if (nj > ni) {   // swapping both pairs leaves every term of R as it is
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            double t = gi[r];
            gi[r] = gj[r];
            gj[r] = t;
            t = vi[r];
            vi[r] = vj[r];
            vj[r] = t;
        }
        const double t = ni;
        ni = nj;
        nj = t;
    }
    double ui[3], uj[3];
    if (ni > 0) {
        const double s = 1.0 / sqrt(ni);
#pragma unroll
        for (int r = 0; r < 3; ++r) ui[r] = gi[r] * s;
    } else {   // H = 0
        ui[0] = 1.0;
        ui[1] = ui[2] = 0.0;
    }
    if (!(nj > 1e-28 * ni)) {   // rank <= 1: the axis least aligned with u_i
        const double ax = fabs(ui[0]), ay = fabs(ui[1]), az = fabs(ui[2]);
        gj[0] = (ax <= ay && ax <= az) ? 1.0 : 0.0;
        gj[1] = (gj[0] == 0.0 && ay <= az) ? 1.0 : 0.0;
        gj[2] = (gj[0] == 0.0 && gj[1] == 0.0) ? 1.0 : 0.0;
    }
    {   // u_j: the part of g_j orthogonal to u_i, normalised
        const double d = gj[0] * ui[0] + gj[1] * ui[1] + gj[2] * ui[2];
#pragma unroll
        for (int r = 0; r < 3; ++r) uj[r] = gj[r] - d * ui[r];
        const double s = 1.0 / sqrt(uj[0] * uj[0] + uj[1] * uj[1] + uj[2] * uj[2]);
#pragma unroll
        for (int r = 0; r < 3; ++r) uj[r] *= s;
    }
    const double uk[3] = {ui[1] * uj[2] - ui[2] * uj[1], ui[2] * uj[0] - ui[0] * uj[2], ui[0] * uj[1] - ui[1] * uj[0]};
    const double vk[3] = {vi[1] * vj[2] - vi[2] * vj[1], vi[2] * vj[0] - vi[0] * vj[2], vi[0] * vj[1] - vi[1] * vj[0]};
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) R[3 * r + c] = ui[r] * vi[c] + uj[r] * vj[c] + uk[r] * vk[c];
}

// The on-device part of one point-to-point step, with gauss_newton_step_warp's calling convention: ONE warp (all 32
// lanes must call it), `scratch` the same 64 doubles of shared memory, the update U left in scratch[16, 32).  From the
// f64 totals in the layout above (sums[28] > 0): the means about the pivot, Sxy, kabsch_rotation, and
// t = mean(t) - R mean(s) (RegistrationCPU.cpp:651) mapped back from pivot to world coordinates.  There is no
// singular system for this estimator.  Lane 0 does the arithmetic: it is one dependent chain.
__device__ __forceinline__ void kabsch_step_warp(const double* sums, const float* pivot, double* scratch) {
    if ((threadIdx.x & 31) == 0) {
        const double inv_n = 1.0 / sums[kCountSlot];
        double ms[3], mt[3], H[9];
        double* U = scratch + 16;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            ms[k] = sums[kP2pSourceSum + k] * inv_n;
            mt[k] = sums[kP2pTargetSum + k] * inv_n;
        }
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
            for (int k = 0; k < 3; ++k) H[3 * j + k] = sums[3 * j + k] * inv_n - mt[j] * ms[k];
        double* R = scratch;   // (9 doubles; dead once U is written)
        kabsch_rotation(H, R);
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            double t = mt[j] + (double)pivot[j];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                U[4 * j + k] = R[3 * j + k];
                t -= R[3 * j + k] * (ms[k] + (double)pivot[k]);
            }
            U[4 * j + 3] = t;
        }
        U[12] = U[13] = U[14] = 0.0;
        U[15] = 1.0;
    }
    __syncwarp();
}

// T <- U T for 4 x 4 row-major matrices, by lanes 0-15 of a warp (all sixteen must call it): lane l writes T[l].
__device__ __forceinline__ void left_multiply_warp(const double* U, double* T) {
    const int lane = threadIdx.x & 31, i = lane >> 2, j = lane & 3;
    double v = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) v += U[i * 4 + k] * T[k * 4 + j];
    __syncwarp(0xffffu);   // every lane has read the old T
    T[lane] = v;
}

}  // namespace o3db

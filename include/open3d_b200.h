/*
 * open3d_b200.h — C ABI of the H100-native ICP + TSDF hot path.
 *
 * This is the drop-in boundary: a flat extern "C" surface (plain pointers and
 * sizes, no torch / Open3D types) that Open3D's L2 "thin dispatch" functions
 * (the *CUDA symbols of cpp/open3d/t/pipelines/kernel, t/geometry/kernel,
 * core/nns and core/hashmap) can forward to.  Each entry point cites the
 * reference interface it replaces (paths relative to cpp/open3d/).
 * INTEGRATION.md shows the reference-side stubs.
 *
 * Conventions
 *  - `*_dev` pointers are device memory on the CURRENT CUDA device, contiguous,
 *    row-major; `*_host` pointers are host memory.  Kernels never free inputs.
 *  - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 *    Calls are asynchronous on `stream` unless they return values to the host,
 *    in which case they synchronise that stream (never the device).
 *  - A handle (o3db_knn, o3db_nns, o3db_icp) may be used on another stream than the one it was created on: the
 *    call first waits for the work queued on the creation stream so far (the creation included), and the creation
 *    stream, on which destroy frees the handle's buffers, is ordered after the call.  Nothing of this is done for a
 *    call on the creation stream.  The thread-safety rule below holds here too: no two calls on one handle at once.
 *  - Return value: O3DB_OK (0) or a negative o3db_status; o3db_last_error()
 *    returns a thread-local message.  There is NO CPU fallback: without a CUDA
 *    device every compute entry point fails with O3DB_ERR_CUDA.
 *  - Thread safety: handles are not internally locked; use one handle per host
 *    thread (the reference has the same rule, cf. core/CUDAUtils.cpp:149-172).
 */
#ifndef OPEN3D_B200_H_
#define OPEN3D_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define O3DB_VERSION_MAJOR 0
#define O3DB_VERSION_MINOR 1

typedef enum {
    O3DB_OK = 0,
    O3DB_ERR_INVALID = -1,   /* bad argument (shape, null, range) */
    O3DB_ERR_CUDA = -2,      /* CUDA runtime / launch failure, or no device */
    O3DB_ERR_SINGULAR = -3,  /* singular 6x6 system (reference raises, TransformationConverter.cpp:219-225) */
    O3DB_ERR_CAPACITY = -4,  /* hash map / buffer capacity exceeded */
    O3DB_ERR_NO_BLOCKS = -5, /* "No block is touched in TSDF volume" (VoxelBlockGridCUDA.cu:193-198) */
    O3DB_ERR_COMM = -6,      /* NCCL not available / communicator failure */
    O3DB_ERR_NO_INLIERS = -7 /* "Invalid inlier_count value 0, must be > 0." (odometry/RGBDOdometry.cpp:449-452) */
} o3db_status;

const char* o3db_last_error(void);
int o3db_version(void);
/* Number of kernels launched by this library in this process (all threads). */
uint64_t o3db_kernel_launch_count(void);

/* ------------------------------------------------------------------------
 * Robust kernels — t/pipelines/registration/RobustKernel.h:15-23 (enum order),
 * RobustKernelImpl.h:35-115 (weights).
 * ---------------------------------------------------------------------- */
typedef enum {
    O3DB_ROBUST_L2 = 0, O3DB_ROBUST_L1 = 1, O3DB_ROBUST_HUBER = 2, O3DB_ROBUST_CAUCHY = 3,
    O3DB_ROBUST_GM = 4, O3DB_ROBUST_TUKEY = 5, O3DB_ROBUST_GENERALIZED = 6
} o3db_robust_method;

typedef struct {
    int method;     /* o3db_robust_method */
    double scale;   /* RobustKernel::scaling_parameter_ */
    double shape;   /* RobustKernel::shape_parameter_ */
} o3db_robust_kernel;

/* ------------------------------------------------------------------------
 * Correspondence search — replaces core::nns::BuildSpatialHashTableCUDA<float>
 * (core/nns/FixedRadiusIndex.h:227, FixedRadiusSearchOps.cu:20-58) and
 * core::nns::HybridSearchCUDA<float,int32> (FixedRadiusIndex.h:364,
 * FixedRadiusSearchOps.cu:162-198), i.e. NearestNeighborSearch::HybridIndex /
 * HybridSearch (core/nns/NearestNeighborSearch.cpp:66-91, 144-165).
 * The index owns a cell-sorted float4 copy of the points; `points_dev` may be
 * freed after creation.
 * ---------------------------------------------------------------------- */
typedef struct o3db_nns o3db_nns;

int o3db_nns_create(const float* points_dev /* [M,3] */, int64_t num_points, double radius,
                    void* stream, o3db_nns** out);
void o3db_nns_destroy(o3db_nns* nns);

/* Hybrid search: up to max_knn (1..32) nearest points with dist^2 <= radius^2,
 * ascending; indices padded with -1, distances with 0 (FixedRadiusSearchImpl.cuh:514-631).
 * Exact ties resolve to the lower point index.  `radius` must not exceed the
 * radius the index was built for.  Any output may be NULL. */
int o3db_nns_hybrid_search(const o3db_nns* nns, const float* queries_dev /* [N,3] */,
                           int64_t num_queries, double radius, int max_knn,
                           int32_t* indices_dev /* [N,max_knn] */, float* distances_dev /* [N,max_knn] */,
                           int32_t* counts_dev /* [N] */, void* stream);

/* ------------------------------------------------------------------------
 * Exact k-nearest-neighbour search — replaces core::nns::NearestNeighborSearch::
 * KnnIndex / KnnSearch (core/nns/NearestNeighborSearch.cpp:27-64, 93-113; on the
 * GPU upstream runs core/nns/KnnSearchOps.cu, a brute-force GEMM, and on the CPU
 * NanoFlannIndex::SearchKnn, NanoFlannIndex.cpp:62-118).
 * The index owns a cell-sorted float4 copy of the points whose cell size is
 * chosen from the data (DESIGN.md §4.17); `points_dev` may be freed after
 * creation.  Creation synchronises `stream` once; a search does not.
 * ---------------------------------------------------------------------- */
typedef struct o3db_knn o3db_knn;

enum { O3DB_INDEX_INT32 = 0, O3DB_INDEX_INT64 = 1 };

/* Errors: an empty dataset, a non-finite coordinate. */
int o3db_knn_create(const float* points_dev /* [M,3] */, int64_t num_points, void* stream, o3db_knn** out);
void o3db_knn_destroy(o3db_knn* knn);

/* The k' = min(knn, M) nearest dataset points of every query, knn in 1..32, ascending by
 * (dist^2, index): exact ties resolve to the lower index.  dist^2 is
 * fmaf(dz, dz, fmaf(dy, dy, dx * dx)) with d = point - query.  Indices are Int32 or
 * Int64 (index_dtype), [N,k'] row-major like the distances; a query with a non-finite
 * coordinate gets a row of -1 and 0.  num_queries == 0 is a no-op.  Either output may
 * be NULL. */
int o3db_knn_search(const o3db_knn* knn, const float* queries_dev /* [N,3] */, int64_t num_queries, int knn_k,
                    int index_dtype, void* indices_dev /* [N,k'] */, float* distances_dev /* [N,k'] */,
                    void* stream);

/* The search FPFH's neighbour lists come from (DESIGN.md §4.24): the k' = min(knn, M) nearest dataset points of every
 * query, knn in 1..128, with dist^2 <= (float)radius * (float)radius when radius > 0 (radius == 0: no cap), ascending
 * by (dist^2, index).  indices_dev / distances_dev [N,k'] Int32 / Float32 get -1 / 0 past counts_dev [N].  For
 * knn <= 32 and radius > 0 the lists equal o3db_nns_hybrid_search's; with radius == 0 they equal o3db_knn_search's.
 * A query with a non-finite coordinate returns O3DB_ERR_INVALID; that check synchronises the stream once. */
int o3db_knn_search_lists(const o3db_knn* knn, const float* queries_dev /* [N,3] */, int64_t num_queries, int knn_k,
                          double radius, int32_t* indices_dev, float* distances_dev, int32_t* counts_dev,
                          void* stream);

/* The index's cell size, fine-cell count and coarse-block count (diagnostics). */
int o3db_knn_index_stats(const o3db_knn* knn, double* cell_size, int64_t* num_cells, int64_t* num_blocks);

/* PointCloud::RemoveStatisticalOutliers (t/geometry/PointCloud.cpp:678-714): mask[i] =
 * avg[i] <= (float)(cloud_mean + std_ratio * std), avg[i] = the mean distance to the
 * k' = min(nb_neighbors, n) nearest points (the point itself included).  The two
 * cloud-wide sums are taken in f64 in a fixed order (upstream: f32, in an order that
 * depends on its reduction), so repeated calls are bit-identical; DESIGN.md §4.17 gives
 * every operation.  nb_neighbors in 1..32.  avg_dev may be NULL.  n == 0 is a no-op;
 * n == 1 keeps nothing (the standard deviation is NaN), as upstream.  Synchronises. */
int o3db_remove_statistical_outliers(const float* positions_dev, int64_t n, int nb_neighbors, double std_ratio,
                                     uint8_t* mask_dev /* [n] */, float* avg_dev /* [n] or NULL */, void* stream);

/* PointCloud::ComputeMetrics (t/geometry/PointCloud.cpp:1805-1835, kernel/Metrics.cpp):
 * two 1-NN searches on the device, then the values in the order of `metrics`, FScore
 * giving one value per radius, into values_host (num_values at least that many).  Counts
 * of distances below a radius are exact integers (upstream counts in f32, exact only up
 * to 2^24 points).  Synchronises. */
enum { O3DB_METRIC_CHAMFER = 0, O3DB_METRIC_HAUSDORFF = 1, O3DB_METRIC_FSCORE = 2 };
int o3db_compute_metrics(const float* points1_dev, int64_t n1, const float* points2_dev, int64_t n2,
                         const int* metrics_host, int num_metrics, const float* fscore_radius_host, int num_radius,
                         float* values_host, int64_t num_values, void* stream);

/* ------------------------------------------------------------------------
 * Point-cloud smoothing — t::geometry::PointCloud::SmoothLaplacian / SmoothTaubin /
 * SmoothMLS / SmoothBilateral (t/geometry/PointCloud.cpp:1074-1198, kernel/
 * PointCloudImpl.h:1341-1753), Float32.  The arithmetic is upstream's, in f32 in
 * neighbour-list order; exp is evaluated in f64 and rounded to f32 (DESIGN.md §4.18).
 * out_dev [n,3] must not alias positions_dev.  n == 0 is a no-op.
 * ---------------------------------------------------------------------- */

/* SmoothLaplacian / SmoothTaubin: `iterations` rounds of num_factors (1 or 2) passes,
 * pass j of a round using factors_host[j] (Laplacian: {lambda}; Taubin: {lambda, mu}).
 * Each pass moves every point by factor x (mean of its k' = min(n, max_nn + 1) nearest
 * points other than itself - the point); k' <= 32.  The neighbourhoods are searched
 * again before every pass, over the current positions, unless fixed_neighborhoods,
 * when the first search serves every pass.  iterations == 0 or max_nn <= 0 copies the
 * positions.  Each index build synchronises once. */
int o3db_smooth_laplacian(const float* positions_dev, int64_t n, int64_t iterations, const double* factors_host,
                          int num_factors, int max_nn, int fixed_neighborhoods, float* out_dev, void* stream);

/* SmoothMLS: each point projected onto the plane of the Gaussian-weighted PCA of its
 * neighbours (fewer than 3: unchanged).  radius > 0 and max_nn in 1..32: the hybrid
 * search; radius <= 0: the min(n, max_nn) <= 32 nearest points with weight 1; radius
 * <= 0 and max_nn <= 0 copies the positions; max_nn <= 0 with radius > 0 (upstream's
 * fixed-radius search) is an error.  normals_dev [n,3] (in/out, or NULL): the fitted
 * plane's normal, or the old normal normalised where no plane is fitted. */
int o3db_smooth_mls(const float* positions_dev, int64_t n, double radius, int max_nn, float* out_dev,
                    float* normals_dev, void* stream);

/* SmoothBilateral: each point with more than one hybrid-search neighbour (radius > 0,
 * max_nn in 1..32) becomes the mean of its neighbours weighted by
 * exp(-d^2 / (2 sigma_s^2) - r^2 / (2 sigma_r^2)), r the offset along its normal.
 * sigma_s, sigma_r > 0.  normals_dev is required (upstream estimates missing normals
 * with its KNN-only EstimateNormals, which this build does not have). */
int o3db_smooth_bilateral(const float* positions_dev, const float* normals_dev, int64_t n, double radius, int max_nn,
                          double sigma_s, double sigma_r, float* out_dev, void* stream);

/* ------------------------------------------------------------------------
 * DBSCAN clustering — t::geometry::PointCloud::ClusterDBSCAN (t/geometry/PointCloud.cpp:
 * 1634-1644), which runs geometry::PointCloud::ClusterDBSCAN (geometry/PointCloudCluster.cpp:
 * 21-97) on the host; Float32.  labels_dev [n] receives upstream's labels exactly (DESIGN.md
 * §4.19):
 *   neighbours  j of i iff d2 < eps * eps, d2 = ((0 + dx dx) + dy dy) + dz dz in f64 on the
 *               f32 coordinates, dx = x_i - x_j, no FMA (nanoflann's metric and radius test,
 *               reached through KDTreeFlann::SearchRadius, geometry/KDTreeFlann.cpp:114-135);
 *   core        at least min_points neighbours, the point itself included (:57);
 *   clusters    the connected components of the core points, numbered 0, 1, ... in the
 *               order of each component's smallest index (:50-94);
 *   border      a non-core point with a core neighbour takes the smallest cluster id among
 *               its core neighbours (:76); every other point is noise, -1.
 * Errors, before any CUDA call: null pointers, n < 0 or n >= INT_MAX, eps <= 0 or not finite,
 * min_points < 0; from the index build: a non-finite coordinate.  n == 0 is a no-op.
 * Synchronises once (the index build's bounding box); the launches depend on the arguments
 * only. */
int o3db_cluster_dbscan(const float* positions_dev /* [n,3] */, int64_t n, double eps, int64_t min_points,
                        int32_t* labels_dev /* [n] */, void* stream);

/* ------------------------------------------------------------------------
 * Farthest-point down-sampling — t::geometry::PointCloud::FarthestPointDownSample
 * (t/geometry/PointCloud.cpp:612-648); Float32.  selected_dev [num_samples] receives the
 * selected indices in selection order, the result of this loop bit for bit (DESIGN.md §4.20):
 *   d[j] = +inf for all j;  f = start_index
 *   repeat num_samples times:
 *       select f
 *       for all j: e = ((dx*dx + dy*dy) + dz*dz), dx = x_j - x_f etc., all f32, each op
 *                  rounded, no FMA (upstream's diff, diff * diff and Sum({1}));  d[j] = min(d[j], e)
 *       f = argmax over the points not yet selected of d[j]; ties go to the lowest index
 *           (the rule of the legacy geometry/PointCloud.cpp:543-554, strict >)
 * Unlike upstream, a cloud with fewer distinct positions than num_samples still gives
 * num_samples distinct indices (DESIGN.md §7).  Upstream returns the selected points in
 * ascending index order; sort the indices to get that order.
 * Errors, before any CUDA call: null pointers, n < 0 or n >= INT_MAX, num_samples < 1 or
 * > n, start_index outside [0, n); after the launch: a non-finite coordinate (selected_dev
 * is then unspecified).  One cooperative launch, one grid-wide barrier per sample; the call
 * synchronises the stream once, to read the non-finite flag. */
int o3db_farthest_point_down_sample(const float* positions_dev /* [n,3] */, int64_t n, int64_t num_samples,
                                    int64_t start_index, int32_t* selected_dev /* [num_samples] */, void* stream);

/* ------------------------------------------------------------------------
 * The library's process-global random engine, utility::random (utility/Random.cpp): one std::mt19937, seeded from
 * std::random_device until o3db_random_seed sets it to std::mt19937(seed), as o3d.utility.random.seed does.  Every
 * random operation of the library draws from it, under one mutex.
 * o3db_random_sample_indices draws num_samples rows of sample_size distinct indices into out_host
 * [num_samples][sample_size], upstream's RandomSampler<size_t> (geometry/PointCloudSegmentation.cpp:30-55): each
 * index from std::uniform_int_distribution<size_t>(0, n-1), a repeat within a row redrawn.  Host only. */
int o3db_random_seed(int seed);
int o3db_random_sample_indices(int64_t n, int sample_size, int num_samples, int64_t* out_host);
/* count draws of upstream's UniformIntGenerator<int>(low, high) (utility/Random.h:63-90): each one
 * std::uniform_int_distribution<int>(low, high) from the engine, with replacement; upstream's messages for low < 0 and
 * low > high.  Host only. */
int o3db_random_uniform_ints(int low, int high, int64_t count, int* out_host);

/* ------------------------------------------------------------------------
 * Global registration by RANSAC — pipelines::registration::RegistrationRANSACBasedOnCorrespondence
 * (pipelines/registration/Registration.cpp:195-379) with TransformationEstimationPointToPoint(false) and the checkers
 * of CorrespondenceChecker.cpp, on Float32 clouds.  The result is that of upstream's function run on one thread
 * (DESIGN.md §4.25):
 *   draws       hypothesis i takes ransac_n draws of std::uniform_int_distribution<int>(0, K-1) from the library's
 *               engine, in order, and is drawn only while i < est_k; afterwards the engine has advanced by exactly
 *               stop * ransac_n draws, stop the first i not below est_k;
 *   hypothesis  f64: means as the sums in sample order times 1/ransac_n, the cross-covariance of the demeaned pairs
 *               times 1/ransac_n, the library's Jacobi Kabsch rotation, t = mean_t - R mean_s; every op rounded, no FMA;
 *   checkers    edge length (similarity), distance (threshold) and normal (the cosine of the angle, computed by the
 *               caller with std::cos); the normal checker passes where either normal pointer is null;
 *   validation  the source transformed in f64, ((T_j0 x + T_j1 y) + T_j2 z) + T_j3; its nearest target point by
 *               ((dx^2 + dy^2) + dz^2) in f64, a match when d^2 < max_correspondence_distance^2, ties to the lowest
 *               index; fitness = matches / n, rmse = sqrt(sum d^2 / matches), the sum over tiles of 128 points in
 *               index order, then over the tiles;
 *   selection   upstream's IsBetterRANSACThan and est_k rule from the inlier ratio of all K pairs.
 * transformation_host [16] receives the best transformation, row-major (the identity when nothing won);
 * correspondence_set_dev [n] the best transformation's nearest target point of each source point, -1 for none.
 * Nothing is drawn and the result is the identity with no correspondences when ransac_n < 3, K < ransac_n,
 * max_correspondence_distance <= 0 or max_iteration <= 0.  Errors: a non-finite distance, non-finite positions (the
 * message names remove_non_finite_points), a pair outside [0, n) x [0, m), counts of 2^31 - 1 or more, null pointers.
 * The call synchronises the stream 2 + 2 * batches times, a batch being 8192 hypotheses (fewer for ransac_n > 512): the
 * index build, each batch's passing count and end state, and the result. */
typedef struct {
    int use_edge_length, use_distance, use_normal;
    double edge_length_similarity;
    double distance_threshold;
    double cos_normal_angle_threshold;
} o3db_ransac_checkers;

typedef struct {
    int64_t drawn;        /* hypotheses drawn: stop */
    int64_t validated;    /* hypotheses that passed the checkers before stop */
    int64_t best_index;   /* draw index of the best hypothesis, -1 for none */
    double fitness;
    double inlier_rmse;
} o3db_ransac_stats;

int o3db_registration_ransac(const float* source_dev /* [n,3] */, const float* source_normals_dev /* or NULL */,
                             int64_t n, const float* target_dev /* [m,3] */,
                             const float* target_normals_dev /* or NULL */, int64_t m,
                             const int64_t* correspondences_dev /* [K,2] */, int64_t K,
                             double max_correspondence_distance, int ransac_n, int max_iteration, double confidence,
                             const o3db_ransac_checkers* checkers /* or NULL */, double* transformation_host /* [16] */,
                             int64_t* correspondence_set_dev /* [n] */, o3db_ransac_stats* stats, void* stream);

/* ------------------------------------------------------------------------
 * Fast Global Registration — pipelines::registration::FastGlobalRegistrationBasedOnCorrespondence and
 * FastGlobalRegistrationBasedOnFeatureMatching (pipelines/registration/FastGlobalRegistration.cpp:285-395, with
 * NormalizePointCloud :143-195, AdvancedMatching :83-141, OptimizePairwiseRegistration :197-264,
 * GetTransformationOriginalScale :268-282 and EvaluateRegistration, Registration.cpp:127-141), on Float32 clouds.
 * The result is that of upstream's function run on one thread, in f64 with every op rounded and the Eigen orders of
 * DESIGN.md §4.26:
 *   pairs       correspondences_dev [K,2] (source row, target row); or, when it is NULL, the mutual nearest rows of
 *               the [n,dim] and [m,dim] feature matrices (f32 squared distance, ties to the lowest row) in ascending
 *               query row, the source's rows being the queries unless the tuple test runs and n < m;
 *   normalise   each cloud's mean (the serial sum in point order / n), scale = the largest centred norm over both
 *               clouds, scale_global = scale, or 1 with use_absolute_scale; "Invalid scale_global" when it is <= 0;
 *   tuples      with tuple_test: nothing when there are at most 2 pairs (upstream's warning on stderr), else up to
 *               100 x pairs trials of three std::uniform_int_distribution<int>(0, pairs-1) draws from the library's
 *               engine, a trial passing when each of its three edges has li*tuple_scale < lj < li/tuple_scale, and the
 *               loop stopping after the trial at which maximum_tuple_count tuples have passed; afterwards the engine
 *               has advanced by exactly 3 x trials draws;
 *   optimise    the identity for fewer than 10 pairs, else iteration_number Geman-McClure steps from par =
 *               scale_global, with par /= division_factor every 4th step while decrease_mu and par >
 *               maximum_correspondence_distance;
 *   result      the inverse of the de-normalised transformation, evaluated on the original clouds: the nearest target
 *               point of each transformed source point with d^2 < maximum_correspondence_distance^2, ties to the
 *               lowest index; fitness = matches / n, rmse = sqrt(sum d^2 / matches), the sum over tiles of 128
 *               points in index order, then over the tiles.
 * transformation_host [16] receives the transformation, row-major; correspondence_set_dev [n] each source point's
 * match, -1 for none.  Errors: a non-finite distance, non-finite positions, a pair outside [0, n) x [0, m), more than
 * (2^31 - 1) / 100 pairs for the tuple test, counts of 2^31 - 1 or more, null pointers.  The call synchronises the
 * stream 3 times, plus once per batch of 16384 tuple trials, plus twice in the feature matching. */
typedef struct {
    double division_factor;
    int use_absolute_scale;
    int decrease_mu;
    double maximum_correspondence_distance;
    int iteration_number;
    double tuple_scale;
    int maximum_tuple_count;
    int tuple_test;
} o3db_fgr_option;

typedef struct {
    int64_t cross;        /* the initial pairs: K, or the mutual feature matches */
    int64_t tuples;       /* tuples that passed the tuple test */
    int64_t trials;       /* tuple trials drawn: the engine advanced by 3 x trials */
    int64_t pairs;        /* the pairs the optimisation ran on */
    double fitness;
    double inlier_rmse;
} o3db_fgr_stats;

int o3db_registration_fgr(const float* source_dev /* [n,3] */, int64_t n, const float* target_dev /* [m,3] */,
                          int64_t m, const int64_t* correspondences_dev /* [K,2] or NULL */, int64_t K,
                          const float* source_feature_dev /* [n,dim] */, const float* target_feature_dev /* [m,dim] */,
                          int dim, const o3db_fgr_option* option, double* transformation_host /* [16] */,
                          int64_t* correspondence_set_dev /* [n] */, o3db_fgr_stats* stats, void* stream);

/* ------------------------------------------------------------------------
 * RANSAC plane segmentation — geometry::PointCloud::SegmentPlane (geometry/PointCloudSegmentation.cpp:157-279), which
 * t::geometry::PointCloud::SegmentPlane (t/geometry/PointCloud.cpp:1646-1666) runs on the host; Float32 positions.
 * The result is that of upstream's function run on one thread (DESIGN.md §4.21):
 *   samples     num_iterations rows drawn up front as o3db_random_sample_indices does, all of them however early the
 *               loop stops;
 *   hypotheses  in f64 from the f32 positions: ComputeTrianglePlane (geometry/TriangleMesh.cpp:1248-1262) for
 *               ransac_n == 3, else GetPlaneFromPoints over the sample in sample order; (0,0,0,0) is skipped;
 *   scoring     a point is an inlier when |(a*x + c*z) + (b*y + d)| < distance_threshold, f64, each op rounded, no FMA
 *               (Eigen's packet order for Vector4d::dot); fitness = inliers / n; rmse = sqrt(error / inliers), error
 *               the sum of the squared distances sequential over each tile of 1024 points in index order, then over
 *               the tiles in order (upstream sums all points in one sequence; DESIGN.md §7);
 *   selection   hypotheses in index order, skipped once evaluated > break; a better one has the higher fitness, or
 *               the same and a lower rmse; each improvement sets break = size_t(min(log(1-p)/log(1-fitness^ransac_n),
 *               num_iterations)), or 0 at fitness 1; evaluated counts the non-degenerate hypotheses not skipped;
 *   result      inliers_dev [n] receives the K points within the threshold of the best hypothesis in ascending
 *               order, *num_inliers = K; plane_dev [4] receives GetPlaneFromPoints over them, with the sums in the
 *               tile order above.  With no valid hypothesis (num_iterations <= 0, every sample collinear, a threshold
 *               <= 0) the plane is (0,0,0,0) and K = 0.
 * stats (optional, host): the best hypothesis's index (-1 for none), the evaluated count, its fitness and rmse.
 * Errors, before any CUDA call, with upstream's messages: probability outside (0, 1], ransac_n < 3, n < ransac_n;
 * also null pointers, n >= INT_MAX, num_iterations * ransac_n >= 2^31.  The call synchronises the stream once. */
typedef struct {
    int64_t best_index;
    int64_t evaluated;
    double fitness;
    double inlier_rmse;
} o3db_segment_stats;

int o3db_segment_plane(const float* positions_dev /* [n,3] */, int64_t n, double distance_threshold, int ransac_n,
                       int num_iterations, double probability, double* plane_dev /* [4] */,
                       int64_t* inliers_dev /* [n] */, int64_t* num_inliers, o3db_segment_stats* stats, void* stream);

/* Reference-layout CSR spatial hash (parity / interop only): exactly the tables
 * BuildSpatialHashTableCUDA produces — cell = floor(p/(2r)), bucket =
 * SpatialHash(cell) % hash_table_size (core/nns/NeighborSearchCommon.h:31-52),
 * cell_splits = exclusive prefix sums (hash_table_size+1 entries), index table
 * = point ids grouped by bucket (order inside a bucket undefined, as upstream). */
int o3db_build_spatial_hash_table(const float* points_dev, int64_t num_points, double radius,
                                  uint32_t hash_table_size, uint32_t* hash_table_index_dev /* [M] */,
                                  uint32_t* hash_table_cell_splits_dev /* [size+1] */, void* stream);

/* ------------------------------------------------------------------------
 * Pose estimation from given correspondences — replaces
 * t::pipelines::kernel::ComputePosePointToPlaneCUDA (kernel/RegistrationImpl.h:93-102,
 * RegistrationCUDA.cu:29-117) including DecodeAndSolve6x6
 * (kernel/TransformationConverter.cpp:189-226).
 *   sums29_dev (optional, device, 29 doubles): the reduction vector
 *     [0..20] lower-tri JtWJ, [21..26] JtWr, [27] sum r, [28] inlier count.
 *   pose_dev (optional, device, 6 doubles): solution of AtA x = -Atb.
 *   residual_host / inlier_count_host (optional): as the reference's by-ref outputs
 *     (forces a stream synchronise).
 * Returns O3DB_ERR_SINGULAR if the system is singular (only detectable when a
 * host output is requested; otherwise pose is zero-filled, as upstream's catch). */
int o3db_compute_pose_point_to_plane(const float* source_dev, const float* target_dev,
                                     const float* target_normals_dev,
                                     const int64_t* correspondences_dev, int64_t n,
                                     const o3db_robust_kernel* kernel, double* sums29_dev,
                                     double* pose_dev, float* residual_host, int* inlier_count_host,
                                     void* stream);

/* ComputePoseColoredICPCUDA (kernel/RegistrationImpl.h:118-131, RegistrationCUDA.cu:119-230). */
int o3db_compute_pose_colored_icp(const float* source_dev, const float* source_colors_dev,
                                  const float* target_dev, const float* target_normals_dev,
                                  const float* target_colors_dev, const float* target_color_gradients_dev,
                                  const int64_t* correspondences_dev, int64_t n,
                                  const o3db_robust_kernel* kernel, double lambda_geometric,
                                  double* sums29_dev, double* pose_dev, float* residual_host,
                                  int* inlier_count_host, void* stream);

/* kernel::ComputeRtPointToPoint (kernel/Registration.cpp:365-404; RegistrationCPU.cpp:497-653: Get3x3SxyLinearSystem,
 * SVD, reflection fix, t = mean(t) - R mean(s)) for a given Int64 correspondence set (-1 = none, n entries, one per
 * source point).  R_host: row-major 3x3 Float64 rotation, t_host: Float64 translation, inlier_count_host (optional): the
 * number of valid correspondences.  The sums and the SVD are f64 on the device.  Returns O3DB_ERR_INVALID with upstream's
 * "No valid correspondence present." when every entry is -1.  When all matches are collinear the rotation is not
 * unique (upstream's neither): a proper rotation is returned. */
int o3db_compute_rt_point_to_point(const float* source_dev, const float* target_dev, const int64_t* correspondences_dev,
                                   int64_t n, double R_host[9], double t_host[3], int* inlier_count_host, void* stream);

/* TransformationEstimationSymmetric, for a given Int64 correspondence set (-1 = none, n entries, one per source point;
 * m target points).  Both clouds need normals ([.,3] f32).  An entry outside [-1, m) returns O3DB_ERR_INVALID with
 * upstream's "SymmetricICP correspondences must be -1 or a target point index ..." (TransformationEstimation.cpp:85-99).
 *   o3db_compute_pose_symmetric: kernel::ComputePoseSymmetric (RegistrationCPU.cpp:124-218, RegistrationImpl.h:324-387)
 *     about the given means (host, the cloud's dtype): the 29 sums of the centred Jacobian [ (s - ms + t - mt) x n ; n ]
 *     with n = n_t + sign(n_s . n_t) n_s, weights of the objective residual (s - t) . n, [27] its sum of squares, and
 *     DecodeAndSolve6x6.  Outputs as o3db_compute_pose_point_to_plane's; pose_dev is required.
 *   o3db_compute_transformation_symmetric: kernel::ComputeTransformationSymmetric (kernel/Registration.cpp:80-135):
 *     the means of the matched pairs, the pose above and PoseToSymmetricTransformation -> row-major 4x4 Float64 on the
 *     host; the identity when no entry is valid.  Synchronises the stream.
 *   o3db_pose_to_symmetric_transformation: PoseToSymmetricTransformation (SymmetricICPImpl.h:19-43), host f64. */
int o3db_compute_pose_symmetric(const float* source_dev, const float* target_dev, const float* source_normals_dev,
                                const float* target_normals_dev, const int64_t* correspondences_dev, int64_t n, int64_t m,
                                const float source_mean_host[3], const float target_mean_host[3],
                                const o3db_robust_kernel* kernel, double* sums29_dev, double* pose_dev,
                                float* residual_host, int* inlier_count_host, void* stream);
int o3db_compute_transformation_symmetric(const float* source_dev, const float* target_dev, const float* source_normals_dev,
                                          const float* target_normals_dev, const int64_t* correspondences_dev, int64_t n,
                                          int64_t m, const o3db_robust_kernel* kernel, double transformation_host[16],
                                          int* inlier_count_host, void* stream);
void o3db_pose_to_symmetric_transformation(const double pose_host[6], const double source_mean_host[3],
                                           const double target_mean_host[3], double transformation_host[16]);

/* TransformationEstimationForDopplerICP (TransformationEstimation.h:356-425): the fields of the C++ constructor.  The
 * C ABI applies its rules: |period| < 1e-3 returns O3DB_ERR_INVALID with "Time period too small.", and a
 * lambda_doppler outside [0, 1] becomes 0.01.  Each kernel is L2 or Tukey (DISPATCH_DUAL_ROBUST_KERNEL_FUNCTION); another
 * kernel returns "Unsupported method." once an iteration would use it.  transform_vehicle_to_sensor: row-major 4x4. */
typedef struct {
    double period;                          /* 0.1 */
    double lambda_doppler;                  /* 0.01 */
    int reject_dynamic_outliers;            /* 0 */
    double doppler_outlier_threshold;       /* 2.0 */
    int64_t outlier_rejection_min_iteration;       /* 2 */
    int64_t geometric_robust_loss_min_iteration;   /* 0 */
    int64_t doppler_robust_loss_min_iteration;     /* 2 */
    o3db_robust_kernel geometric_kernel;    /* L2 */
    o3db_robust_kernel doppler_kernel;      /* L2 */
    double transform_vehicle_to_sensor[16]; /* identity */
} o3db_doppler_params;

/* kernel::ComputePoseDopplerICP (kernel/Registration.cpp:193-312, RegistrationCPU.cpp:336-493,
 * RegistrationImpl.h:525-643) for a given Int64 correspondence set (-1 = none, n entries): source points, dopplers [n]
 * and directions [n,3] (never transformed), target points and normals, all f32.  current_transform_host is the
 * accumulated row-major 4x4 Float64 transformation (initial guess included) and `iteration` the index within the scale:
 * they give the velocity v_s_in_S and the three switches.  Outputs as o3db_compute_pose_point_to_plane's
 * (DecodeAndSolve6x6: O3DB_ERR_SINGULAR with upstream's message); [28] counts rejected dynamic points too. */
int o3db_compute_pose_doppler_icp(const float* source_dev, const float* source_dopplers_dev,
                                  const float* source_directions_dev, const float* target_dev,
                                  const float* target_normals_dev, const int64_t* correspondences_dev, int64_t n,
                                  const double current_transform_host[16], int64_t iteration,
                                  const o3db_doppler_params* params, double* sums29_dev, double* pose_dev,
                                  float* residual_host, int* inlier_count_host, void* stream);

/* registration::GetInformationMatrix (registration/Registration.cpp:446-485, pybind get_information_matrix): the 6x6
 * Float64 information matrix GTG of a registration — a clone of the source is transformed, matched to the target by the
 * hybrid search (k = 1), and the Jacobians of the matched TARGET points are reduced
 * (kernel::ComputeInformationMatrix[CUDA], RegistrationCUDA.cu:492-573, RegistrationImpl.h:686-715).  Raises (returns
 * O3DB_ERR_INVALID with upstream's message) when there is no correspondence.  information_host: row-major 6x6.
 * o3db_compute_information_matrix is the kernel-level twin for a given Int64 correspondence set (-1 = none). */
int o3db_get_information_matrix(const float* source_dev, int64_t n, const float* target_dev, int64_t m,
                                double max_correspondence_distance, const double transformation_host[16],
                                double information_host[36], void* stream);
int o3db_compute_information_matrix(const float* target_dev, const int64_t* correspondences_dev, int64_t n,
                                    double information_host[36], int64_t* num_correspondences_host, void* stream);

/* kernel::PoseToTransformation (kernel/TransformationConverter.cpp:81-104,
 * TransformationConverterImpl.h:22-42); host math, f64. */
void o3db_pose_to_transformation(const double pose_host[6], double transformation_host[16]);

/* t::geometry::kernel::transform::TransformPointsCUDA / TransformNormalsCUDA
 * (t/geometry/kernel/Transform.h:42-47, TransformImpl.h:20-62): in place,
 * T (row-major 4x4, host f64) is cast to f32 first as upstream does. */
int o3db_transform_points(const double transformation_host[16], float* points_dev, int64_t n, void* stream);
int o3db_transform_normals(const double transformation_host[16], float* normals_dev, int64_t n, void* stream);

/* ------------------------------------------------------------------------
 * t::geometry::PointCloud::VoxelDownSample(voxel_size, "mean") (t/geometry/PointCloud.cpp:496-560),
 * the pyramid build in front of the ICP loop (registration/Registration.cpp:237-240, 266-269).
 * One output point per occupied voxel floor(p / voxel_size): the mean of the positions and of
 * the optional normals / colors (not re-normalised, as upstream).  Output buffers need room for
 * n points; *num_out_host receives the voxel count (stream synchronise).  Output order is
 * undefined (upstream: hash-map slot order).
 * ---------------------------------------------------------------------- */
int o3db_voxel_down_sample(const float* positions_dev, const float* normals_dev /* may be NULL */,
                           const float* colors_dev /* may be NULL */, int64_t n, double voxel_size,
                           float* positions_out_dev, float* normals_out_dev, float* colors_out_dev,
                           int64_t* num_out_host, void* stream);

/* Same with up to 4 arbitrary [n,3] f32 point attributes (upstream averages every attribute of the
 * cloud, PointCloud.cpp:536-552 — e.g. "color_gradients" through the ColoredICP pyramid).
 * attrs_dev / attrs_out_dev are HOST arrays of num_attrs device pointers. */
int o3db_voxel_down_sample_attrs(const float* positions_dev, const float* const* attrs_dev, int num_attrs,
                                 int64_t n, double voxel_size, float* positions_out_dev,
                                 float* const* attrs_out_dev, int64_t* num_out_host, void* stream);

/* t::geometry::PointCloud::EstimateColorGradients with the hybrid search (t/geometry/PointCloud.cpp:
 * 723-767, kernel/PointCloudImpl.h:1066-1165 EstimateColorGradientsUsingHybridSearchCUDA): the
 * "color_gradients" attribute ColoredICP reads on the target.  Normal equations accumulated in f32 in
 * the reference's order, then the 3x3 solve:
 *   O3DB_GRADIENT_SOLVER_REFERENCE (what o3db_estimate_color_gradients uses): the reference's own
 *     solve_svd3x3<float> (core/linalg/kernel/SVD3x3.h:1131-2215, 4-sweep fast SVD, singular values
 *     < 1e-10 dropped) — bit-identical to the reference's CPU kernel on identical inputs;
 *   O3DB_GRADIENT_SOLVER_EXACT: exact pseudo-inverse of the same f32 system (f64 Jacobi), for callers
 *     who want the mathematically exact least-squares gradient (the fast SVD is off by a median 12 %
 *     on these condition-1e5 systems, DESIGN.md).
 * max_nn in 1..32 (reference default 30).  Points with < 4 neighbours get a zero gradient. */
#define O3DB_GRADIENT_SOLVER_REFERENCE 0
#define O3DB_GRADIENT_SOLVER_EXACT 1
int o3db_estimate_color_gradients(const float* positions_dev, const float* normals_dev, const float* colors_dev,
                                  int64_t n, double radius, int max_nn, float* color_gradients_dev /* [n,3] */,
                                  void* stream);
int o3db_estimate_color_gradients_solver(const float* positions_dev, const float* normals_dev,
                                         const float* colors_dev, int64_t n, double radius, int max_nn,
                                         int solver, float* color_gradients_dev /* [n,3] */, void* stream);

/* t::geometry::PointCloud::EstimateNormals(max_nn, radius) with the hybrid search (t/geometry/PointCloud.cpp:856-984,
 * kernel/PointCloudImpl.h:512-638 and 746-1065): the hybrid search of the cloud on itself, then per point the
 * covariance of its neighbours (f64 sums, Bessel's correction, stored f32; identity below 3 neighbours) and the
 * normal of the reference's fast 3x3 eigen solve, oriented as upstream:
 *   has_normals == 0: normals_dev is output only; a zero normal becomes (0,0,1);
 *   has_normals != 0: normals_dev holds the prior normals on entry; the new normal is flipped where its dot with
 *     the prior is negative, and a zero normal stays zero.
 * covariances_dev ([n,9] row-major, may be NULL) receives upstream's transient "covariances" attribute.  The
 * covariances are bit-identical to the reference's CPU kernel on identical neighbour lists; the normals differ only
 * where libm's acosf / cosf are not correctly rounded (DESIGN.md).  max_nn in 1..32 (reference default 30); n == 0 is
 * a no-op.  Synchronises the stream. */
int o3db_estimate_normals(const float* positions_dev, int64_t n, double radius, int max_nn, int has_normals,
                          float* normals_dev /* [n,3] */, float* covariances_dev /* [n,9] or NULL */, void* stream);

/* PointCloud::OrientNormalsToAlignWithDirection (PointCloudImpl.h:261-294): in place, a normal whose dot with
 * direction is negative is flipped and a zero normal becomes direction. */
int o3db_orient_normals_to_align_with_direction(float* normals_dev, int64_t n, const float direction_host[3],
                                                void* stream);

/* PointCloud::OrientNormalsTowardsCameraLocation (PointCloudImpl.h:296-351): in place, a normal that points away from
 * camera - p is flipped; a zero normal becomes (camera - p) / |camera - p|, or (0,0,1) where that is zero. */
int o3db_orient_normals_towards_camera_location(const float* positions_dev, float* normals_dev, int64_t n,
                                                const float camera_host[3], void* stream);

/* t::geometry::PointCloud::ComputeBoundaryPoints (t/geometry/PointCloud.cpp:803-853, kernel/PointCloudImpl.h:354-506):
 * the hybrid search of the cloud on itself (radius > 0 and finite, max_nn in 1..32; upstream's default is 30); the
 * first entry of each neighbour list is dropped as the point itself; the other m neighbours' angles in the plane of
 * the point's normal are sorted, and mask_dev[i] = 1 where the largest gap between consecutive angles, the wrap-around
 * included, exceeds angle_threshold degrees.  The frame and the dot products are f32 in upstream's order with no FMA;
 * atan2 is evaluated in f64 and rounded to f32 (DESIGN.md §4.22).  m == 0 gives 0.  A normal whose frame is NaN
 * (exactly (0,0,±1), zero, or a NaN component) gives a largest gap of 0, as upstream.
 * max_gap_dev ([n] or NULL) receives each point's largest gap in radians (0 where m == 0).  Non-finite positions and
 * infinite normal components return O3DB_ERR_INVALID.  n == 0 is a no-op.  Synchronises the stream. */
int o3db_compute_boundary_points(const float* positions_dev, const float* normals_dev /* [n,3] */, int64_t n,
                                 double radius, int max_nn, double angle_threshold, uint8_t* mask_dev /* [n] */,
                                 float* max_gap_dev /* [n] or NULL */, void* stream);

/* t::pipelines::registration::ComputeFPFHFeature (t/pipelines/registration/Feature.cpp:23-277,
 * kernel/FeatureImpl.h:23-293): the 33-bin FPFH feature of each point over its neighbour list, the min(max_nn, n)
 * nearest points (max_nn in 4..128) capped at dist^2 <= (float)radius^2 when radius > 0 (the hybrid search), uncapped
 * when radius == 0 (KNN only).  The first entry of each list is dropped as the point itself.  indices_dev ([num_indices]
 * Int64, any order, repeats allowed) selects rows: fpfh_dev receives one row per distinct index in ascending point
 * order, each equal to that point's row of the call without indices; num_indices == -1 selects every point.
 * fpfh_dev holds [rows, 33]; *num_rows receives the row count.  Pair features are f32 in upstream's order with no FMA,
 * acos / atan2 evaluated in f64 and rounded to f32 (DESIGN.md §4.24).  Non-finite positions or normal components and
 * indices outside [0, n) return O3DB_ERR_INVALID.  n == 0 or num_indices == 0 gives no rows.  Synchronises the
 * stream. */
int o3db_compute_fpfh_feature(const float* positions_dev, const float* normals_dev /* [n,3] */, int64_t n, int max_nn,
                              double radius, const int64_t* indices_dev, int64_t num_indices,
                              float* fpfh_dev /* [rows,33] */, int64_t* num_rows, void* stream);

/* t::pipelines::registration::CorrespondencesFromFeatures (t/pipelines/registration/Feature.cpp:279-333): for each
 * source row i of [n, dim] the nearest target row of [m, dim] by the f32 sum over d of fmaf(s - t, s - t, acc), ties
 * to the lowest index.  corres_dev ([n, 2] Int64) receives (i, nearest) rows; with mutual_filter only the rows whose
 * target's nearest source is i, in source order, when there are more than mutual_consistent_ratio * n of them (f32, as
 * upstream), else every row.  *num_corres receives the row count, *num_mutual (or NULL) the mutual count.  n == 0
 * gives no rows; m == 0 with n > 0 returns O3DB_ERR_INVALID.  Synchronises the stream. */
int o3db_correspondences_from_features(const float* source_dev /* [n,dim] */, int64_t n,
                                       const float* target_dev /* [m,dim] */, int64_t m, int dim, int mutual_filter,
                                       float mutual_consistent_ratio, int64_t* corres_dev /* [n,2] */,
                                       int64_t* num_corres, int64_t* num_mutual, void* stream);

/* t::geometry::PointCloud::RemoveRadiusOutliers (t/geometry/PointCloud.cpp:650-676): mask_dev[i] = 1 when at least
 * nb_points points, point i included, lie within search_radius of it, with the predicate of upstream's CUDA radius
 * search: d = p - q in f32, dist = fma(d2, d2, fma(d1, d1, fma(d0, d0, 0))), a neighbour iff dist <= r * r, r the
 * radius rounded to f32 (DESIGN.md §4.23).  nb_points < 1 or search_radius <= 0 give upstream's error; a NaN or
 * infinite radius and non-finite positions return O3DB_ERR_INVALID.  nb_points > n keeps nothing.  n == 0 is a
 * no-op.  Synchronises the stream once, for the index's bounding box. */
int o3db_remove_radius_outliers(const float* positions_dev /* [n,3] */, int64_t n, int64_t nb_points,
                                double search_radius, uint8_t* mask_dev /* [n] */, void* stream);

/* t::geometry::PointCloud::RemoveDuplicatedPoints (t/geometry/PointCloud.cpp:740-760): two points are duplicates when
 * their coordinates are equal bit for bit (so -0.0 != 0.0, and NaNs with equal bits are duplicates); mask_dev[i] = 1
 * for the lowest index of each group.  Any bit pattern is accepted.  n == 0 is a no-op.  Does not synchronise. */
int o3db_remove_duplicated_points(const float* positions_dev /* [n,3] */, int64_t n, uint8_t* mask_dev /* [n] */,
                                  void* stream);

/* t::geometry::PointCloud::RemoveNonFinitePoints (t/geometry/PointCloud.cpp:716-738): mask_dev[i] = 0 when remove_nan
 * and a coordinate is NaN, or remove_inf and a coordinate is infinite; 1 otherwise.  n == 0 is a no-op.  Does not
 * synchronise. */
int o3db_remove_non_finite_points(const float* positions_dev /* [n,3] */, int64_t n, int remove_nan, int remove_inf,
                                  uint8_t* mask_dev /* [n] */, void* stream);

/* ------------------------------------------------------------------------
 * Fused, device-resident ICP loop — replaces
 * t::pipelines::registration::ICP / MultiScaleICP / DoSingleScaleICPIterations /
 * ComputeRegistrationResult (registration/Registration.cpp:24-62, 93-106, 275-444)
 * for TransformationEstimationPointToPlane (TransformationEstimation.cpp:196-227)
 * on one scale without down-sampling.
 * ---------------------------------------------------------------------- */
typedef struct {
    double max_correspondence_distance;
    int max_iteration;          /* ICPConvergenceCriteria::max_iteration_ (Registration.h:43-48) */
    double relative_fitness;    /* ICPConvergenceCriteria::relative_fitness_ */
    double relative_rmse;       /* ICPConvergenceCriteria::relative_rmse_ */
    o3db_robust_kernel kernel;  /* TransformationEstimationPointToPlane::kernel_ */
    double cell_scale;          /* search-grid cell = cell_scale * radius (0 => default) */
} o3db_icp_options;

typedef struct {
    double transformation[16];  /* RegistrationResult::transformation_ (row-major 4x4 f64) */
    double fitness;             /* RegistrationResult::fitness_ */
    double inlier_rmse;         /* RegistrationResult::inlier_rmse_ */
    int converged;              /* RegistrationResult::converged_ */
    int num_iterations;         /* RegistrationResult::num_iterations_ */
    int status;                 /* O3DB_OK or O3DB_ERR_SINGULAR */
    int64_t num_correspondences;
} o3db_icp_result;

typedef struct o3db_icp o3db_icp;
typedef struct o3db_comm o3db_comm;

/* Builds the target index, clones + cell-sorts the source (the caller's arrays
 * are never modified, as Registration.cpp:398-404 clones) and applies
 * init_source_to_target.  `comm` may be NULL (single GPU); with a communicator
 * the source arrays are this rank's shard, the target is replicated, and every
 * iteration all-reduces the 30-double system (SURVEY.md §8e). */
int o3db_icp_create(const float* source_dev, int64_t n, const float* target_dev,
                    const float* target_normals_dev, int64_t m,
                    const double init_source_to_target_host[16], const o3db_icp_options* options,
                    o3db_comm* comm, void* stream, o3db_icp** out);
/* Same loop for TransformationEstimationForColoredICP (TransformationEstimation.cpp:229-296,
 * kernel/RegistrationImpl.h:337-425): colours are [.,3] f32 in the reference's value range, the
 * target's color_gradients come from o3db_estimate_color_gradients (or upstream's
 * EstimateColorGradients); lambda_geometric as upstream (default 0.968).  Everything else
 * (search, convergence rule, result) is identical to the point-to-plane handle and the same
 * iterate / finish / reset / destroy calls apply. */
int o3db_icp_create_colored(const float* source_dev, const float* source_colors_dev, int64_t n,
                            const float* target_dev, const float* target_normals_dev,
                            const float* target_colors_dev, const float* target_color_gradients_dev, int64_t m,
                            const double init_source_to_target_host[16], const o3db_icp_options* options,
                            double lambda_geometric, o3db_comm* comm, void* stream, o3db_icp** out);
/* Same loop for TransformationEstimationPointToPoint (TransformationEstimation.cpp:101-159,
 * kernel/Registration.cpp:365-404), the estimator registration::ICP uses by default: positions only
 * (AssertInputMultiScaleICP, Registration.cpp:119-219, asks this estimator for nothing else), no robust kernel
 * (options->kernel is ignored, the class has none) and no singular-system status.  Search, convergence rule, result
 * and the iterate / finish / state / reset / destroy calls are those of the point-to-plane handle. */
int o3db_icp_create_point_to_point(const float* source_dev, int64_t n, const float* target_dev, int64_t m,
                                   const double init_source_to_target_host[16], const o3db_icp_options* options,
                                   o3db_comm* comm, void* stream, o3db_icp** out);
/* Same loop for TransformationEstimationSymmetric (TransformationEstimation.cpp:229-292, kernel/Registration.cpp:80-135):
 * both clouds need normals; the working source's normals are rotated with its points every iteration, as
 * PointCloud::Transform does upstream.  options->kernel is the estimator's robust kernel.  Single GPU only: a
 * communicator is rejected (O3DB_ERR_INVALID).  Iterate / finish / state / reset / destroy as for the other handles. */
int o3db_icp_create_symmetric(const float* source_dev, const float* source_normals_dev, int64_t n, const float* target_dev,
                              const float* target_normals_dev, int64_t m, const double init_source_to_target_host[16],
                              const o3db_icp_options* options, o3db_comm* comm, void* stream, o3db_icp** out);
/* Same loop for TransformationEstimationForDopplerICP: the source needs Doppler values ([n] f32) and directions
 * ([n,3] f32, in the sensor's vehicle frame, never transformed), the target normals.  Every iteration derives the
 * velocity from the accumulated transformation and applies the switches of `params` on the device.  options->kernel is
 * ignored (the params carry both kernels).  Single GPU only: a communicator is rejected (O3DB_ERR_INVALID). */
int o3db_icp_create_doppler(const float* source_dev, const float* source_dopplers_dev, const float* source_directions_dev,
                            int64_t n, const float* target_dev, const float* target_normals_dev, int64_t m,
                            const double init_source_to_target_host[16], const o3db_icp_options* options,
                            const o3db_doppler_params* params, o3db_comm* comm, void* stream, o3db_icp** out);
/* Restore the state right after o3db_icp_create (source re-gathered, T = init). */
int o3db_icp_reset(o3db_icp* icp, void* stream);
/* Enqueue up to `iterations` ICP iterations (asynchronous, no host sync). */
int o3db_icp_iterate(o3db_icp* icp, int iterations, void* stream);
/* Final ComputeRegistrationResult (Registration.cpp:424-431) + read-back.
 * correspondences_dev (optional, [N] int64, -1 = none) in the caller's source order;
 * per_iteration_host (optional): 2 doubles (fitness, inlier_rmse) per executed iteration. */
int o3db_icp_finish(o3db_icp* icp, o3db_icp_result* result_host, int64_t* correspondences_dev,
                    double* per_iteration_host, void* stream);
/* The loop's state after the last executed iteration WITHOUT the final evaluation pass: transformation, and the
 * fitness / inlier_rmse that iteration's own search measured.  What MultiScaleICP keeps between scales
 * (Registration.cpp:406-431 re-runs ComputeRegistrationResult only after the last scale). */
int o3db_icp_state(o3db_icp* icp, o3db_icp_result* result_host, double* per_iteration_host, void* stream);
void o3db_icp_destroy(o3db_icp* icp);

/* One-shot convenience: create + iterate(max_iteration) + finish + destroy. */
int o3db_icp_point_to_plane(const float* source_dev, int64_t n, const float* target_dev,
                            const float* target_normals_dev, int64_t m,
                            const double init_source_to_target_host[16],
                            const o3db_icp_options* options, o3db_icp_result* result_host,
                            int64_t* correspondences_dev, double* per_iteration_host, void* stream);
int o3db_icp_point_to_point(const float* source_dev, int64_t n, const float* target_dev, int64_t m,
                            const double init_source_to_target_host[16], const o3db_icp_options* options,
                            o3db_icp_result* result_host, int64_t* correspondences_dev, double* per_iteration_host,
                            void* stream);
int o3db_icp_symmetric(const float* source_dev, const float* source_normals_dev, int64_t n, const float* target_dev,
                       const float* target_normals_dev, int64_t m, const double init_source_to_target_host[16],
                       const o3db_icp_options* options, o3db_icp_result* result_host, int64_t* correspondences_dev,
                       double* per_iteration_host, void* stream);
int o3db_icp_doppler(const float* source_dev, const float* source_dopplers_dev, const float* source_directions_dev, int64_t n,
                     const float* target_dev, const float* target_normals_dev, int64_t m,
                     const double init_source_to_target_host[16], const o3db_icp_options* options,
                     const o3db_doppler_params* params, o3db_icp_result* result_host, int64_t* correspondences_dev,
                     double* per_iteration_host, void* stream);
int o3db_icp_colored(const float* source_dev, const float* source_colors_dev, int64_t n, const float* target_dev,
                     const float* target_normals_dev, const float* target_colors_dev,
                     const float* target_color_gradients_dev, int64_t m,
                     const double init_source_to_target_host[16], const o3db_icp_options* options,
                     double lambda_geometric, o3db_icp_result* result_host, int64_t* correspondences_dev,
                     double* per_iteration_host, void* stream);
/* Same through HOST buffers (pageable or pinned): copies inputs host->device,
 * runs, copies the result (and optional correspondences) back. */
int o3db_icp_point_to_plane_host(const float* source_host, int64_t n, const float* target_host,
                                 const float* target_normals_host, int64_t m,
                                 const double init_source_to_target_host[16],
                                 const o3db_icp_options* options, o3db_icp_result* result_host,
                                 int64_t* correspondences_host, double* per_iteration_host);

/* ------------------------------------------------------------------------
 * Multi-GPU: one process per GPU; NCCL is dlopen()ed at run time
 * (libnccl.so.2 — torch's bundled copy if torch is loaded, else the system one).
 * The reference has no collective layer (SURVEY.md fact 3).
 * o3db_comm_create is collective (every rank must call it): besides ncclCommInitRank it allocates a 1 KB-per-rank
 * mailbox on every GPU, exchanges CUDA IPC handles (one ncclAllGather) and maps every peer's mailbox, so that the
 * sharded ICP loop can exchange its 30-double system inside the iteration kernel over NVLink (DESIGN.md 5);
 * if any rank cannot map any peer, all ranks agree to use ncclAllReduce instead.
 * ---------------------------------------------------------------------- */
#define O3DB_UNIQUE_ID_BYTES 128
int o3db_comm_get_unique_id(uint8_t id_out[O3DB_UNIQUE_ID_BYTES]);
int o3db_comm_create(const uint8_t id[O3DB_UNIQUE_ID_BYTES], int rank, int world_size, o3db_comm** out);
int o3db_comm_allreduce_f64(o3db_comm* comm, double* buf_dev, int count, void* stream);
/* 1 when the ranks exchange the per-iteration system INSIDE the iteration kernel over NVLink / NVSwitch peer memory
 * (every rank could map every other rank's mailbox through CUDA IPC at o3db_comm_create), 0 when each iteration is
 * kernel + ncclAllReduce + finalize kernel.  Identical on all ranks.  (Set O3DB_COMM_NO_PEER to force NCCL.) */
int o3db_comm_uses_peer_memory(const o3db_comm* comm);
void o3db_comm_destroy(o3db_comm* comm);

/* ------------------------------------------------------------------------
 * TSDF voxel block grid — replaces, for the slam::Model layout
 * (t/pipelines/slam/Model.cpp:23-36: tsdf f32[1], weight u16[1], color u16[3],
 * keys int32x3), core::HashMap (core/hashmap/HashMap.cpp:117-216) with the CUDA
 * backend (core/hashmap/CUDA/StdGPUHashBackend.h), DepthTouchCUDA
 * (t/geometry/kernel/VoxelBlockGrid.h:345-356, VoxelBlockGridCUDA.cu:106-227)
 * and IntegrateCUDA<u16,u8,f32,u16,u16> / <f32,f32,f32,u16,u16>
 * (VoxelBlockGrid.h:369-381, VoxelBlockGridImpl.h:151-308).
 * ---------------------------------------------------------------------- */
typedef struct o3db_vbg o3db_vbg;

typedef enum { O3DB_DEPTH_U16 = 0, O3DB_DEPTH_F32 = 1 } o3db_depth_dtype;
typedef enum { O3DB_COLOR_NONE = 0, O3DB_COLOR_U8 = 1, O3DB_COLOR_F32 = 2 } o3db_color_dtype;

/* VoxelBlockGrid ctor (t/geometry/VoxelBlockGrid.cpp:34-92): block_count is the
 * initial capacity (slam::Model est_block_count); with_color allocates u16x3. */
int o3db_vbg_create(float voxel_size, int block_resolution, int64_t block_count, int with_color,
                    void* stream, o3db_vbg** out);
void o3db_vbg_destroy(o3db_vbg* vbg);

/* HashMap::Size / GetCapacity / Reserve (HashMap.cpp:47-77, 210-216). */
int64_t o3db_vbg_size(o3db_vbg* vbg, void* stream);
int64_t o3db_vbg_capacity(const o3db_vbg* vbg);
int o3db_vbg_reserve(o3db_vbg* vbg, int64_t capacity, void* stream);

/* HashMap::Activate (HashMap.cpp:166-181) / Find (:183-197) on int32x3 keys.
 * buf_indices_dev [n] int32 (slot in the key/value buffers; -1 for Find misses),
 * masks_dev [n] u8 (Activate: 1 for exactly one inserter of each NEW key;
 * Find: 1 if present).  Activate grows (rehash) like upstream when
 * size + n > capacity. */
int o3db_vbg_activate(o3db_vbg* vbg, const int32_t* keys_dev, int64_t n, int32_t* buf_indices_dev,
                      uint8_t* masks_dev, void* stream);
int o3db_vbg_find(o3db_vbg* vbg, const int32_t* keys_dev, int64_t n, int32_t* buf_indices_dev,
                  uint8_t* masks_dev, void* stream);
/* HashMap::GetActiveIndices (:199-203): writes Size() buf indices, returns the count. */
int64_t o3db_vbg_active_indices(o3db_vbg* vbg, int32_t* buf_indices_dev, int64_t max_count, void* stream);

/* Raw buffers (HashMap::GetKeyTensor / GetValueTensor): keys [capacity,3] int32,
 * tsdf [capacity,res^3] f32, weight [capacity,res^3] u16, color [capacity,res^3,3] u16.
 * Pointers are invalidated by a growth (Reserve). */
int32_t* o3db_vbg_key_buffer(o3db_vbg* vbg);
float* o3db_vbg_tsdf_buffer(o3db_vbg* vbg);
uint16_t* o3db_vbg_weight_buffer(o3db_vbg* vbg);
uint16_t* o3db_vbg_color_buffer(o3db_vbg* vbg);
/* The 64-bit key hash used by the table == utility::MiniVecHash<int,3>
 * (core/hashmap/Dispatch.h:67-81); exposed for bit-exact parity tests. */
int o3db_hash_keys(const int32_t* keys_dev, int64_t n, uint64_t* hashes_dev, void* stream);

/* VoxelBlockGrid::GetUniqueBlockCoordinates(depth, ...) (VoxelBlockGrid.cpp:212-245)
 * -> DepthTouchCUDA.  Writes the unique frustum block keys ([*,3] int32, order
 * undefined as upstream) to block_coords_dev (capacity max_blocks; upstream's
 * frustum map capacity is (W/4)(H/4)*4) and their number to *num_blocks_host
 * (stream synchronise).  intrinsic: 3x3, extrinsic: 4x4 world->camera, host f64. */
int o3db_vbg_unique_block_coordinates(o3db_vbg* vbg, const void* depth_dev, int depth_dtype,
                                      int rows, int cols, const double intrinsic_host[9],
                                      const double extrinsic_host[16], float depth_scale,
                                      float depth_max, float trunc_voxel_multiplier,
                                      int32_t* block_coords_dev, int64_t max_blocks,
                                      int64_t* num_blocks_host, void* stream);

/* VoxelBlockGrid::Integrate(block_coords, depth, color, ...) (VoxelBlockGrid.cpp:292-326):
 * Activate + Find + IntegrateCUDA.  color_dev may be NULL (depth-only overload). */
int o3db_vbg_integrate(o3db_vbg* vbg, const int32_t* block_coords_dev, int64_t num_blocks,
                       const void* depth_dev, int depth_dtype, const void* color_dev, int color_dtype,
                       int rows, int cols, const double depth_intrinsic_host[9],
                       const double color_intrinsic_host[9], const double extrinsic_host[16],
                       float depth_scale, float depth_max, float trunc_voxel_multiplier, void* stream);

/* slam::Model::Integrate (t/pipelines/slam/Model.cpp:91-106) as ONE fused,
 * host-sync-free pipeline: frustum touch + global activate + integrate (two launches per frame).
 *
 * Capacity: the reference grows the map inside HashMap::Activate (HashMap.cpp:166-181).  Here the FIRST frame of a
 * handle (and the first one after o3db_vbg_reserve) sizes the map synchronously from the touch kernel's own count;
 * later frames run asynchronously and the map is grown ahead of need from what earlier frames added (3 frames x
 * twice the largest per-frame increase seen, at least 3 x 2048 blocks).  A frame that still does not fit (a camera
 * jump adding more blocks than that) is DROPPED AS A WHOLE on the device, together with every later frame: nothing
 * is integrated, the table is restored, the volume is exactly the state before that frame.  The next call that can
 * see it (at most two calls later; o3db_vbg_size / _last_frustum_blocks see it immediately) returns
 * O3DB_ERR_CAPACITY with "fused frame #K needed N blocks" in o3db_last_error(); call o3db_vbg_reserve(>= N) — which
 * also re-arms the handle — and resubmit frames K, K+1, ... (K counts fused frames of this handle from 0). */
int o3db_vbg_integrate_frame(o3db_vbg* vbg, const void* depth_dev, int depth_dtype,
                             const void* color_dev, int color_dtype, int rows, int cols,
                             const double intrinsic_host[9], const double extrinsic_host[16],
                             float depth_scale, float depth_max, float trunc_voxel_multiplier,
                             void* stream);
/* Stateless twins of the reference's DepthTouchCUDA / IntegrateCUDA<...> (t/geometry/kernel/VoxelBlockGrid.h:345-381,
 * VoxelBlockGridCUDA.cu:106-244) for an integration that keeps the reference's own core::HashMap: nothing but the
 * arguments of those functions is needed — block indices / keys / value buffers are the reference hash map's tensors.
 *   o3db_depth_touch: unique block coordinates of a depth frame (stride must be 4, VoxelBlockGrid.cpp:221); sdf_trunc
 *     is passed as the reference passes it.  Synchronises the stream (the count sizes the output, as upstream).
 *   o3db_integrate_blocks: per-voxel fusion of the listed blocks.  value_layout selects the reference's two value
 *     layouts: O3DB_VALUES_U16 (weight UInt16, colour UInt16 — the slam::Model layout, fast path) or O3DB_VALUES_F32
 *     (weight Float32, colour Float32); tsdf is Float32 in both.  All four IntegrateCUDA instantiations are covered
 *     by {u16 depth + u8 colour, f32 depth + f32 colour} x {U16, F32}. */
#define O3DB_VALUES_U16 0
#define O3DB_VALUES_F32 1
int o3db_depth_touch(const void* depth_dev, int depth_dtype, int rows, int cols, const double intrinsic_host[9],
                     const double extrinsic_host[16], int block_resolution, float voxel_size, float sdf_trunc,
                     float depth_scale, float depth_max, int stride, int32_t* block_coords_dev, int64_t max_blocks,
                     int64_t* num_blocks_host, void* stream);
int o3db_integrate_blocks(const void* depth_dev, int depth_dtype, const void* color_dev, int color_dtype, int rows,
                          int cols, const int32_t* block_indices_dev, int64_t num_blocks,
                          const int32_t* block_keys_dev, float* tsdf_dev, void* weight_dev, void* color_buf_dev,
                          int value_layout, const double depth_intrinsic_host[9], const double color_intrinsic_host[9],
                          const double extrinsic_host[16], int block_resolution, float voxel_size, float sdf_trunc,
                          float depth_scale, float depth_max, void* stream);

/* Same through HOST images (pinned recommended): H2D copies included. */
int o3db_vbg_integrate_frame_host(o3db_vbg* vbg, const void* depth_host, int depth_dtype,
                                  const void* color_host, int color_dtype, int rows, int cols,
                                  const double intrinsic_host[9], const double extrinsic_host[16],
                                  float depth_scale, float depth_max, float trunc_voxel_multiplier,
                                  void* stream);
/* Throughput form of the same call for a pre-recorded sequence: n_frames images of
 * identical size/dtype, frame f at depth_ptrs[f] / color_ptrs[f] (device pointers if
 * `host_images` is 0, host pointers — pinned recommended — otherwise), extrinsics_host is
 * n_frames x 16 doubles.  Semantically identical to calling o3db_vbg_integrate_frame[_host]
 * n_frames times in order (same kernels, same order, bit-identical volume); it only removes
 * the per-call host overhead of the caller's language binding. */
int o3db_vbg_integrate_sequence(o3db_vbg* vbg, int64_t n_frames, const void* const* depth_ptrs,
                                int depth_dtype, const void* const* color_ptrs, int color_dtype,
                                int rows, int cols, const double intrinsic_host[9],
                                const double* extrinsics_host, float depth_scale, float depth_max,
                                float trunc_voxel_multiplier, int host_images, void* stream);

/* Device-side execution time of the fused integrate launches since the last reset: per launch, %globaltimer of the last
 * CTA's end minus the earliest CTA's start (after its griddepcontrol.wait), summed.  Unlike CUDA events between the two
 * frame kernels this does not disable their programmatic overlap, so it is the kernel's duration inside an undisturbed
 * frame stream.  Synchronises the stream. */
int o3db_vbg_exec_stats(o3db_vbg* vbg, double* integrate_exec_ms, int64_t* launches, int reset, void* stream);

/* Block keys of the last integrated frame (Model::frustum_block_coords_): copies
 * up to max_blocks keys, returns the count (stream synchronise). */
int64_t o3db_vbg_last_frustum_blocks(o3db_vbg* vbg, int32_t* block_coords_dev, int64_t max_blocks,
                                     void* stream);

/* ------------------------------------------------------------------------
 * VoxelBlockGrid::RayCast (t/geometry/VoxelBlockGrid.cpp:328-402) = kernel::voxel_grid::EstimateRange
 * (kernel/VoxelBlockGridImpl.h:310-555) + RayCast (:578-1120), the step after Integrate in
 * slam::Model::SynthesizeModelFrame (slam/Model.cpp:38-66).
 *
 * block_coords_dev: [num_blocks,3] int32 keys that bound the rays (upstream: frustum_block_coords_),
 *   or NULL = the blocks touched by the last o3db_vbg_integrate_frame (no host round trip).
 * K: 3x3, E: 4x4 world->camera, both host f64 row-major.
 * range_dev (optional for ray_cast): [height/down][width/down][2] f32 (min, max) — upstream's "range"
 *   rendering.  Unlike upstream there is no fragment buffer and hence no overflow mode.
 * Outputs are row-major [height][width][C]; every pointer may be NULL (attribute not requested).
 * Rendering "color" from a grid created without colour yields zeros.
 * ---------------------------------------------------------------------- */
typedef struct {
    float* depth;            /* C=1: t_intersect * depth_scale, 0 = no surface */
    float* vertex;           /* C=3: camera-frame point */
    float* color;            /* C=3: trilinear colour / 255 */
    float* normal;           /* C=3: camera-frame, MINUS the normalised TSDF gradient (as upstream) */
    int64_t* index;          /* C=8: linear voxel ids of the 8 interpolation corners */
    uint8_t* mask;           /* C=8: corner valid (bool) */
    float* interp_ratio;     /* C=8 */
    float* interp_ratio_dx;  /* C=8 */
    float* interp_ratio_dy;  /* C=8 */
    float* interp_ratio_dz;  /* C=8 */
} o3db_raycast_outputs;

int o3db_vbg_estimate_range(o3db_vbg* vbg, const int32_t* block_coords_dev, int64_t num_blocks,
                            const double intrinsic_host[9], const double extrinsic_host[16], int height,
                            int width, int down_factor, float depth_min, float depth_max,
                            float* range_dev, void* stream);
int o3db_vbg_ray_cast(o3db_vbg* vbg, const int32_t* block_coords_dev, int64_t num_blocks,
                      const double intrinsic_host[9], const double extrinsic_host[16], int width, int height,
                      const o3db_raycast_outputs* outputs_host, float depth_scale, float depth_min,
                      float depth_max, float weight_threshold, float trunc_voxel_multiplier,
                      int range_map_down_factor, float* range_dev, void* stream);

/* ------------------------------------------------------------------------
 * VoxelBlockGrid::ExtractPointCloud (t/geometry/VoxelBlockGrid.cpp:404-434; slam::Model::ExtractPointCloud,
 * slam/Model.cpp:108-111, forwards to it) = BufferRadiusNeighbors (VoxelBlockGrid.cpp:22-51) + kernel::voxel_grid::
 * ExtractPointCloud (kernel/VoxelBlockGridImpl.h:1122-1381): one point per voxel o and axis i where o and o + e_i both
 * have weight > weight_threshold and tsdf_i * tsdf_o < 0, at the linear zero crossing, with the interpolated TSDF
 * gradient as normal and the interpolated colour / 255 (grids with colour only).
 *
 * Rows come in a deterministic order (upstream's is an atomic counter's): ascending block slot (the order of
 * o3db_vbg_active_indices), then the linear voxel index (z*R + y)*R + x, then axis 0, 1, 2; two calls on an unchanged
 * volume give identical bits.  max_points < 0: every point (upstream's estimated_point_number = -1); max_points >= 0:
 * the first min(max_points, total) rows of that order.  The surface may hold at most INT32_MAX points.
 *
 * Outputs: *num_points and [*num_points, 3] f32 device buffers owned by the handle, valid until the next extract on
 * it or o3db_vbg_destroy; *colors is NULL for a grid without colour, all three are NULL when there are no points.
 * Synchronises the stream once (the point count); reports a frame dropped for capacity like o3db_vbg_size.
 * ---------------------------------------------------------------------- */
int o3db_vbg_extract_point_cloud(o3db_vbg* vbg, float weight_threshold, int64_t max_points, int64_t* num_points,
                                 float** points, float** normals, float** colors, void* stream);

/* ------------------------------------------------------------------------
 * VoxelBlockGrid::ExtractTriangleMesh (t/geometry/VoxelBlockGrid.cpp:436-472; slam::Model::ExtractTriangleMesh
 * forwards to it) = BufferRadiusNeighbors + kernel::voxel_grid::ExtractTriangleMesh (kernel/VoxelBlockGridImpl.h:
 * 1385-1780), marching cubes over the cubes of 8 voxels: a cube contributes when all 8 corners exist with weight >
 * weight_threshold; its case is the 8-bit tsdf < 0 pattern (-0.0 is not negative).  The edge (o, o + e_i) gets a
 * vertex when its corners differ in that bit and one of the up to four cubes sharing it contributes; the vertex has
 * the point cloud's position, normal and colour expressions (a corner at exactly 0 gives a vertex at ratio 0).
 *
 * Vertices come in o3db_vbg_extract_point_cloud's order (block slot, voxel, axis); triangles by block slot, voxel and
 * the case table's order, as Int32 vertex indices wound as upstream winds them.  Each case's polygons are upstream's;
 * they may be split along other diagonals (DESIGN.md §4.27).  Two calls on an unchanged volume give identical bits.
 * estimated_vertex_number > 0 only sizes the buffers ahead of the count: the mesh is always complete.  The surface may
 * hold at most INT32_MAX vertices and INT32_MAX triangles.
 *
 * Outputs: *num_vertices, *num_triangles, [*num_vertices, 3] f32 and [*num_triangles, 3] i32 device buffers owned by
 * the handle, valid until the next o3db_vbg_extract_triangle_mesh on it or o3db_vbg_destroy (an extract_point_cloud
 * call does not touch them); *colors is NULL for a grid without colour, all four are NULL for an empty surface.
 * Synchronises the stream once (the two counts); reports a frame dropped for capacity like o3db_vbg_size.
 * ---------------------------------------------------------------------- */
int o3db_vbg_extract_triangle_mesh(o3db_vbg* vbg, float weight_threshold, int64_t estimated_vertex_number,
                                   int64_t* num_vertices, int64_t* num_triangles, float** vertices, float** normals,
                                   float** colors, int32_t** triangles, void* stream);

/* ------------------------------------------------------------------------
 * Point clouds from depth / RGB-D images and back (t/geometry/kernel/ paths).
 *
 * o3db_unproject: PointCloud::CreateFromDepthImage / CreateFromRGBDImage without normals (t/geometry/PointCloud.cpp:
 * 1414-1469) -> kernel::pointcloud::Unproject (kernel/PointCloud.cpp:21-65, kernel/PointCloudImpl.h:43-144).  The
 * strided grid is (rows / stride) x (cols / stride); strided pixel (i, j) is image pixel (x, y) = (j*stride, i*stride)
 * with d = depth / depth_scale; it gives a point when 0 < d < depth_max, at RigidTransform(InverseTransformation(
 * extrinsic), Unproject(x, y, d)) in f32, and, with a colour image, the colour pixel at (x, y) as f32 without scaling
 * (a u8 image gives 0..255, as upstream's rgbd.color_.To(Float32)).  Rows come row-major over the strided grid
 * (upstream's order is an atomic counter's); two calls give identical bits.  points_dev / colors_dev need room for
 * the whole strided grid; *num_points receives the count (one stream synchronise).
 *
 * o3db_project: PointCloud::ProjectToDepthImage / ProjectToRGBDImage (PointCloud.cpp:1471-1530) ->
 * kernel::pointcloud::Project (kernel/PointCloudCUDA.cu:26-162).  A point is moved by extrinsic, projected, and
 * u, v rounded half away from zero; it is rejected when !InBoundary(u, v) || zc <= 0 || zc > depth_max.  Each pixel
 * takes the point with the least (float bits of d = zc * depth_scale, point index), the reference CUDA kernel's
 * packed atomicMin, for depth-only images too; every pixel of depth_dev ([rows][cols] f32) and color_dev
 * ([rows][cols][3] f32, with colors_dev) is written, 0 where no point lands.  The reference CPU kernel
 * (PointCloudCPU.cpp:21-90) differs at an exact depth tie, where it keeps the colour of the last writer.
 * Asynchronous.
 *
 * Unlike upstream, both reject (O3DB_ERR_INVALID) null pointers, stride < 1, a depth_scale that is not finite and
 * positive, negative image sizes, a strided grid or point count of 2^31 or more, and colour dtypes other than
 * O3DB_COLOR_U8 / O3DB_COLOR_F32.  Each call runs a fixed number of kernels, whatever its sizes.
 * ---------------------------------------------------------------------- */
int o3db_unproject(const void* depth_dev, int depth_dtype, int rows, int cols,
                   const void* color_dev /* NULL or [rows][cols][3] */, int color_dtype,
                   const double intrinsic_host[9], const double extrinsic_host[16],
                   float depth_scale, float depth_max, int stride,
                   float* points_dev, float* colors_dev /* [(rows/stride)*(cols/stride)][3] */,
                   int64_t* num_points, void* stream);
int o3db_project(const float* points_dev, const float* colors_dev /* NULL: depth only */, int64_t n,
                 const double intrinsic_host[9], const double extrinsic_host[16],
                 float depth_scale, float depth_max, int rows, int cols,
                 float* depth_dev /* [rows][cols] */, float* color_dev /* [rows][cols][3] or NULL */, void* stream);

/* ------------------------------------------------------------------------
 * RGB-D odometry, PointToPlane method — slam::Model::TrackFrameToModel (slam/Model.cpp:68-89) ->
 * odometry::RGBDOdometryMultiScale (odometry/RGBDOdometry.cpp:56-206).
 *
 * Image members used by the pyramid (t/geometry/Image.cpp:409-520 over t/geometry/kernel/ImageImpl.h:86-315),
 * device buffers, row-major [rows][cols](x3), Float32 unless noted:
 * ---------------------------------------------------------------------- */
int o3db_image_clip_transform(const void* src_dev, int depth_dtype /* O3DB_DEPTH_U16 | _F32 */, int rows, int cols,
                              float scale, float min_value, float max_value, float clip_fill, float* dst_dev,
                              void* stream);
int o3db_image_pyr_down_depth(const float* src_dev, int rows, int cols, float diff_threshold, float invalid_fill,
                              float* dst_dev /* [rows/2][cols/2] */, void* stream);
int o3db_image_create_vertex_map(const float* depth_dev, int rows, int cols, const double intrinsic_host[9],
                                 float invalid_fill, float* vertex_dev /* [rows][cols][3] */, void* stream);
int o3db_image_create_normal_map(const float* vertex_dev, int rows, int cols, float invalid_fill,
                                 float* normal_dev /* [rows][cols][3] */, void* stream);
/* Image::FilterBilateral (Image.cpp:248-285).  Upstream forwards to NPP's nppiFilterBilateralGaussBorder
 * (kernel/NPPImage.cpp:319-376: radius kernel_size/2, nValSquareSigma = value_sigma^2, nPosSquareSigma =
 * dist_sigma^2, replicated border), a closed-source library; this evaluates NPP's documented definition
 *   out = sum(w v) / sum(w),  w = exp(-(dx^2+dy^2)/(2 dist_sigma^2)) * exp(-(v - v_center)^2/(2 value_sigma^2))
 * in f32.  PARITY UNPINNED against NPP (DESIGN.md). */
int o3db_image_filter_bilateral(const float* src_dev, int rows, int cols, int kernel_size, float value_sigma,
                                float dist_sigma, float* dst_dev, void* stream);

/* odometry::ComputeOdometryResultPointToPlane (RGBDOdometry.cpp:432-459) = kernel
 * ComputeOdometryResultPointToPlaneCUDA (kernel/RGBDOdometryCUDA.cu:37-125) + DecodeAndSolve6x6 +
 * PoseToTransformation: one Gauss-Newton step.  delta_transformation_host: 4x4 f64 row-major;
 * inlier_rmse = sum(HuberLoss) / inlier_count, fitness = inlier_count / (rows*cols) (as upstream);
 * sums29_host (optional): the 29 reduced scalars.  Errors: O3DB_ERR_SINGULAR, O3DB_ERR_NO_INLIERS. */
int o3db_compute_odometry_result_point_to_plane(const float* source_vertex_map_dev,
                                                const float* target_vertex_map_dev,
                                                const float* target_normal_map_dev, int rows, int cols,
                                                const double intrinsic_host[9],
                                                const double init_source_to_target_host[16],
                                                float depth_outlier_trunc, float depth_huber_delta,
                                                double delta_transformation_host[16], double* inlier_rmse_host,
                                                double* fitness_host, double* sums29_host, void* stream);

typedef struct {
    int max_iteration;        /* OdometryConvergenceCriteria (RGBDOdometry.h:33-52) */
    double relative_rmse;
    double relative_fitness;
} o3db_odometry_criteria;

typedef struct {
    double transformation[16]; /* OdometryResult::transformation_ (source -> target, 4x4 f64) */
    double inlier_rmse;        /* OdometryResult::inlier_rmse_ */
    double fitness;            /* OdometryResult::fitness_ */
    int status;                /* O3DB_OK, O3DB_ERR_SINGULAR or O3DB_ERR_NO_INLIERS */
    int iterations;            /* Gauss-Newton steps executed over all levels */
} o3db_odometry_result;

/* RGBDOdometryMultiScale(..., Method::PointToPlane) with the whole coarse-to-fine loop on the device.
 * criteria[0] applies to the coarsest level (upstream's criteria_list order); num_levels <= 8.
 * Depth images may be UInt16 or Float32 independently (input frame vs. ray-cast model frame).
 * per_iteration_host (optional): (inlier_rmse, fitness) of every executed step. */
int o3db_rgbd_odometry_multi_scale_point_to_plane(const void* source_depth_dev, int source_dtype,
                                                  const void* target_depth_dev, int target_dtype, int rows,
                                                  int cols, const double intrinsic_host[9],
                                                  const double init_source_to_target_host[16], float depth_scale,
                                                  float depth_max, const o3db_odometry_criteria* criteria,
                                                  int num_levels, float depth_outlier_trunc,
                                                  float depth_huber_delta, o3db_odometry_result* result_host,
                                                  double* per_iteration_host, void* stream);

/* Measurement aid (bench.py): when enabled, CUDA events bracket the touch and the
 * integrate kernel of every o3db_vbg_integrate_frame call (up to 4096 frames per
 * read); o3db_vbg_profile_read synchronises and returns the summed device times. */
int o3db_vbg_profile(o3db_vbg* vbg, int enable);
int o3db_vbg_profile_read(o3db_vbg* vbg, double* touch_ms, double* integrate_ms, int64_t* frames);

#ifdef __cplusplus
}
#endif
#endif /* OPEN3D_B200_H_ */

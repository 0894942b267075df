/*
 * b200match — C ABI of the H100 (sm_90a) descriptor-matching engine.
 *
 * Drop-in boundary for the one hot path of AliceVision's featureMatching step.  Every entry point below is what
 * a reference-side adaptor binds (see INTEGRATION.md and alicevision_b200/adaptor/):
 *
 *   Surface 1  matching::ArrayMatcher<Scalar,Metric>         src/aliceVision/matching/ArrayMatcher.hpp:39,51,65
 *              (reference implementation replaced: ArrayMatcher_bruteForce.hpp:42-142)
 *   Surface 2  matchingImageCollection::IImageCollectionMatcher::Match
 *                                                            src/aliceVision/matchingImageCollection/IImageCollectionMatcher.hpp:36-41
 *              (reference implementation replaced: ImageCollectionMatcher_generic.cpp:30-123 with
 *               matching/RegionsMatcher.hpp:126-176 inside)
 *
 * Plain pointers and sizes only.  All functions return 0 on success, non-zero on failure (never throw, never
 * abort); b200m_last_error() returns a thread-local message.  There is NO CPU fallback inside the library: without
 * a CUDA device every compute entry point fails with B200M_ERR_CUDA.
 */
#ifndef B200MATCH_H_
#define B200MATCH_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200m_ctx b200m_ctx;       /* one engine instance bound to one GPU */
typedef struct b200m_db b200m_db;         /* a built ArrayMatcher database (Surface 1) */
typedef struct b200m_result b200m_result; /* output of b200m_match_pairs (Surface 2) */

/* descriptor element types: feature::Regions::Type_id() "f" / "h" and IsBinary() (feature/Regions.hpp:157-161) */
enum { B200M_F32 = 0, B200M_U8 = 1, B200M_BIN = 2 };
/* metrics: feature::L2_Simple (metric.hpp:27), feature::L2_Vectorized (metric.hpp:48,128), feature::Hamming (Hamming.hpp:76) */
enum { B200M_L2_SIMPLE = 0, B200M_L2_VECTORIZED = 1, B200M_HAMMING = 2 };
/* status codes */
enum { B200M_OK = 0, B200M_ERR_ARG = 1, B200M_ERR_CUDA = 2, B200M_ERR_EMPTY = 3, B200M_ERR_UNSUPPORTED = 4, B200M_ERR_INTERNAL = 5 };
/* how far b200m_match_pairs goes */
enum {
  B200M_STAGE_DEVICE = 0, /* kernels only: match records stay in HBM (kernel-boundary timing) */
  B200M_STAGE_RAW = 1,    /* + records copied to pinned host memory, grouped per pair, not de-duplicated */
  B200M_STAGE_FULL = 2    /* + host finishing == RegionsMatcher::Match output (RegionsMatcher.hpp:153-175) and cross check */
};

/* == matching::IndMatch (matching/IndMatch.hpp:25-65; _distance exists because ALICEVISION_DEBUG_MATCHING is defined, :18) */
typedef struct { uint32_t i, j; float distance_ratio, distance; } b200m_match;

const char* b200m_last_error(void);
int b200m_version(void);
/* number of CUDA devices visible (0 when none / no driver); never fails */
int b200m_device_count(void);

/* ---- context ------------------------------------------------------------------------------------------------ */
/* device: CUDA ordinal.  stream: a cudaStream_t to enqueue on (e.g. the caller's), or NULL for an internal stream. */
int b200m_ctx_create(int device, void* stream, b200m_ctx** out);
void b200m_ctx_destroy(b200m_ctx* ctx);
/* host threads used by the finishing stage (default: hardware concurrency, capped at 32) */
int b200m_ctx_set_host_threads(b200m_ctx* ctx, int n);
/* force every L2 pair through the exact CUDA-core kernels (testing / A-B comparison); default 0 */
int b200m_ctx_set_force_exact(b200m_ctx* ctx, int on);
/* tensor-core kernel variant (A-B comparison): 4 = half-norms folded into the GEMM, 256-query work items (default);
 * half-norms added in the epilogue: 2 = 256-query work items, 3 = 128-query work items, 1 = 128-query work items with the
 * exactness pass in a separate kernel */
int b200m_ctx_set_tc_variant(b200m_ctx* ctx, int variant);

/* debug / test hook, host only: the checked fp32 -> uchar conversion the upload staging applies to integer-valued fp32 descriptors
 * (which = 0: the dispatching implementation, AVX2 when available; 1: the scalar one).  1 = every value was an integer in 0..255 and dst
 * holds them; 0 = some value is not (dst unspecified); -1 = bad arguments. */
int b200m_debug_convert_f32_u8(const float* src, uint8_t* dst, size_t n, int which);

/* debug: per-tile SM-clock trace of CTA 0 of the tensor-core kernel (4 roles x 512 tiles x 4 stamps: TMA producer, the two
 * consumer warpgroups, unused; of the u8 kernel when the last batch had uchar-stored pairs, else of the fp16 kernel);
 * enable!=0 allocates,
 * out (may be NULL) receives up to n values after synchronising */
int b200m_debug_trace(b200m_ctx* ctx, int enable, long long* out, int n);

/* ---- Surface 1: ArrayMatcher ---------------------------------------------------------------------------------- */
/* Build (ArrayMatcher.hpp:39).  Copies `rows x dim` elements to the device (the reference borrows the pointer,
 * ArrayMatcher_bruteForce.hpp:49).  rows < 1 -> B200M_ERR_EMPTY, like Build returning false (:44-48). */
int b200m_db_create(b200m_ctx* ctx, const void* data, int rows, int dim, int dtype, int metric, b200m_db** out);
void b200m_db_destroy(b200m_db* db);
/* SearchNeighbours (ArrayMatcher.hpp:65).  idx[nq*nn] database indices, dist[nq*nn] float (L2, squared) or
 * uint32 (Hamming), ascending per query.  nn > rows or nq < 1 -> B200M_ERR_ARG (bruteForce.hpp:105-108). nn <= 16. */
int b200m_knn(b200m_ctx* ctx, const b200m_db* db, const void* query, int nq, int nn, int32_t* idx, void* dist);

/* ---- Surface 2: image-collection matching ---------------------------------------------------------------------- */
/* Register / replace one view's regions (feature::Regions of one descType: DescriptorRawData(), RegionCount(),
 * DescriptorLength(), GetRegionsPositions(); feature/Regions.hpp:57-62,158,187).  xy = n x 2 float positions
 * (needed by B200M_STAGE_FULL only; may be NULL otherwise).  n == 0 is allowed (view skipped when matched). */
int b200m_upload_view(b200m_ctx* ctx, uint32_t view_id, const void* desc, int n, int dim, int dtype, const float* xy);
/* The same for n views of one descriptor type in one call (the copies of consecutive views are pipelined). */
int b200m_upload_views(b200m_ctx* ctx, int n_views, const uint32_t* view_ids, const void* const* descs, const int* counts, int dim, int dtype,
                       const float* const* xys);
/* Asynchronous form: returns once the views are registered; the descriptor copies run on an upload thread and stream
 * behind the call.  `descs` must stay valid until the next b200m_match_pairs, b200m_wait_uploads, b200m_upload_view(s),
 * b200m_clear_views or b200m_remove_view on this context RETURNS (positions are copied before returning).
 * b200m_match_pairs waits only for the views of the batch it is about to enqueue and processes the pair list in the order
 * the views arrive, so searching overlaps the host->device copies. */
int b200m_upload_views_async(b200m_ctx* ctx, int n_views, const uint32_t* view_ids, const void* const* descs, const int* counts, int dim,
                             int dtype, const float* const* xys);
/* Block until no upload reads caller memory any more; returns the first error an asynchronous upload hit. */
int b200m_wait_uploads(b200m_ctx* ctx);
int b200m_clear_views(b200m_ctx* ctx);
/* Drop one view (device buffers are released in stream order); unknown id -> B200M_ERR_ARG.  Used by the IRegionsMatcher
 * adaptor (matching/RegionsMatcher.hpp:49-78), whose database and query regions live only as long as the matcher / the call. */
int b200m_remove_view(b200m_ctx* ctx, uint32_t view_id);

/* Match a list of (I, J) view-id pairs: I = database image, J = query image (RegionsMatcher.hpp:157-158).
 * Scalar descriptors of 128 components take the tensor-core kernel when their values allow it (integers, |v| <= 1024) and the
 * exact CUDA-core kernel otherwise; other scalar lengths (AKAZE float 64, LIOP uchar 144; regionsFactory.hpp:25-27) take a generic
 * exact kernel; binary descriptors must be 64 bytes (AKAZE_BinaryRegions).
 * dist_ratio as given on the CLI (main_featureMatching.cpp:102): squared internally for L2, used as is for Hamming.
 * cross != 0 reproduces --crossMatching (ImageCollectionMatcher_generic.cpp:83-111). Pairs are processed and
 * reported in PairSet (lexicographic) order; pairs whose result is empty are reported with zero matches (the adaptor
 * must not insert them, :116-119). */
int b200m_match_pairs(b200m_ctx* ctx, const uint32_t* pairs, int n_pairs, float dist_ratio, int cross, int stage, b200m_result** out);

int b200m_result_num_pairs(const b200m_result* r);
/* pair_ids: n_pairs x 2; offsets: n_pairs + 1 (into matches); all pointers owned by the result. */
int b200m_result_get(const b200m_result* r, const uint32_t** pair_ids, const int64_t** offsets, const b200m_match** matches);
void b200m_result_free(b200m_result* r);

/* ---- guided matching (the step after the path) ------------------------------------------------------------------------ */
/* matching::guidedMatching<Mat3Model, FundamentalEpipolarDistanceError>(model, camL, lRegions, camR, rRegions, errorTh,
 * distRatio, matches) for cameras without distortion (matching/guidedMatching.hpp:206-268; called with
 * errorTh = Square(precision), distRatio = Square(ratio) by GeometricFilterMatrix_F_AC.hpp:381-389): for every feature of the
 * LEFT view, among the features of the RIGHT view whose epipolar error (multiview/relativePose/FundamentalError.hpp:52-64,
 * F row-major, x_right^T F x_left = 0) is below errorTh, the two smallest squared descriptor distances
 * (Regions::SquaredDescriptorDistance: L2 for scalar, squared Hamming for binary); kept iff best < distRatio * second.
 * Both views must have been uploaded with positions.  The result holds one pair (view_left, view_right) whose matches are
 * IndMatch(i = left feature, j = right feature), sorted by (i, j), ratio and distance 0 as in the reference. */
int b200m_guided_match(b200m_ctx* ctx, uint32_t view_left, uint32_t view_right, const double* F, double errorTh, double distRatio, b200m_result** out);
/* The same with the model named: B200M_MODEL_FUNDAMENTAL (above) or B200M_MODEL_HOMOGRAPHY = HomographyAsymmetricError
 * (multiview/relativePose/HomographyError.hpp:23-31: |x_right - (H x_left).head<2>() / (H x_left)[2]|^2), what
 * GeometricFilterMatrix_H_AC.hpp:217-225 calls. */
enum { B200M_MODEL_FUNDAMENTAL = 0, B200M_MODEL_HOMOGRAPHY = 1 };
int b200m_guided_match_model(b200m_ctx* ctx, uint32_t view_left, uint32_t view_right, int model, const double* M, double errorTh, double distRatio,
                             b200m_result** out);
/* matching::guidedMatching<Mat3Model, FundamentalEpipolarDistanceError | HomographyAsymmetricError> + IndMatch::getDeduplicated
 * (guidedMatching.hpp:206-268) for every pair (L = pairs[2k], R = pairs[2k+1]) of resident views, one model per pair:
 *   M        n_pairs x 9 row-major (F: x_R^T F x_L = 0; H: x_R ~ H x_L), model = B200M_MODEL_FUNDAMENTAL | B200M_MODEL_HOMOGRAPHY
 *   errorTh  n_pairs values, already squared (Square(m_dPrecision_robust) differs per pair)
 *   distRatio already squared, one for the call
 * The result holds one pair per input pair, in input order (empty lists included); each list is what b200m_guided_match_model
 * returns for that pair: IndMatch(i = left, j = right) in ascending i, ratio and distance 0.  A pair whose views differ in
 * descriptor type, or with an empty view, gets an empty list.  Waits only for the views the list references; long lists run in
 * internal batches of at most 8192 pairs and a bounded left-feature total (B200M_GUIDED_LEFT_CAP overrides that bound).  b200m_guided_match and
 * b200m_guided_match_model are this call on a list of one pair. */
int b200m_guided_match_pairs(b200m_ctx* ctx, const uint32_t* pairs, int n_pairs, int model, const double* M, const double* errorTh, double distRatio,
                             b200m_result** out);
/* Position-only guided matching, what GeometricFilterMatrix_H_AC::Geometry_guided_matching runs with distanceRatio < 0 (featureMatching's
 * guided homography filter): matching::guidedMatching<Mat3Model, ErrorT>(model, xLeft, xRight, errorTh, matches) (guidedMatching.hpp:37-70)
 * for every pair of resident views.  For every left feature, the right feature of smallest error (HomographyAsymmetricError or
 * FundamentalEpipolarDistanceError) below errorTh, the first j on ties; no descriptor is read.  Then IndMatch::getDeduplicated.
 * Arguments as in b200m_guided_match_pairs, without distRatio.  The positions are the geometry positions when set
 * (b200m_set_view_geometry), else the upload positions.
 *   decorate = 0: that list, IndMatch(i = left, j = right) sorted by (i, j), ratio and distance 0.  As in the reference, with
 *                 errorTh = +inf a left feature without a finite error below DBL_MAX contributes IndMatch() = (0, 0).
 *   decorate = 1: then IndMatchDecorator<float>::getDeduplicated on the upload positions of both views (GeometricFilterMatrix_H_AC.hpp:197-199):
 *                 on the device for a left view in general position (all x distinct, all y distinct), else the reference's std::set.
 *                 Both views need upload positions (else B200M_ERR_ARG).
 * A pair with an empty view, or whose views differ in describer type, gets an empty list.  Batches as b200m_guided_match_pairs. */
int b200m_guided_match_positions_pairs(b200m_ctx* ctx, const uint32_t* pairs, int n_pairs, int model, const double* M, const double* errorTh,
                                       int decorate, b200m_result** out);

/* Positions guided matching uses for one uploaded view instead of its (float) upload positions: n x 2 doubles, typically
 * camera::IntrinsicBase::getUndistortedPixel of every feature (matching/guidedMatching.hpp:229-248, :395, :416): the reference
 * matches on undistorted positions whenever the intrinsic is valid.  b200m_guided_match, b200m_guided_match_model,
 * b200m_guided_match_pairs and b200m_guided_match_fast_pairs use them when they are set; a view with geometry positions needs no upload positions.
 * n must equal the view's feature count (else B200M_ERR_ARG); xy == NULL drops them; unknown view -> B200M_ERR_ARG.
 * Re-uploading or removing the view drops them.  The array is copied before the call returns. */
int b200m_set_view_geometry(b200m_ctx* ctx, uint32_t view_id, const double* xy, int n);

/* matching::guidedMatchingFundamentalFast<FundamentalEpipolarDistanceError> (matching/guidedMatching.hpp:353-460), what
 * StructureEstimationFromKnownPoses::match (sfm/pipeline/structureFromKnownPoses/StructureEstimationFromKnownPoses.cpp:72-163)
 * runs for every pair of its list, for every pair (L = pairs[2k], R = pairs[2k+1]) of resident views:
 *   F         n_pairs x 9 row-major (x_R^T F x_L = 0)
 *   epipole2  n_pairs x 3, NOT normalised (as epipole_from_P returns it)
 *   wh        n_pairs x 2 = (widthR, heightR), each >= 2 (else B200M_ERR_ARG)
 *   errorTh, distRatio already squared, as StructureEstimationFromKnownPoses.cpp:138-150 passes them.
 * Left features are bucketed by where their epipolar line meets the right image's border; each right feature compares against
 * every left feature of the bucket range its +-sqrt(errorTh) band reaches (no geometric-error test), keeping the left feature's
 * best right feature iff best < distRatio * second.  The result holds one pair per input pair, in input order (empty lists
 * included); matches = IndMatch(i = left feature, j = right feature) in ascending i, ratio and distance 0, NOT de-duplicated
 * (the reference does not).  Descriptors as for b200m_guided_match; a pair whose views differ in descriptor type, or with an
 * empty view, gets an empty list.  Waits only for the views the list references; long lists run in internal batches of
 * bounded size.  Instrumentation: b200m_last_records = candidate (left, right) distances evaluated.
 * Where the reference is undefined - an epipole at infinity (epipole2[2] == 0) or a right feature exactly at the epipole - it
 * indexes its buckets with NaN cast to int; here a line with a non-finite coefficient has no end points: the left feature
 * joins no bucket and the right feature has no candidates. */
int b200m_guided_match_fast_pairs(b200m_ctx* ctx, const uint32_t* pairs, int n_pairs, const double* F, const double* epipole2,
                                  const int32_t* wh, double errorTh, double distRatio, b200m_result** out);

/* ---- Surface 2 on several GPUs from one process --------------------------------------------------------------------- */
/* Which shard (0..n_shards-1) each pair goes to: database images (first id) in ascending order are dealt round-robin over
 * the shards, direction alternating every round; all pairs of one database image stay together (its descriptors are
 * reused out of L2, ImageCollectionMatcher_generic.cpp:45-50 groups the same way).  Host-only, no GPU needed. */
int b200m_shard_pairs(const uint32_t* pairs, int n_pairs, int n_shards, int32_t* shard_of);
/* The sharding b200m_multi_match and bench.py use: 2-D blocks of the (symmetric) pair matrix, so that a shard needs only part of the
 * views (8 shards: half of them, 4 shards: at most three quarters), which is what bounds the end-to-end rate once every shard has to
 * stage its views through the same host.  View ids are dealt cyclically into g classes, the folded blocks {class(I), class(J)} are
 * assigned heaviest-first to the least loaded shard; g is picked per call for balance (<= 3 %) then for the fewest views per shard.
 * Pairs of one shard keep PairSet order, so all pairs of one database image stay adjacent (L2 reuse;
 * ImageCollectionMatcher_generic.cpp:45-50 groups the same way).  Host-only. */
int b200m_shard_pairs_2d(const uint32_t* pairs, int n_pairs, int n_shards, int32_t* shard_of);

typedef struct b200m_multi b200m_multi;   /* one engine context per device + one host thread each */
int b200m_multi_create(const int* devices, int n_devices, b200m_multi** out);
void b200m_multi_destroy(b200m_multi* m);
int b200m_multi_num_devices(const b200m_multi* m);
b200m_ctx* b200m_multi_ctx(b200m_multi* m, int k);
/* One IImageCollectionMatcher::Match call on all devices: shards the pair list (b200m_shard_pairs), uploads to each GPU
 * only the views its shard references (asynchronously, overlapped with its first pairs), runs b200m_match_pairs
 * (B200M_STAGE_FULL) per device on its own host thread and merges the results in PairSet order.  No data-path
 * collective: pairs are independent.  Views are given as in b200m_upload_views; previous views of the contexts are dropped. */
int b200m_multi_match(b200m_multi* m, int n_views, const uint32_t* view_ids, const void* const* descs, const int* counts, int dim, int dtype,
                      const float* const* xys, const uint32_t* pairs, int n_pairs, float dist_ratio, int cross, b200m_result** out);
/* max over devices of the GPU time of the last b200m_multi_match, ms */
double b200m_multi_last_gpu_ms(const b200m_multi* m);

/* ---- geometric filtering: a-contrario RANSAC fundamental matrix (K10) -------------------------------------------- */
/* GeometricFilterMatrix_F_AC::geometricEstimation_Mat_ACRANSAC<Fundamental7PSolver, Mat3Model> for every pair of a list, results
 * in input order.  Every pair starts from the same generator state, as the reference passes the std::mt19937 by value.
 *   offsets    n_pairs + 1 ascending correspondence offsets
 *   corr       offsets[n_pairs] x 4 doubles (xI, yI, xJ, yJ): the pair's xI / xJ matrices (fillMatricesWithUndistortFeaturesMatches)
 *   wh         n_pairs x 4 = (widthI, heightI, widthJ, heightJ), each >= 1
 *   mt_state   625 words: the caller's std::mt19937 as its operator<< writes it (624 words, then the position)
 *   max_iteration  ACRANSAC's nIter; precision: its upper bound (+inf = pure a-contrario mode)
 * Out: valid[n_pairs] (minNFA < 0), n_inliers[n_pairs], inliers (at offsets, the reference's order), F[9 * n_pairs] (row-major,
 * x_J^T F x_I = 0; unnormalised when valid), error_max[n_pairs] (ACRANSAC's first result), min_nfa[n_pairs],
 * iterations[n_pairs] (loop iterations executed).  A pair with at most 7 correspondences returns (0, 0) and no iteration. */
int b200m_acransac_fundamental_pairs(b200m_ctx* ctx, int n_pairs, const int64_t* offsets, const double* corr, const int32_t* wh,
                                     const uint32_t* mt_state, int64_t max_iteration, double precision, uint8_t* valid,
                                     int32_t* n_inliers, uint32_t* inliers, double* F, double* error_max, double* min_nfa,
                                     int32_t* iterations);
/* ---- geometric filtering: a-contrario RANSAC homography (K10, homography_matrix filter) ---------------------------- */
/* GeometricFilterMatrix_H_AC::geometricEstimation (ACRANSAC over RelativePoseKernel<Homography4PSolver, HomographyAsymmetricError,
 * UnnormalizerI>, point-to-point error) for every pair of a list, results in input order.  Arguments and outputs as in
 * b200m_acransac_fundamental_pairs, with H[9 * n_pairs] (row-major, x_J ~ H x_I; unnormalised when valid) in place of F.  A pair
 * with at most 4 correspondences returns (0, 0) and no iteration.
 * Generator: the reference passes its std::mt19937 by reference, so a single-threaded filter starts pair k where pair k - 1 left
 * off.  A batch cannot reproduce that chain (each pair's draw count depends on its data), so:
 *   mt_state_per_pair  0: mt_state is 625 words, the start state of every pair; 1: n_pairs x 625 words, one per pair
 *   mt_state_out       NULL, or n_pairs x 625 words: each pair's generator state after its estimation (its input state when the
 *                      pair is too small to draw).  A caller that needs the sequential chain runs the pairs one call each and
 *                      passes the previous pair's output state on. */
int b200m_acransac_homography_pairs(b200m_ctx* ctx, int n_pairs, const int64_t* offsets, const double* corr, const int32_t* wh,
                                    const uint32_t* mt_state, int mt_state_per_pair, int64_t max_iteration, double precision, uint8_t* valid,
                                    int32_t* n_inliers, uint32_t* inliers, double* H, double* error_max, double* min_nfa, int32_t* iterations,
                                    uint32_t* mt_state_out);
/* ---- geometric filtering: a-contrario RANSAC fundamental matrix of two equidistant cameras (K10, spherical) ------------- */
/* GeometricFilterMatrix_F_AC::geometricEstimation_Spherical_Mat (ACRANSAC over RelativePoseSphericalKernel<Fundamental7PSphericalSolver,
 * EpipolarSphericalDistanceError>), the branch the fundamental_matrix filter takes when both cameras of a pair are
 * camera::Equidistant, for every pair of a list, results in input order.  No image size: the kernel works on unit vectors without
 * normalisation, logalpha0 = pi, errorVectorDimension = 2, thresholdNormalizer = 1.
 *   bearings   offsets[n_pairs] x 6 doubles (xI, yI, zI, xJ, yJ, zJ): the caller's lift of each correspondence,
 *              toUnitSphere(removeDistortion(ima2cam(x))) of the xI / xJ columns the planar call would take
 * Other arguments and outputs as in b200m_acransac_homography_pairs (the reference passes this generator by reference too), with
 * F[9 * n_pairs] (row-major, x_J^T F x_I = 0 on the bearings; no unnormalisation) and error_max = sqrt of the largest inlier's
 * squared residual when valid.  A pair with at most 7 correspondences returns (0, 0) and no iteration. */
int b200m_acransac_fundamental_spherical_pairs(b200m_ctx* ctx, int n_pairs, const int64_t* offsets, const double* bearings,
                                               const uint32_t* mt_state, int mt_state_per_pair, int64_t max_iteration, double precision,
                                               uint8_t* valid, int32_t* n_inliers, uint32_t* inliers, double* F, double* error_max,
                                               double* min_nfa, int32_t* iterations, uint32_t* mt_state_out);
/* ---- geometric filtering: a-contrario RANSAC essential matrix of two pinhole cameras (K10, essential_matrix filter) ------ */
/* GeometricFilterMatrix_E_AC::geometricEstimation (ACRANSAC over RelativePoseKernel_K<Essential5PSolver,
 * FundamentalEpipolarDistanceError, Mat3Model>) for every pair of a list, results in input order.  The 5-point solver runs on
 * K^-1 x; the residual is the point-to-line error of F = K_J^-T E K_I^-1 on the pixels; no normalisation, errorVectorDimension = 0.5,
 * logalpha0 = log10(2 D / A * .5) of (widthJ, heightJ), maxThreshold = precision^2.
 *   corr       offsets[n_pairs] x 4 doubles (xI, yI, xJ, yJ), as for b200m_acransac_fundamental_pairs
 *   wh         n_pairs x 4 = (widthI, heightI, widthJ, heightJ), each >= 1
 *   K          n_pairs x 18 doubles: K_I then K_J, row-major (camera::Pinhole::K()); finite and invertible
 * Other arguments and outputs as in b200m_acransac_homography_pairs (the reference passes this generator by reference too), with
 * E[9 * n_pairs] (row-major, x_J^T F x_I = 0 with F as above) and error_max = sqrt of the largest inlier's squared residual, in
 * pixels, when valid.  A pair with at most 5 correspondences returns (0, 0) and no iteration. */
int b200m_acransac_essential_pairs(b200m_ctx* ctx, int n_pairs, const int64_t* offsets, const double* corr, const int32_t* wh, const double* K,
                                   const uint32_t* mt_state, int mt_state_per_pair, int64_t max_iteration, double precision, uint8_t* valid,
                                   int32_t* n_inliers, uint32_t* inliers, double* E, double* error_max, double* min_nfa, int32_t* iterations,
                                   uint32_t* mt_state_out);
/* GeometricFilterMatrix_F_AC::geometricEstimation_Mat_ACRANSAC<Fundamental10PSolver, Fundamental10PModel> (the
 * fundamental_with_distortion filter on a planar pair) for every pair: ACRANSAC over RelativePoseKernel<Fundamental10PSolver,
 * FundamentalEpipolarDistanceError, UnnormalizerT, Fundamental10PModel>, 10-point samples, at most 10 models a sample.
 * Arguments as in b200m_acransac_fundamental_pairs (one generator state that every pair starts from: the filter takes it by value).
 * F[9 * n_pairs]: the model's matrix (Fundamental10PModel::getMatrix(), row-major, unnormalised N2^T F N1 like the F call's).  It is
 * the reference's model matrix: the solver fits [x_I, y_I, 1 + l1 r_I^2] F [x_J, y_J, 1 + l2 r_J^2]^T = 0 on preconditioned points,
 * while the residual, errorMax and a guided step read it as the point-to-line error of F x_I on undistorted pixels.
 * L[2 * n_pairs]: the same model's (l1, l2) (getRadialDistortion()), in preconditioned units: the unnormaliser leaves it as is; 0 for
 * a pair without a model.  The filter does not use L.  A pair with at most 10 correspondences returns (0, 0) and no iteration. */
int b200m_acransac_fundamental_distortion_pairs(b200m_ctx* ctx, int n_pairs, const int64_t* offsets, const double* corr, const int32_t* wh,
                                                const uint32_t* mt_state, int64_t max_iteration, double precision, uint8_t* valid,
                                                int32_t* n_inliers, uint32_t* inliers, double* F, double* L, double* error_max, double* min_nfa,
                                                int32_t* iterations);
/* instrumentation of the last a-contrario RANSAC call (b200m_acransac_fundamental_pairs, b200m_acransac_homography_pairs,
 * b200m_acransac_fundamental_spherical_pairs, b200m_acransac_essential_pairs or b200m_acransac_fundamental_distortion_pairs): stats =
 * {models evaluated in the a-contrario mode, of them skipped by the histogram bound, scored exactly, kernel launches}; returns its GPU
 * time in ms */
double b200m_acransac_last_stats(const b200m_ctx* ctx, int64_t stats[4]);
/* the `better` events of the last a-contrario RANSAC call's pair `pair` (F, H, spherical F, E or F10): the iterations at which a better model was found
 * and the new minNFA of each (the first `cap`, at most 256; either pointer may be NULL); returns their number.  The getters of the
 * last call take the context's lock, so a concurrent call on the same context cannot rewrite what they read. */
int b200m_acransac_last_trace(const b200m_ctx* ctx, int pair, int32_t* iters, double* nfa, int cap);
/* debug, every model: 1 (default) = certified skip of models that cannot beat the running minNFA; 0 = score every model exactly */
int b200m_ctx_set_acransac_skip(b200m_ctx* ctx, int on);
/* ---- geometric filtering: homography growing (K12) ------------------------------------------------------------------ */
/* filterMatchesByHGrowing (GeometricFilterMatrix_HGrowing.cpp:108-194, the homography_growing filter) for every work item of a list,
 * results in input order.  A work item is one (pair, describer type) with its putatives in the caller's order:
 *   offsets    n_items + 1 ascending, offsets[0] = 0; item k owns putatives offsets[k] .. offsets[k + 1] - 1, at most 262144
 *   feat       offsets[n_items] x 8 floats: xI, yI, scaleI, orientationI, xJ, yJ, scaleJ, orientationJ (the two PointFeatures)
 *   parameters GrowParameters (tolerances >= 0 and finite, min_inliers_to_refine >= 1, nb_refining_iterations 0..64) and
 *              HGrowingFilteringParam (max_nb_homographies 0..64, min_nb_matches_per_h >= 0); the reference's defaults are
 *              20, 10, 5, 6, 8, 10, 20
 * Outputs (max_h = max_nb_homographies):
 *   n_homographies[n_items]; H[n_items x max_h x 9] (row-major, x_J ~ H x_I); counts[n_items x max_h];
 *   inliers[offsets[n_items]]: item k's stored matches as putative indices (0-based within the item) from inliers[offsets[k]] on, in
 *              outGeometricInliers order (homography by homography, each in putative order); the rest of its range is left as is
 *   trace[n_items x max_h x 3] or NULL: per round, the chosen seed's position in that round's remaining list (-1: no seed grew, which
 *              ends the item) and the best set's size before and after refineHomography
 *   rounds[n_items] or NULL: the rounds each item ran
 * The whole list is checked before anything runs; a bad argument returns B200M_ERR_ARG and queues nothing. */
int b200m_hgrowing_pairs(b200m_ctx* ctx, int n_items, const int64_t* offsets, const float* feat, double similarity_tolerance,
                         double affinity_tolerance, double homography_tolerance, int min_inliers_to_refine, int nb_refining_iterations,
                         int max_nb_homographies, int min_nb_matches_per_h, int32_t* n_homographies, double* H, int32_t* counts,
                         int32_t* inliers, int32_t* trace, int32_t* rounds);
/* instrumentation of the last b200m_hgrowing_pairs: stats = {seeds grown (speculative grows included), seeds the reference skips as
 * already used, rounds over all items}; returns its GPU time in ms */
double b200m_hgrowing_last_stats(const b200m_ctx* ctx, int64_t stats[3]);
/* debug: seeds per item grown speculatively per window (default 256, 1..4096); 1 is the reference's sequential loop.  Results do not
 * depend on it. */
int b200m_ctx_set_hgrowing_window(b200m_ctx* ctx, int window);
/* host only: std::mt19937(seed) as 625 words (see mt_state) */
void b200m_mt19937_seed(uint32_t seed, uint32_t state[625]);
/* host only (debug): the engine's sampler on the CPU.  `draws` consecutive randSample(g, 0, range, 7) from `state`: the samples in
 * their order (draws x 7), and the state after each draw (draws x 625) when states != NULL.  range >= 8. */
int b200m_debug_rand_sample(const uint32_t state[625], int range, int draws, uint32_t* out, uint32_t* states);
/* the same for sample_size 4 (Homography4PSolver; range >= 5) or 7: out is draws x sample_size */
int b200m_debug_rand_sample_k(const uint32_t state[625], int sample_size, int range, int draws, uint32_t* out, uint32_t* states);

/* ---- instrumentation ------------------------------------------------------------------------------------------ */
/* The b200m_last_* getters report the last successful b200m_match_pairs, b200m_guided_match(_model, _pairs), b200m_guided_match_positions_pairs,
 * b200m_guided_match_fast_pairs or b200m_knn on the context, whichever came last; a value that call does not measure reads 0 (b200m_knn sets only
 * b200m_last_tc_pairs: 1 when it ran on the tensor-core kernel).  They take the context's lock.  The a-contrario RANSAC calls have
 * their own (b200m_acransac_last_stats) and leave these alone. */
/* GPU time of the last call between its first and last enqueue (CUDA events on the context's stream), ms */
double b200m_last_gpu_ms(const b200m_ctx* ctx);
/* summed device time of the search kernel launches (tensor-core / exact / Hamming) in the last call, ms; the guided calls: their
 * search kernel (b200m_guided_match_fast_pairs: its candidate kernel) */
double b200m_last_search_kernel_ms(const b200m_ctx* ctx);
/* kernel launches issued by the last call */
int b200m_last_launches(const b200m_ctx* ctx);
/* pairs of the last call that ran on the tensor-core kernel */
int b200m_last_tc_pairs(const b200m_ctx* ctx);
/* candidates whose re-scored best distance differed from the tensor-core value (must stay 0); cumulative over the context's life */
unsigned b200m_exactness_errors(const b200m_ctx* ctx);
/* total raw records (matches before host finishing) produced by the last call; b200m_guided_match(_model, _pairs) and
 * b200m_guided_match_positions_pairs: its matches, b200m_guided_match_fast_pairs: the candidate distances it evaluated */
int64_t b200m_last_records(const b200m_ctx* ctx);
/* pairs of the last call that ran on the tensor-core FILTER kernel for real-valued fp32 descriptors (fp16-rounded GEMM + rigorous error
 * bound + exact re-scoring in the reference's arithmetic), and the queries among them the bound could not decide, which were searched
 * exactly over the whole database image (exact_rows fallback) */
int b200m_last_real_tc_pairs(const b200m_ctx* ctx);
int64_t b200m_last_fallback_rows(const b200m_ctx* ctx);
/* the tensor-core pairs of the last call (counted in b200m_last_tc_pairs too) whose two views are stored as uchar and ran on the 8-bit
 * tensor cores (exact int32 distances) */
int b200m_last_u8_tc_pairs(const b200m_ctx* ctx);
/* the u8 pairs of the last b200m_match_pairs (counted in b200m_last_u8_tc_pairs too) that ran on the u8 norm-GEMM kernel: query view
 * without a component above 127, database view of at least 128 rows whose squared norms fit its limbs (<= 1,011,967), and
 * B200M_U8_NORM_GEMM not set to 0 */
int b200m_last_u8_norm_gemm_pairs(const b200m_ctx* ctx);
/* batches the last b200m_match_pairs split its directed pairs into (skipped pairs included); 0 after the other calls */
int b200m_last_batches(const b200m_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* B200MATCH_H_ */

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
 * consumer warpgroups, unused); enable!=0 allocates,
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

/* ---- instrumentation ------------------------------------------------------------------------------------------ */
/* GPU time of the last b200m_match_pairs between its first and last enqueue (CUDA events on the context's stream), ms */
double b200m_last_gpu_ms(const b200m_ctx* ctx);
/* summed device time of the search kernel launches (tensor-core / exact / Hamming) in the last call, ms */
double b200m_last_search_kernel_ms(const b200m_ctx* ctx);
/* kernel launches issued by the last call */
int b200m_last_launches(const b200m_ctx* ctx);
/* pairs of the last call that ran on the tensor-core kernel */
int b200m_last_tc_pairs(const b200m_ctx* ctx);
/* candidates whose re-scored best distance differed from the tensor-core value (must stay 0) */
unsigned b200m_exactness_errors(const b200m_ctx* ctx);
/* total raw records (matches before host finishing) produced by the last call */
int64_t b200m_last_records(const b200m_ctx* ctx);
/* pairs of the last call that ran on the tensor-core FILTER kernel for real-valued fp32 descriptors (fp16-rounded GEMM + rigorous error
 * bound + exact re-scoring in the reference's arithmetic), and the queries among them the bound could not decide, which were searched
 * exactly over the whole database image (exact_rows fallback) */
int b200m_last_real_tc_pairs(const b200m_ctx* ctx);
int64_t b200m_last_fallback_rows(const b200m_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* B200MATCH_H_ */

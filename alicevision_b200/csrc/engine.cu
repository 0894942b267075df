// Host side of the engine behind the C ABI (include/b200match.h): view residency in HBM, pair batching,
// kernel launches on one CUDA stream, record read-back and the host "finishing" stage that reproduces
// RegionsMatcher::Match's tail (matching/RegionsMatcher.hpp:153-175) and the cross check
// (matchingImageCollection/ImageCollectionMatcher_generic.cpp:83-111).
//
// There is deliberately no CPU search path in this file: every distance is computed by a CUDA kernel.
#include "../../include/b200match.h"

#include "common.cuh"
#include "finish.cuh"
#include "guided.cuh"
#include "acransac.cuh"
#include "hgrowing.cuh"
#include "guided_fast.cuh"
#include "hamming.cuh"
#include "l2_exact.cuh"
#include "l2_tc.cuh"
#include "prep.cuh"
#include "verify.cuh"
#include "hostconv.hpp"
#include "cuda_owner.cuh"

#include <cub/cub.cuh>
#include <pthread.h>
#include <sched.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <fstream>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <queue>
#include <set>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

using namespace b200m;

// ------------------------------------------------------------------------------------------------ errors
static thread_local std::string g_err;
static int fail(int code, const std::string& msg) { g_err = msg; return code; }
namespace b200m { int set_error(int code, const std::string& msg) { return fail(code, msg); } }   // for CK and the other translation units

// ------------------------------------------------------------------------------------------------ small thread pool
// CPUs of the NUMA node a GPU hangs off (sysfs), intersected with the CPUs this process may use; empty set = unknown / do not pin.
// With one engine process (or context) per GPU the staging copies, the pinned ring and the finishing threads then stay on the
// socket whose PCIe root the GPU is attached to (round-1 verdict: GPUs 0-3 / 4-7 sit on different nodes and nothing was pinned).
struct CpuSet { cpu_set_t set; int count = 0; CpuSet() { CPU_ZERO(&set); } };
static CpuSet numa_cpus_of_device(int device) {
  CpuSet out;
  if (const char* e = getenv("B200M_NUMA")) if (atoi(e) == 0) return out;
  char bus[64] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) { cudaGetLastError(); return out; }
  for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
  int node = -1;
  { std::ifstream f(std::string("/sys/bus/pci/devices/") + bus + "/numa_node"); if (!(f >> node)) node = -1; }
  if (node < 0) return out;
  std::string list;
  { std::ifstream f("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist"); if (!std::getline(f, list)) return out; }
  cpu_set_t allowed; CPU_ZERO(&allowed);
  if (sched_getaffinity(0, sizeof(allowed), &allowed) != 0) return out;
  size_t pos = 0;
  while (pos < list.size()) {                       // "0-31,64-95"
    size_t end = list.find(',', pos); if (end == std::string::npos) end = list.size();
    const std::string tok = list.substr(pos, end - pos);
    int a = 0, b = 0;
    if (sscanf(tok.c_str(), "%d-%d", &a, &b) == 2) {} else if (sscanf(tok.c_str(), "%d", &a) == 1) b = a; else { pos = end + 1; continue; }
    for (int c = a; c <= b && c < CPU_SETSIZE; ++c) if (CPU_ISSET(c, &allowed)) { CPU_SET(c, &out.set); ++out.count; }
    pos = end + 1;
  }
  if (out.count < 2) { CPU_ZERO(&out.set); out.count = 0; }   // a node with (almost) no usable CPU: leave the threads alone
  return out;
}
static void pin_this_thread(const CpuSet& cs) { if (cs.count > 0) pthread_setaffinity_np(pthread_self(), sizeof(cs.set), &cs.set); }

class Pool {
 public:
  explicit Pool(int n, const CpuSet& cs = CpuSet()) : cs_(cs) { resize(n); }
  ~Pool() { stop(); }
  void resize(int n) {
    stop();
    quit_ = false;
    for (int i = 0; i < std::max(1, n); ++i) th_.emplace_back([this] { pin_this_thread(cs_); run(); });
  }
  void submit(std::function<void()> f) {
    { std::lock_guard<std::mutex> l(mu_); q_.push(std::move(f)); ++pending_; }
    cv_.notify_one();
  }
  void wait() { std::unique_lock<std::mutex> l(mu_); done_.wait(l, [this] { return pending_ == 0; }); }
  int size() const { return (int)th_.size(); }

 private:
  void stop() {
    { std::lock_guard<std::mutex> l(mu_); quit_ = true; }
    cv_.notify_all();
    for (auto& t : th_) t.join();
    th_.clear();
  }
  void run() {
    for (;;) {
      std::function<void()> f;
      {
        std::unique_lock<std::mutex> l(mu_);
        cv_.wait(l, [this] { return quit_ || !q_.empty(); });
        if (q_.empty()) return;
        f = std::move(q_.front()); q_.pop();
      }
      f();
      { std::lock_guard<std::mutex> l(mu_); if (--pending_ == 0) done_.notify_all(); }
    }
  }
  std::vector<std::thread> th_;
  std::queue<std::function<void()>> q_;
  std::mutex mu_;
  std::condition_variable cv_, done_;
  int pending_ = 0;
  bool quit_ = false;
  CpuSet cs_;
};

// Completion tracking for one group of pool tasks (one batch of finishing work).
struct TaskGroup {
  std::mutex mu; std::condition_variable cv; int left = 0;
  void add(int n) { std::lock_guard<std::mutex> l(mu); left += n; }
  void done() { std::lock_guard<std::mutex> l(mu); if (--left == 0) cv.notify_all(); }
  void wait() { std::unique_lock<std::mutex> l(mu); cv.wait(l, [this] { return left == 0; }); }
};

// Recycles large host blocks (per-batch finishing arenas, result arrays) across calls: a fresh 100 MB allocation costs
// ~25k page faults on first touch, more than the copy that fills it.  Shared by the context and its results.
struct Recycler {
  struct Block { b200m_match* p = nullptr; size_t cap = 0; };
  std::mutex mu; std::vector<Block> free_blocks;
  Block take(size_t n) {
    n = std::max<size_t>(n, 1);
    {
      std::lock_guard<std::mutex> l(mu);
      size_t best = free_blocks.size();
      for (size_t i = 0; i < free_blocks.size(); ++i)
        if (free_blocks[i].cap >= n && (best == free_blocks.size() || free_blocks[i].cap < free_blocks[best].cap)) best = i;
      if (best != free_blocks.size()) { Block b = free_blocks[best]; free_blocks.erase(free_blocks.begin() + best); return b; }
    }
    Block b; b.cap = n + n / 8; b.p = static_cast<b200m_match*>(::operator new(b.cap * sizeof(b200m_match)));
    return b;
  }
  void give(Block b) {
    if (!b.p) return;
    std::lock_guard<std::mutex> l(mu);
    if (free_blocks.size() >= 24) {          // keep the pool bounded: drop the smallest
      size_t sm = 0;
      for (size_t i = 1; i < free_blocks.size(); ++i) if (free_blocks[i].cap < free_blocks[sm].cap) sm = i;
      if (free_blocks[sm].cap < b.cap) std::swap(free_blocks[sm], b);
      ::operator delete(b.p);
      return;
    }
    free_blocks.push_back(b);
  }
  ~Recycler() { for (auto& b : free_blocks) ::operator delete(b.p); }
};

// ------------------------------------------------------------------------------------------------ data model
struct ViewHost {
  uint32_t id = 0;
  int m = 0, dim = 0, dtype = 0, m_pad = 0;
  void* raw = nullptr; __half* h16 = nullptr; float* nbh = nullptr; float* nrm = nullptr; __half* aug16 = nullptr;
  __half* augq16 = nullptr; float* err = nullptr; uint32_t* stats = nullptr;   // real-valued tensor-core path (prep.cuh): query-side limbs, rounding-error bounds
  void* arena = nullptr; void* raw_own = nullptr;     // the one allocation all device buffers of the view live in; a separately owned `raw`
  bool stored_u8 = false;     // dtype == DT_F32 whose values are integers in 0..255: staged and kept on the device as uchar (hostconv.hpp)
  int32_t* nb32 = nullptr;    // uchar-stored tensor-core views: int32 squared norms of the u8 kernel (prep.cuh)
  uint8_t* limb8 = nullptr;   // ... and the 32 norm limbs per row of the u8 norm-GEMM kernel (prep.cuh)
  float* d_xy = nullptr; uint32_t* d_yrank = nullptr;   // positions + rank of y on the device (device finishing stage, finish.cuh)
  double2* d_geom = nullptr;  // b200m_set_view_geometry: the (undistorted) positions guided matching uses instead of xy; own allocation
  bool failed = false;       // its upload job failed: the device buffers were never filled
  std::vector<float> xy;      // m x 2 positions (host copy: finishing of views that are not in general position, cross check)
  uint32_t flags = 0; bool flags_known = true;
  uint64_t seq = 0;           // upload order (monotonic per context)
  bool ready = false;         // copies + preparation kernel complete on the device and flags read back
  // "all x distinct and all y distinct", decided by the first finishing task that needs it
  struct PosLazy { std::mutex mu; int state = 0; };
  std::shared_ptr<PosLazy> pos = std::make_shared<PosLazy>();
  bool generic_pos() const;
  int store_dtype() const { return stored_u8 ? (int)DT_U8 : dtype; }
  bool tc_capable() const { return dtype != DT_BIN && dim == 128 && m > 0; }
  bool tc_ok() const { return tc_capable() && (flags & VF_EXACT_MASK) == 0; }
  // real-valued rows may take the tensor-core FILTER path (MODE_REAL): fp16 range and the half-norm limbs must hold, integers need not
  bool real_ok() const { return tc_capable() && (flags & (VF_RANGE | VF_NORM)) == 0 && m <= REAL_MAX_ROWS; }
  // uchar-stored tensor-core view as the query / the database of the u8 norm-GEMM kernel (l2_tc.cuh NG).  A database needs one full tile of
  // rows: then at least two chunks hold real rows, and a chunk of padding (whose value the limbs set lower than the u8 kernel's) can never
  // be one of the two smallest chunk minima the pre-test reads.
  bool ng_query_ok() const { return limb8 && store_dtype() == DT_U8 && (flags & VF_U8_WIDE) == 0; }
  bool ng_db_ok() const { return limb8 && store_dtype() == DT_U8 && (flags & VF_U8_NORMCAP) == 0 && m >= tc::BN; }
};

struct UploadJob {
  int n_views = 0, dim = 0; size_t esz = 1;
  std::vector<int> slots; std::vector<const void*> descs; std::vector<int> counts;
  std::shared_ptr<std::vector<int>> bad = std::make_shared<std::vector<int>>();   // per view: the checked f32 -> u8 conversion hit a value it cannot hold
};

constexpr int PAIR_CAP = 4096;            // directed pairs per batch
constexpr long CAND_CAP = 4l << 20;       // candidate slots per batch (sum of m_j)
constexpr long ITEM_CAP = CAND_CAP / 64 + PAIR_CAP;
constexpr long SLOT_CAP = 8l << 20;       // database rows per batch (sum of m_i): scratch of the device finishing stage
constexpr int META_INTS = 3 * PAIR_CAP + 3;   // pinned per-batch read-back: counts | offsets (+1) | finishing counts | fallback rows of the real-valued path

struct BatchBuf {
  DeviceBuffer<PairDev> d_pairs; DeviceBuffer<WorkItem> d_items; DeviceBuffer<Cand> d_cands; DeviceBuffer<int> d_count, d_off;
  DeviceBuffer<Rec> d_out;
  DeviceBuffer<FinMatch> d_fin; DeviceBuffer<int> d_fin_count; DeviceBuffer<uint32_t> d_scratch;   // device finishing stage (finish.cuh)
  DeviceBuffer<uint32_t> d_candx; DeviceBuffer<uint4> d_fb; DeviceBuffer<int> d_fb_count;      // fallback lists: d_fb_count = [overflow count, total]
  DeviceBuffer<uint4> d_fb_pair; DeviceBuffer<int> d_fb_pair_cnt;    // real-valued path: 5th candidate word, fallback list (pair, query)
  PinnedBuffer<PairDev> h_pairs; PinnedBuffer<WorkItem> h_items; PinnedBuffer<int> h_meta; PinnedBuffer<Rec> h_out;
  Event ev_meta, ev_copy, ev_tab;
  // the regions of the meta block (META_INTS): per-pair record counts, record offsets (np + 1, the last one the batch's total),
  // per-pair counts of the device finishing stage, and the fallback rows of the real-valued path
  int* meta_counts() const { return h_meta; }
  int* meta_offsets() const { return h_meta + PAIR_CAP; }
  int* meta_fin_counts() const { return h_meta + 2 * PAIR_CAP + 2; }
  int* meta_fallback_rows() const { return h_meta + 3 * PAIR_CAP + 2; }
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// grow-only device scratch of b200m_knn (Surface 1)
struct KnnScratch {
  DeviceBuffer<> raw; DeviceBuffer<__half> h16; DeviceBuffer<float> nbh, nrm; DeviceBuffer<__half> aug16, augq16; DeviceBuffer<float> err;
  DeviceBuffer<Cand> cands; DeviceBuffer<int32_t> idx; DeviceBuffer<uint32_t> dist; DeviceBuffer<WorkItem> items; DeviceBuffer<uint8_t> small;
};

// grow-only scratch of b200m_guided_match_fast_pairs (guided_fast.cuh): one batch of pairs at a time
struct GuidedFastScratch {
  enum { PAIRS, LBUCKET, BEST, SECOND, BCOUNT, BOFF, CSR, RSTART, RCOUNT, RCOFF, RPAIR, KEEP, KPOS, OUT, PSTART, EXPAND, TEMP, NBUF };
  DeviceBuffer<> d[NBUF];
  PinnedBuffer<FastPair> h_pairs;
  PinnedBuffer<> h_meta;                      // read-back of the candidate total and the per-pair starts
  PinnedBuffer<uint2> h_out;                  // read-back of the matches
  Event ev_c0, ev_c1;                         // candidate-kernel timing
};

// grow-only scratch of b200m_guided_match_pairs and b200m_guided_match_positions_pairs (guided.cuh): one batch of pairs at a time
struct GuidedScratch {
  enum { PAIRS, BESTJ, KEEP, KPOS, OUT, EXPAND, TEMP, YRANK, REC, KEEP2, NBUF };
  DeviceBuffer<> d[NBUF];
  PinnedBuffer<GuidedPair> h_pairs;
  PinnedBuffer<const uint32_t*> h_yrank;      // position-only call: per pair, the left view's yrank when it is decorated on the device
  PinnedBuffer<> h_out;                       // read-back of the per-pair starts and the matches, one copy
  Event ev_k0, ev_k1;                         // search-kernel timing
};

// grow-only scratch of b200m_acransac_fundamental_pairs, b200m_acransac_homography_pairs and
// b200m_acransac_fundamental_spherical_pairs (acransac.cuh); the last call's instrumentation and trace, whichever model it estimated
struct AcransacScratch {
  DeviceBuffer<char> d;
  bool skip = true;                                   // certified skip (b200m_ctx_set_acransac_skip)
  double last_ms = 0; int64_t stats[4] = {0, 0, 0, 0};
  std::vector<int32_t> trace; std::vector<double> trace_nfa; std::vector<int32_t> n_trace;   // last call: kTraceCap entries per pair
  Event ev0, ev1;
};

// grow-only scratch of b200m_hgrowing_pairs (hgrowing.cuh): the call's features and outputs, and one batch's lists, bitsets, seed
// slots and grow-warp bitsets; the last call's instrumentation
struct HgrowingScratch {
  DeviceBuffer<char> d;
  int window = 256;                                   // seeds per item and window (b200m_ctx_set_hgrowing_window)
  double last_ms = 0; int64_t stats[3] = {0, 0, 0};
  Event ev0, ev1;
};

// What the last b200m_match_pairs, b200m_guided_match_pairs (and its one-pair forms), b200m_guided_match_positions_pairs, b200m_guided_match_fast_pairs
// or b200m_knn measured (b200m_last_*);
// a field the call does not measure is 0
struct LastCall {
  double gpu_ms, search_ms;
  int launches, tc_pairs, real_pairs, u8_pairs;
  int64_t records, fallback_rows;
  int batches;                // b200m_match_pairs only
  int u8_norm_gemm_pairs;     // b200m_match_pairs only: the u8 pairs on the norm-GEMM kernel
};

// Members are released in reverse order of declaration, after ~b200m_ctx has stopped the uploader and the pool and freed the views:
// the streams go last.
struct b200m_ctx {
  ~b200m_ctx();
  int device = 0, num_sms = 148;
  Stream stream, copy_stream, up_stream, tab_stream, pack_stream;
  AcransacScratch acr;
  HgrowingScratch hgr;
  KnnScratch knn;
  GuidedFastScratch gf;
  long gf_left_cap = 1l << 21;    // left features per internal batch of b200m_guided_match_fast_pairs (B200M_GUIDED_FAST_LEFT_CAP)
  GuidedScratch gm;
  long gm_left_cap = 1l << 21;    // left features per internal batch of b200m_guided_match_pairs (B200M_GUIDED_LEFT_CAP)
  bool pipe_streams = true;       // tables / packing+finishing on their own streams (B200M_PIPE_STREAMS=0: everything on the search stream)
  EncodeTiledFn encode = nullptr;
  std::deque<ViewHost> views;     // deque: references stay valid while pool tasks (position checks) run
  std::unordered_map<uint32_t, int> slot_of;
  std::vector<int> free_slots;    // slots of removed views (b200m_remove_view), reused by later uploads
  DeviceBuffer<ViewDev> d_views; DeviceBuffer<uint32_t> d_flags; int view_cap = 0;
  BatchBuf buf[2]; bool bufs_ready = false;
  // upload staging: pageable caller memory -> pinned ring (parallel memcpy on the pool) -> async H2D
  static constexpr int NSTG = 24;
  PinnedBuffer<char> stg[NSTG]; Event stg_ev[NSTG];
  PinnedBuffer<ViewDev> h_views;  // pinned mirror of the device view table (source of the async table updates)
  PinnedBuffer<uint32_t> h_flags; // pinned: per-slot exactness flags, copied back behind each view's preparation kernel
  std::vector<Event> view_ev;     // per slot: recorded on up_stream when the view is complete on the device
  Event ev_alloc;                 // search stream -> upload stream: the view buffers of the current job are allocated
  // uploader thread (one job at a time, FIFO)
  std::thread up_thread; std::mutex up_mu; std::condition_variable up_cv;
  std::deque<UploadJob> up_jobs; bool up_quit = false; int up_active = 0;
  uint64_t up_issued_seq = 0, next_seq = 0;   // last view whose ready event was recorded / last sequence number handed out
  int up_rc = 0; std::string up_err;
  // the entry points that touch views, batch buffers or the stream serialise on this lock: one context may be shared by
  // several host threads (e.g. IRegionsMatcher adaptors created from an OpenMP region); calls simply queue up
  mutable std::recursive_mutex api_mu;
  DeviceBuffer<unsigned> d_err;
  DeviceBuffer<long long> d_trace;  // optional pipeline trace of CTA 0 (debug)
  std::vector<Event> tev;         // search-kernel timing events, reused across calls
  Event ev_start, ev_end;
  std::unique_ptr<Pool> pool;
  CpuSet cpus;                    // CPUs of the GPU's NUMA node (pool, uploader thread); empty = not pinned
  bool u8_staging = true;         // stage integer-valued fp32 descriptors as uchar (B200M_U8_STAGING=0 disables)
  bool device_finish = true;      // finishing stage on the device for views in general position (B200M_DEVICE_FINISH=0 disables)
  std::shared_ptr<Recycler> recycler = std::make_shared<Recycler>();
  bool force_exact = false;
  bool real_tc = true;            // real-valued fp32 pairs on the tensor-core filter kernel (B200M_REAL_TC=0: exact CUDA-core kernel as in round 1)
  bool u8_norm_gemm = true;       // u8 pairs whose views pass its gates on the norm-GEMM kernel (B200M_U8_NORM_GEMM=0: all on the u8 kernel)
  int first_batch_pairs = 16;     // while uploads are in flight: pairs of the first batch (then 2x per batch): how soon the GPU starts (B200M_FIRST_BATCH)
  long real_fused_rows = 6144;    // average database rows per item from which the real-valued re-scoring runs inside the filter kernel
  int tc_variant = 4;             // tensor-core kernel (l2_tc.cuh): 4 (default) = half-norms folded into the GEMM (AUG), 256-query work items;
                                  // half-norms added in the epilogue: 2 = 256-query items, 3 = 128-query items, 1 = 128-query items and
                                  // the stand-alone exactness pass (2-4 re-score in the kernel when the database images are long)
  LastCall last{};
  unsigned err_total = 0;
};

struct b200m_db { b200m_ctx* ctx; ViewHost v; int metric; ViewDev dev; };

struct b200m_result {
  std::vector<uint32_t> pair_ids; std::vector<int64_t> offsets;
  Recycler::Block matches;                  // uninitialised storage filled by parallel copies; returned to the recycler on free
  std::shared_ptr<Recycler> recycler;
  ~b200m_result() { if (recycler) recycler->give(matches); else if (matches.p) ::operator delete(matches.p); }
};

// ------------------------------------------------------------------------------------------------ helpers
// Device buffers of one view (stream-ordered allocations out of the default pool).
// ONE stream-ordered allocation per view, carved into its buffers (a view of 1024 features paid more for its ten allocations and ten
// frees than for its copy): raw | h16 | nbh | nrm | aug16 | augq16 | err | nb32 | limb8 | stats | yrank | xy, each 256-byte aligned; stats and
// yrank are adjacent so that one memset zeroes both.
// u8_norms: the int32 norms and the norm limbs of the u8 search kernels for a uchar-stored view (not for b200m_db_create's databases, which
// only MODE_KNN reads).
static int alloc_view_buffers(b200m_ctx* c, ViewHost& v, bool u8_norms = true) {
  const size_t esz = v.store_dtype() == DT_F32 ? 4 : 1;
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  const bool tcv = v.tc_capable(), pos = !v.xy.empty();
  if (tcv) v.m_pad = (v.m + tc::ROW_PAD - 1) / tc::ROW_PAD * tc::ROW_PAD;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += al(std::max<size_t>(bytes, 1)); return o; };
  const size_t o_raw = take(std::max<size_t>((size_t)v.m * v.dim * esz, 256));
  const size_t o_h16 = tcv ? take((size_t)v.m * 128 * 2) : 0, o_nbh = tcv ? take((size_t)v.m_pad * 4) : 0, o_nrm = tcv ? take((size_t)v.m_pad * 4) : 0;
  const size_t o_aug = tcv ? take((size_t)v.m_pad * 32) : 0, o_augq = tcv ? take((size_t)v.m_pad * 32) : 0, o_err = tcv ? take((size_t)v.m_pad * 4) : 0;
  const bool nb32 = tcv && u8_norms && v.store_dtype() == DT_U8;
  const size_t o_nb32 = nb32 ? take((size_t)v.m_pad * 4) : 0, o_limb = nb32 ? take((size_t)v.m_pad * 32) : 0;
  const size_t o_stats = tcv ? take(16) : 0;
  const size_t o_yrank = pos ? take((size_t)v.m * 4) : 0, o_xy = pos ? take((size_t)v.m * 8) : 0;
  char* base = nullptr;
  CK(cudaMallocAsync((void**)&base, off, c->stream));
  v.arena = base;
  v.raw = base + o_raw;
  if (tcv) {
    v.h16 = (__half*)(base + o_h16); v.nbh = (float*)(base + o_nbh); v.nrm = (float*)(base + o_nrm); v.aug16 = (__half*)(base + o_aug);
    v.augq16 = (__half*)(base + o_augq); v.err = (float*)(base + o_err); v.stats = (uint32_t*)(base + o_stats);
    v.nb32 = nb32 ? (int32_t*)(base + o_nb32) : nullptr;
    v.limb8 = nb32 ? (uint8_t*)(base + o_limb) : nullptr;
  }
  if (pos) { v.d_yrank = (uint32_t*)(base + o_yrank); v.d_xy = (float*)(base + o_xy); }
  return B200M_OK;
}
static void free_view_buffers(b200m_ctx* c, ViewHost& v) {
  if (v.arena) cudaFreeAsync(v.arena, c->stream);
  if (v.raw_own) cudaFreeAsync(v.raw_own, c->stream);      // fp32 re-upload of a view whose uchar staging failed late
  if (v.d_geom) cudaFreeAsync(v.d_geom, c->stream);        // re-uploading or removing a view drops its geometry positions
  v.arena = nullptr; v.raw_own = nullptr; v.d_geom = nullptr;
  v.raw = nullptr; v.h16 = nullptr; v.nbh = nullptr; v.nrm = nullptr; v.aug16 = nullptr; v.d_xy = nullptr; v.d_yrank = nullptr;
  v.augq16 = nullptr; v.err = nullptr; v.stats = nullptr; v.nb32 = nullptr; v.limb8 = nullptr;
}

// The shutdown that has to stay in this order; the owners among the members release the rest.  Also runs on the partly built
// context of a failed b200m_ctx_create (no uploader thread, no pool, streams missing).
b200m_ctx::~b200m_ctx() {
  {
    std::unique_lock<std::mutex> l(up_mu);
    up_cv.wait(l, [this] { return up_active == 0; });
    up_quit = true;
  }
  up_cv.notify_all();
  if (up_thread.joinable()) up_thread.join();
  if (pool) pool->wait();
  if (up_stream) cudaStreamSynchronize(up_stream);
  if (stream) cudaStreamSynchronize(stream);
  for (auto& v : views) free_view_buffers(this, v);      // stream-ordered
  if (stream) cudaStreamSynchronize(stream);
}

static int make_view_dev(b200m_ctx* c, const ViewHost& v, ViewDev& d) {
  std::memset(&d, 0, sizeof(d));
  d.raw = v.raw; d.h16 = v.h16; d.nbh = v.nbh; d.nrm = v.nrm; d.aug16 = v.aug16; d.m = v.m; d.dim = v.dim; d.dtype = v.store_dtype();
  d.yrank = v.d_yrank; d.augq16 = v.augq16; d.err = v.err; d.stats = v.stats;
  if (v.tc_capable()) {
    const cuuint64_t gdim[2] = {128, (cuuint64_t)v.m};
    const cuuint64_t gstr[1] = {256};
    const cuuint32_t estr[2] = {1, 1};
    {
      const cuuint32_t box[2] = {64, 128};
      CUresult r = c->encode(&d.tmap128, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)v.h16, gdim, gstr, box, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) return fail(B200M_ERR_CUDA, "cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
    }
    {
      const cuuint64_t adim[2] = {16, (cuuint64_t)v.m_pad};
      const cuuint64_t astr[1] = {32};
      const cuuint32_t abox[2] = {16, 128};
      CUresult r = c->encode(&d.tmap_aug, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)v.aug16, adim, astr, abox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) return fail(B200M_ERR_CUDA, "cuTensorMapEncodeTiled(aug) failed: " + std::to_string((int)r));
      r = c->encode(&d.tmap_augq, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)v.augq16, adim, astr, abox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) return fail(B200M_ERR_CUDA, "cuTensorMapEncodeTiled(augq) failed: " + std::to_string((int)r));
    }
    if (v.nb32 && v.store_dtype() == DT_U8) {
      // the uchar rows themselves as the u8 kernel's operand: 128-byte rows, the same SWIZZLE_128B layout as one fp16 K-block
      const cuuint64_t ustr[1] = {128};
      const cuuint32_t ubox[2] = {128, 128};
      d.nb32 = v.nb32;
      CUresult r = c->encode(&d.tmap_u8, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, (void*)v.raw, gdim, ustr, ubox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) return fail(B200M_ERR_CUDA, "cuTensorMapEncodeTiled(u8) failed: " + std::to_string((int)r));
      // the norm limbs of the norm-GEMM kernel: 32-byte rows in the 32-byte-swizzled layout of the fp16 augmentation columns
      const cuuint64_t ldim[2] = {32, (cuuint64_t)v.m_pad};
      const cuuint64_t lstr[1] = {32};
      const cuuint32_t lbox[2] = {32, 128};
      r = c->encode(&d.tmap_limb, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, (void*)v.limb8, ldim, lstr, lbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) return fail(B200M_ERR_CUDA, "cuTensorMapEncodeTiled(limb) failed: " + std::to_string((int)r));
    }
  }
  return B200M_OK;
}

static int run_prep(b200m_ctx* c, const ViewHost& v, uint32_t* d_flag, cudaStream_t st, bool zero_stats = true) {
  (void)c;
  if (!v.tc_capable()) return B200M_OK;
  const int grid = (v.m_pad + 7) / 8;
  if (zero_stats) CK(cudaMemsetAsync(v.stats, 0, 16, st));
  if (v.store_dtype() == DT_F32) prep_view_kernel<float><<<grid, 256, 0, st>>>((const float*)v.raw, v.m, v.h16, v.nbh, v.nrm, v.m_pad, d_flag, v.aug16, v.augq16, v.err, v.stats, nullptr, nullptr);
  else prep_view_kernel<uint8_t><<<grid, 256, 0, st>>>((const uint8_t*)v.raw, v.m, v.h16, v.nbh, v.nrm, v.m_pad, d_flag, v.aug16, v.augq16, v.err, v.stats, v.nb32, v.limb8);
  CK(cudaGetLastError());
  return B200M_OK;
}

static bool positions_generic(const std::vector<float>& xy, int m) {
  std::vector<float> xs(m), ys(m);
  for (int i = 0; i < m; ++i) { xs[i] = xy[2 * i]; ys[i] = xy[2 * i + 1]; }
  std::sort(xs.begin(), xs.end()); std::sort(ys.begin(), ys.end());
  return std::adjacent_find(xs.begin(), xs.end()) == xs.end() && std::adjacent_find(ys.begin(), ys.end()) == ys.end();
}
bool ViewHost::generic_pos() const {
  std::lock_guard<std::mutex> l(pos->mu);
  if (pos->state == 0) pos->state = (!xy.empty() && positions_generic(xy, m)) ? 2 : 1;
  return pos->state == 2;
}

static int ensure_view_capacity(b200m_ctx* c, int need) {
  if (need <= c->view_cap) return B200M_OK;
  int cap = std::max(256, c->view_cap * 2);
  while (cap < need) cap *= 2;
  DeviceBuffer<ViewDev> nv; DeviceBuffer<uint32_t> nf; PinnedBuffer<ViewDev> nh; PinnedBuffer<uint32_t> nhf;
  int rc;
  CK(cudaStreamSynchronize(c->stream));
  CK(cudaStreamSynchronize(c->up_stream));
  if ((rc = nh.reserve(sizeof(ViewDev) * cap)) || (rc = nhf.reserve(sizeof(uint32_t) * cap)) || (rc = nv.reserve(sizeof(ViewDev) * cap)) ||
      (rc = nf.reserve(sizeof(uint32_t) * cap)))
    return rc;
  std::memset(nhf, 0, sizeof(uint32_t) * cap);
  CK(cudaMemset(nf, 0, sizeof(uint32_t) * cap));
  if (c->view_cap) {
    std::memcpy(nh, c->h_views, sizeof(ViewDev) * c->view_cap);
    std::memcpy(nhf, c->h_flags, sizeof(uint32_t) * c->view_cap);
    CK(cudaMemcpy(nv, c->d_views, sizeof(ViewDev) * c->view_cap, cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy(nf, c->d_flags, sizeof(uint32_t) * c->view_cap, cudaMemcpyDeviceToDevice));
  }
  c->h_views = std::move(nh); c->h_flags = std::move(nhf); c->d_views = std::move(nv); c->d_flags = std::move(nf);   // the old tables go with the locals
  c->view_ev.resize(cap);
  c->view_cap = cap;
  return B200M_OK;
}

static int ensure_batch_buffers(b200m_ctx* c) {
  if (c->bufs_ready) return B200M_OK;
  for (BatchBuf& b : c->buf) {
    int rc;
    if ((rc = b.d_pairs.reserve(sizeof(PairDev) * PAIR_CAP)) || (rc = b.d_items.reserve(sizeof(WorkItem) * ITEM_CAP)) ||
        (rc = b.d_cands.reserve(sizeof(Cand) * CAND_CAP)) || (rc = b.d_count.reserve(sizeof(int) * PAIR_CAP)) ||
        (rc = b.d_off.reserve(sizeof(int) * (PAIR_CAP + 1))) || (rc = b.d_out.reserve(sizeof(Rec) * CAND_CAP)) ||
        (rc = b.d_fin.reserve(sizeof(FinMatch) * CAND_CAP)) || (rc = b.d_fin_count.reserve(sizeof(int) * PAIR_CAP)) ||
        (rc = b.d_scratch.reserve(sizeof(uint32_t) * 2 * SLOT_CAP)) ||
        (rc = b.d_candx.reserve(sizeof(uint32_t) * CAND_CAP)) || (rc = b.d_fb.reserve(sizeof(uint4) * CAND_CAP)) ||
        (rc = b.d_fb_count.reserve(2 * sizeof(int))) || (rc = b.d_fb_pair.reserve(sizeof(uint4) * (size_t)PAIR_CAP * FB_PER_PAIR)) ||
        (rc = b.d_fb_pair_cnt.reserve(sizeof(int) * PAIR_CAP)) ||
        (rc = b.h_pairs.reserve(sizeof(PairDev) * PAIR_CAP)) || (rc = b.h_items.reserve(sizeof(WorkItem) * ITEM_CAP)) ||
        (rc = b.h_meta.reserve(sizeof(int) * META_INTS)) || (rc = b.h_out.reserve(sizeof(Rec) * CAND_CAP)) ||
        (rc = b.ev_meta.create(cudaEventDisableTiming)) || (rc = b.ev_copy.create(cudaEventDisableTiming)) ||
        (rc = b.ev_tab.create(cudaEventDisableTiming)))
      return rc;
  }
  CK(cudaFuncSetAttribute(tc::l2_top2_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::Lay<false>::SMEM_BYTES));
  CK(cudaFuncSetAttribute(tc::l2_top2_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::Lay<true>::SMEM_BYTES));
  CK(cudaFuncSetAttribute(tc::l2_top2_tc_kernel<true, tc::MODE_REAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::Lay<true, true>::SMEM_BYTES));
  CK(cudaFuncSetAttribute(tc::l2_top2_tc_kernel<true, tc::MODE_KNN>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::Lay<true>::SMEM_BYTES));
  CK(cudaFuncSetAttribute(tc::l2_top2_tc_u8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::Lay<false, false, true>::SMEM_BYTES));
  CK(cudaFuncSetAttribute(tc::l2_top2_tc_u8ng_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::Lay<false, false, true, true>::SMEM_BYTES));
  CK(cudaFuncSetAttribute(exact_rows_pairs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, XP_SMEM));
  CK(cudaFuncSetAttribute(exact_top2_kernel<float, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, EX_SMEM));
  CK(cudaFuncSetAttribute(exact_top2_kernel<uint8_t, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, EX_SMEM));
  CK(cudaFuncSetAttribute(exact_top2_kernel<float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, EX_SMEM));
  CK(cudaFuncSetAttribute(exact_top2_kernel<uint8_t, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, EX_SMEM));
  c->bufs_ready = true;
  return B200M_OK;
}

static cudaEvent_t timing_event(b200m_ctx* c, size_t& used) {
  if (used == c->tev.size()) { c->tev.emplace_back(); c->tev.back().create(); }   // a failed creation shows in the cudaEventRecord that follows
  return c->tev[used++];
}

// ------------------------------------------------------------------------------------------------ finishing (host)
namespace {

struct DecoKey { float x1, y1, x2, y2; b200m_match m; };
// The reference's comparator (matching/IndMatchDecorator.hpp:34-49) is not a strict weak order; its effect is
// defined by libstdc++'s std::set insertion walk, so the general path uses the same container with an
// equivalent predicate: "a before b" iff they differ in some coordinate, their left x differ, and a.y1 < b.y1.
struct DecoBefore {
  bool operator()(const DecoKey& a, const DecoKey& b) const {
    const bool same = a.x1 == b.x1 && a.y1 == b.y1 && a.x2 == b.x2 && a.y2 == b.y2;
    return !same && a.x1 != b.x1 && a.y1 < b.y1;
  }
};

// IndMatchDecorator<float>::getDeduplicated (IndMatchDecorator.hpp:57-69,84-98) of out[0..cnt) with the positions xi (left) and xj
// (right), m x 2 each, literally: the same container and insertion order.  Returns the number kept, written back to out.
int decorator_dedup(b200m_match* out, int cnt, const float* xi, const float* xj) {
  std::vector<DecoKey> keys; keys.reserve(cnt);
  for (int k = 0; k < cnt; ++k) { const b200m_match& m = out[k]; keys.push_back(DecoKey{xi[2 * m.i], xi[2 * m.i + 1], xj[2 * m.j], xj[2 * m.j + 1], m}); }
  std::set<DecoKey, DecoBefore> st(keys.begin(), keys.end());
  cnt = 0;
  for (const auto& k : st) out[cnt++] = k.m;
  return cnt;
}

// recs -> final IndMatches of one directed pair, written to out[0..n) (capacity n). Returns the number kept.
int finish_directed(const Rec* recs, int n, bool hamming, bool full, const ViewHost& vi, const ViewHost& vj, b200m_match* out) {
  int cnt = 0;
  for (int k = 0; k < n; ++k) {
    const Rec& r = recs[k];
    if (r.i == 0xFFFFFFFFu) continue;
    b200m_match m;
    m.i = r.i; m.j = r.j;                                    // IndMatch(i = database index, j = query index), RegionsMatcher.hpp:157-158
    if (hamming) {
      uint32_t d1, d2; std::memcpy(&d1, &r.d1, 4); std::memcpy(&d2, &r.d2, 4);
      m.distance_ratio = (float)(d1 / d2);                   // integer division, matching/filters.hpp:64 on unsigned
      m.distance = (float)d1;
    } else {
      m.distance_ratio = r.d1 / r.d2;                        // float division, filters.hpp:64
      m.distance = r.d1;
    }
    out[cnt++] = m;
  }
  if (!full || cnt == 0) return cnt;
  // IndMatch::getDeduplicated (IndMatch.hpp:52-58): every query j appears once, so this is a sort by (i, j).
  std::sort(out, out + cnt, [](const b200m_match& a, const b200m_match& b) { return a.i < b.i || (a.i == b.i && a.j < b.j); });
  // IndMatchDecorator::getDeduplicated (IndMatchDecorator.hpp:57-69,84-98)
  const float* xi = vi.xy.data(); const float* xj = vj.xy.data();
  if (vi.generic_pos()) {
    // All left x distinct and all left y distinct: two matches are "equivalent" iff they share the left feature,
    // the first inserted (smallest j) wins, and the in-order walk is ascending left y.
    int w = 0;
    for (int k = 0; k < cnt; ++k)
      if (k == 0 || out[k].i != out[k - 1].i) out[w++] = out[k];
    cnt = w;
    std::sort(out, out + cnt, [xi](const b200m_match& a, const b200m_match& b) { return xi[2 * a.i + 1] < xi[2 * b.i + 1]; });
  } else {
    cnt = decorator_dedup(out, cnt, xi, xj);
  }
  return cnt;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ C ABI
extern "C" {

const char* b200m_last_error(void) { return g_err.c_str(); }
int b200m_version(void) { return 100; }
int b200m_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int b200m_ctx_create(int device, void* stream, b200m_ctx** out) {
  if (!out) return fail(B200M_ERR_ARG, "out is null");
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return fail(B200M_ERR_CUDA, "no CUDA device: this engine has no CPU path"); }
  if (device < 0 || device >= n) return fail(B200M_ERR_ARG, "bad device ordinal");
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) return fail(B200M_ERR_UNSUPPORTED, "this build contains sm_90a code only (found sm_" + std::to_string(prop.major * 10 + prop.minor) + ")");
  std::unique_ptr<b200m_ctx> c(new b200m_ctx());
  c->device = device; c->num_sms = prop.multiProcessorCount;
  int rc;
  if (stream) c->stream.borrow((cudaStream_t)stream);
  else if ((rc = c->stream.create())) return rc;
  if ((rc = c->copy_stream.create()) || (rc = c->up_stream.create()) || (rc = c->tab_stream.create()) || (rc = c->pack_stream.create()) ||
      (rc = c->ev_alloc.create(cudaEventDisableTiming)))
    return rc;
  if (const char* e = getenv("B200M_PIPE_STREAMS")) c->pipe_streams = atoi(e) != 0;
  cudaDriverEntryPointQueryResult qres;
  void* fn = nullptr;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (!fn || qres != cudaDriverEntryPointSuccess) return fail(B200M_ERR_CUDA, "cuTensorMapEncodeTiled not available in this driver");
  c->encode = (EncodeTiledFn)fn;
  cudaMemPool_t mp;
  CK(cudaDeviceGetDefaultMemPool(&mp, device));
  uint64_t thr = ~0ull;
  CK(cudaMemPoolSetAttribute(mp, cudaMemPoolAttrReleaseThreshold, &thr));
  if ((rc = c->d_err.reserve(sizeof(unsigned int)))) return rc;
  CK(cudaMemset(c->d_err, 0, sizeof(unsigned int)));
  if ((rc = c->ev_start.create()) || (rc = c->ev_end.create())) return rc;
  c->cpus = numa_cpus_of_device(device);
  int ht = c->cpus.count > 0 ? c->cpus.count : (int)std::thread::hardware_concurrency();
  if (const char* e = getenv("B200M_HOST_THREADS")) ht = std::max(1, atoi(e));     // several engine processes sharing one host (one per GPU)
  c->pool.reset(new Pool(std::min(std::max(ht, 1), 32), c->cpus));
  if (const char* e = getenv("B200M_U8_STAGING")) c->u8_staging = atoi(e) != 0;
  if (const char* e = getenv("B200M_DEVICE_FINISH")) c->device_finish = atoi(e) != 0;
  if (const char* e = getenv("B200M_FIRST_BATCH")) c->first_batch_pairs = std::max(1, atoi(e));
  if (const char* e = getenv("B200M_REAL_TC")) c->real_tc = atoi(e) != 0;
  if (const char* e = getenv("B200M_U8_NORM_GEMM")) c->u8_norm_gemm = atoi(e) != 0;
  if (const char* e = getenv("B200M_REAL_FUSED_ROWS")) c->real_fused_rows = std::max(0l, atol(e));
  if (const char* e = getenv("B200M_GUIDED_FAST_LEFT_CAP")) c->gf_left_cap = std::max(1l, atol(e));
  if (const char* e = getenv("B200M_GUIDED_LEFT_CAP")) c->gm_left_cap = std::max(1l, atol(e));
  *out = c.release();
  return B200M_OK;
}

void b200m_ctx_destroy(b200m_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  delete c;
}

int b200m_ctx_set_host_threads(b200m_ctx* c, int n) {
  if (!c || n < 1) return fail(B200M_ERR_ARG, "bad arguments");
  c->pool->resize(std::min(n, 256));
  return B200M_OK;
}
int b200m_ctx_set_tc_variant(b200m_ctx* c, int variant) {
  if (!c || variant < 1 || variant > 4) return fail(B200M_ERR_ARG, "tc variant must be 1 (128-query items, stand-alone exactness pass), 2 (256-query items), 3 (128-query items) or 4 (256-query items, half-norms folded into the GEMM)");
  c->tc_variant = variant;
  return B200M_OK;
}
// Debug: enable (n>0) / read back the per-tile pipeline trace of CTA 0 of the tensor-core kernel.
// out receives 4 roles x TRACE_TILES x 4 SM-clock stamps: role 0 the TMA producer (slot free, loads issued), roles 1 and 2 the two
// consumer warpgroups (before / after the tile's wait, MMAs complete, epilogue done); role 3 is unused.
int b200m_debug_trace(b200m_ctx* c, int enable, long long* out, int n) {
  if (!c) return fail(B200M_ERR_ARG, "ctx is null");
  CK(cudaSetDevice(c->device));
  const size_t total = 4ull * ptx::TRACE_TILES * 4;
  if (enable && !c->d_trace) { if (int rc = c->d_trace.reserve(total * 8)) return rc; CK(cudaMemset(c->d_trace, 0, total * 8)); }
  if (out && c->d_trace) { CK(cudaStreamSynchronize(c->stream)); CK(cudaMemcpy(out, c->d_trace, std::min<size_t>(total, (size_t)n) * 8, cudaMemcpyDeviceToHost)); }
  if (!enable) c->d_trace = DeviceBuffer<long long>();
  return B200M_OK;
}
// Debug / test hook (host only, no GPU needed): the checked fp32 -> uchar conversion of the staging path (hostconv.hpp).
// which: 0 = the dispatching entry point (AVX2 when the CPU has it), 1 = the scalar reference.  Returns 1 when every value was an integer in 0..255.
int b200m_debug_convert_f32_u8(const float* src, uint8_t* dst, size_t n, int which) {
  if ((!src || !dst) && n) return -1;
  return (which == 1 ? f32_to_u8_checked_scalar(src, dst, n) : f32_to_u8_checked(src, dst, n)) ? 1 : 0;
}

int b200m_ctx_set_force_exact(b200m_ctx* c, int on) {
  if (!c) return fail(B200M_ERR_ARG, "ctx is null");
  c->force_exact = on != 0;
  return B200M_OK;
}

// ---- Surface 2: views -------------------------------------------------------------------------------------------
// Uploads run on their own thread and their own stream (`up_stream`): caller memory is pageable, so descriptors go through
// a ring of pinned staging buffers (pool threads memcpy chunks k+1..k+4 into pinned memory while the copy engine moves
// chunk k; the H2D of a chunk is issued four chunks behind its memcpy) and each view's preparation kernel, the copy of its
// exactness flags to pinned host memory and its "ready" event follow its last chunk.  b200m_match_pairs only waits for the
// views of the batch it is about to enqueue, so the search kernels of the first pairs run while later views are still
// being copied (the pair list is processed in order of view arrival when uploads are in flight).
static void publish_issued(b200m_ctx* c, uint64_t seq) {
  { std::lock_guard<std::mutex> l(c->up_mu); c->up_issued_seq = std::max(c->up_issued_seq, seq); }
  c->up_cv.notify_all();
}

static int run_upload(b200m_ctx* c, const UploadJob& job) {
  CK(cudaSetDevice(c->device));
  const bool timing = getenv("B200M_TIMING") != nullptr;
  auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  const double t_begin = now();
  CK(cudaStreamWaitEvent(c->up_stream, c->ev_alloc, 0));   // the stream-ordered allocations were made on the search stream
  // A chunk = what one staging buffer carries: a byte range of a view's descriptors copied as they are (CK_RAW), a range of an
  // integer-valued fp32 view converted to uchar on the way (CK_U8: `bytes` staged bytes = elements, read from 4x as many source
  // bytes), or the view's positions (CK_XY, after its last descriptor chunk).
  enum { CK_RAW = 0, CK_U8 = 1, CK_XY = 2 };
  struct Chunk { int view; int kind; size_t off, bytes; bool last; };
  std::vector<Chunk> chunks;
  const char* e_ch = getenv("B200M_UP_CHUNK_MB"); const char* e_parts = getenv("B200M_UP_PARTS");
  const size_t CH = (size_t)(e_ch ? std::max(1, atoi(e_ch)) : 4) << 20;
  const int max_parts = e_parts ? std::max(1, atoi(e_parts)) : 1;   // measured: splitting a chunk over threads is slower (profiles/r01d_upload_staging.md)
  for (int i = 0; i < job.n_views; ++i) {
    const ViewHost& v = c->views[job.slots[i]];
    const bool has_xy = v.d_xy != nullptr;
    const bool u8 = v.stored_u8;
    const size_t bytes = (size_t)job.counts[i] * job.dim * (u8 ? 1 : job.esz);
    const size_t step = u8 ? CH / 4 : CH;                  // a converted chunk reads 4x its size: keep the task length the same
    if (bytes == 0) chunks.push_back({i, CK_RAW, 0, 0, true});      // empty view: only its ready event
    for (size_t off = 0; off < bytes; off += step) chunks.push_back({i, u8 ? CK_U8 : CK_RAW, off, std::min(step, bytes - off), !has_xy && off + step >= bytes});
    if (has_xy && bytes) {
      const size_t xb = (size_t)job.counts[i] * 8;
      for (size_t off = 0; off < xb; off += CH) chunks.push_back({i, CK_XY, off, std::min(CH, xb - off), off + CH >= xb});
    }
  }
  for (int k = 0; k < b200m_ctx::NSTG; ++k) {
    int rc;
    if ((rc = c->stg_ev[k].create(cudaEventDisableTiming))) return rc;
    if (c->stg[k].capacity() < CH) CK(cudaEventSynchronize(c->stg_ev[k]));   // the last H2D out of the buffer that is replaced is done
    if ((rc = c->stg[k].reserve(CH))) return rc;
  }
  std::vector<int>& bad = *job.bad;
  double t_ring = 0, t_task = 0, t_fin = 0;                // B200M_TIMING: where the issuing thread waits
  auto finish_view = [&](int i) -> int {                   // runs right after the last chunk of view i was enqueued
    const int slot = job.slots[i];
    ViewHost& v = c->views[slot];
    if (v.stored_u8 && __atomic_load_n(&bad[i], __ATOMIC_ACQUIRE)) {
      // The probe of the first rows said "integers in 0..255" but a later value is not: upload the view as fp32 after all
      // (rare: the copy below goes through the driver's own pageable staging).  Buffers change -> the view table entry is rewritten.
      void* nr = nullptr;
      const size_t fb = (size_t)v.m * v.dim * 4;
      CK(cudaMallocAsync(&nr, std::max<size_t>(fb, 256), c->up_stream));
      CK(cudaMemcpyAsync(nr, job.descs[i], fb, cudaMemcpyHostToDevice, c->up_stream));
      v.raw = nr; v.raw_own = nr; v.stored_u8 = false;          // the uchar-sized region of the arena stays unused until the view goes
      int rc = make_view_dev(c, v, c->h_views[slot]);
      if (rc) return rc;
      CK(cudaMemcpyAsync(c->d_views + slot, c->h_views + slot, sizeof(ViewDev), cudaMemcpyHostToDevice, c->up_stream));
    }
    const bool flagged = v.tc_capable() || v.d_xy;
    if (flagged) CK(cudaMemsetAsync(c->d_flags + slot, 0, 4, c->up_stream));
    {
      // one memset for the per-view accumulators: stats (atomicMax) and, when the ranks are summed over several k ranges, yrank right behind
      const bool rank_sums = v.d_xy && v.m > PR_KRANGE;
      if (v.tc_capable()) CK(cudaMemsetAsync(v.stats, 0, rank_sums ? (size_t)((char*)v.d_yrank - (char*)v.stats) + (size_t)v.m * 4 : 16, c->up_stream));
      else if (rank_sums) CK(cudaMemsetAsync(v.d_yrank, 0, (size_t)v.m * 4, c->up_stream));
    }
    if (v.tc_capable()) {
      int rc = run_prep(c, v, c->d_flags + slot, c->up_stream, false);
      if (rc) return rc;
    }
    if (v.d_xy) {
      pos_rank_kernel<<<dim3((v.m + PR_THREADS - 1) / PR_THREADS, (v.m + PR_KRANGE - 1) / PR_KRANGE), PR_THREADS, 0, c->up_stream>>>((const float2*)v.d_xy, v.m, v.d_yrank, c->d_flags + slot);
      CK(cudaGetLastError());
    }
    if (flagged) CK(cudaMemcpyAsync(c->h_flags + slot, c->d_flags + slot, 4, cudaMemcpyDeviceToHost, c->up_stream));
    CK(cudaEventRecord(c->view_ev[slot], c->up_stream));
    publish_issued(c, v.seq);
    return B200M_OK;
  };
  const char* e_lag = getenv("B200M_UP_LAG");
  const int LAG = std::max(1, std::min(b200m_ctx::NSTG - 2, e_lag ? atoi(e_lag) : 12));   // chunks between a memcpy and its H2D (= memcpys in flight)
  std::vector<std::unique_ptr<TaskGroup>> grp(chunks.size());
  struct WaitAll {                                          // on every exit path: no staging task may outlive `grp`, `chunks` or the caller's buffers
    std::vector<std::unique_ptr<TaskGroup>>& g;
    ~WaitAll() { for (auto& x : g) if (x) x->wait(); }
  } wait_all{grp};
  auto issue_h2d = [&](size_t k) -> int {
    const Chunk& ch = chunks[k];
    const int sidx = (int)(k % b200m_ctx::NSTG);
    const double tw0 = timing ? now() : 0;
    grp[k]->wait();
    if (timing) t_task += now() - tw0;
    const ViewHost& v = c->views[job.slots[ch.view]];
    if (ch.bytes && !(ch.kind == CK_U8 && __atomic_load_n(&bad[ch.view], __ATOMIC_ACQUIRE))) {
      char* dst = ch.kind == CK_XY ? (char*)v.d_xy : (char*)v.raw;
      CK(cudaMemcpyAsync(dst + ch.off, c->stg[sidx], ch.bytes, cudaMemcpyHostToDevice, c->up_stream));
      CK(cudaEventRecord(c->stg_ev[sidx], c->up_stream));
    }
    if (ch.last) { const double tf0 = timing ? now() : 0; const int rc = finish_view(ch.view); if (timing) t_fin += now() - tf0; return rc; }
    return B200M_OK;
  };
  for (size_t k = 0; k < chunks.size(); ++k) {
    const Chunk& ch = chunks[k];
    const int sidx = (int)(k % b200m_ctx::NSTG);
    const double tr0 = timing ? now() : 0;
    CK(cudaEventSynchronize(c->stg_ev[sidx]));             // the H2D that last used this staging buffer is done (no-op when never recorded)
    if (timing) t_ring += now() - tr0;
    grp[k].reset(new TaskGroup());
    if (ch.bytes) {
      char* d = (char*)c->stg[sidx]; TaskGroup* g = grp[k].get();
      if (ch.kind == CK_U8) {
        grp[k]->add(1);
        const float* sp = (const float*)job.descs[ch.view] + ch.off; const size_t n = ch.bytes; int* flag = &bad[ch.view];
        c->pool->submit([=] {
          if (!__atomic_load_n(flag, __ATOMIC_RELAXED) && !f32_to_u8_checked(sp, (uint8_t*)d, n)) __atomic_store_n(flag, 1, __ATOMIC_RELEASE);
          g->done();
        });
      } else {
        // the pageable -> pinned copy of one chunk may be split over pool threads (B200M_UP_PARTS; default 1)
        const int parts = (int)std::max<size_t>(1, std::min<size_t>((size_t)max_parts, ch.bytes >> 19));
        grp[k]->add(parts);
        const char* sp = ch.kind == CK_XY ? (const char*)c->views[job.slots[ch.view]].xy.data() + ch.off : (const char*)job.descs[ch.view] + ch.off;
        for (int q = 0; q < parts; ++q) {
          const size_t a0 = ch.bytes * q / parts, a1 = ch.bytes * (q + 1) / parts;
          c->pool->submit([=] { std::memcpy(d + a0, sp + a0, a1 - a0); g->done(); });
        }
      }
    }
    if (k >= (size_t)LAG) { int rc = issue_h2d(k - LAG); if (rc) return rc; }
  }
  for (size_t k = chunks.size() >= (size_t)LAG ? chunks.size() - LAG : 0; k < chunks.size(); ++k) { int rc = issue_h2d(k); if (rc) return rc; }
  if (timing) { const double t_end = now(); CK(cudaStreamSynchronize(c->up_stream)); fprintf(stderr, "[b200m] upload job n=%d (%zu chunks): copies issued in %.2f ms (waiting: ring %.2f, staging tasks %.2f; per-view finish calls %.2f), drain %.2f ms\n", job.n_views, chunks.size(), t_end - t_begin, t_ring, t_task, t_fin, now() - t_end); }
  return B200M_OK;
}

static void uploader_main(b200m_ctx* c) {
  pin_this_thread(c->cpus);
  for (;;) {
    UploadJob job;
    {
      std::unique_lock<std::mutex> l(c->up_mu);
      c->up_cv.wait(l, [c] { return c->up_quit || !c->up_jobs.empty(); });
      if (c->up_jobs.empty()) return;
      job = std::move(c->up_jobs.front()); c->up_jobs.pop_front();
    }
    const int rc = run_upload(c, job);
    {
      std::lock_guard<std::mutex> l(c->up_mu);
      if (rc && !c->up_rc) { c->up_rc = rc; c->up_err = g_err; }
      if (rc) for (int slot : job.slots) c->views[slot].failed = true;   // never filled: a later job's sequence numbers must not make them look ready
      --c->up_active;
    }
    c->up_cv.notify_all();
  }
}

// Blocks until every queued upload has issued all its copies (caller memory is no longer read). Returns the first
// error an upload hit since the last call.
static int wait_uploads(b200m_ctx* c) {
  std::unique_lock<std::mutex> l(c->up_mu);
  c->up_cv.wait(l, [c] { return c->up_active == 0; });
  const int rc = c->up_rc;
  if (rc) { g_err = c->up_err; c->up_rc = 0; }
  return rc;
}

// Blocks until the view's copies, preparation kernel and flag copy are COMPLETE on the device; then its exactness flags are known.
static int ensure_view_ready(b200m_ctx* c, int slot) {
  ViewHost& v = c->views[slot];
  if (v.ready) return B200M_OK;
  {
    std::unique_lock<std::mutex> l(c->up_mu);
    c->up_cv.wait(l, [&] { return c->up_issued_seq >= v.seq || c->up_rc != 0 || c->up_active == 0 || v.failed; });
    if (c->up_rc) { g_err = c->up_err; return c->up_rc; }
    if (v.failed) return fail(B200M_ERR_CUDA, "the upload of view " + std::to_string(v.id) + " failed earlier; upload it again");
    if (c->up_issued_seq < v.seq) return fail(B200M_ERR_INTERNAL, "view was never uploaded");
  }
  CK(cudaEventSynchronize(c->view_ev[slot]));
  if (!v.flags_known) { v.flags = c->h_flags[slot]; v.flags_known = true; }
  v.ready = true;
  return B200M_OK;
}

int b200m_wait_uploads(b200m_ctx* c) {
  if (!c) return fail(B200M_ERR_ARG, "ctx is null");
  return wait_uploads(c);
}

int b200m_upload_views_async(b200m_ctx* c, int n_views, const uint32_t* view_ids, const void* const* descs, const int* counts, int dim, int dtype,
                             const float* const* xys) {
  if (!c) return fail(B200M_ERR_ARG, "ctx is null");
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  if (n_views < 0 || dim < 1 || dtype < 0 || dtype > 2 || (n_views > 0 && (!view_ids || !descs || !counts))) return fail(B200M_ERR_ARG, "bad view arguments");
  for (int i = 0; i < n_views; ++i) if (counts[i] < 0 || (counts[i] > 0 && !descs[i])) return fail(B200M_ERR_ARG, "bad view arguments");
  {
    // one view id may appear once per call: two entries would share one slot (and one set of device buffers) inside the job
    std::vector<uint32_t> ids(view_ids, view_ids + n_views);
    std::sort(ids.begin(), ids.end());
    if (std::adjacent_find(ids.begin(), ids.end()) != ids.end()) return fail(B200M_ERR_ARG, "a view id appears twice in one upload call");
  }
  CK(cudaSetDevice(c->device));
  const bool timing = getenv("B200M_TIMING") != nullptr;
  const auto t_reg0 = std::chrono::steady_clock::now();
  int rc = wait_uploads(c);              // one job at a time: slot table, staging ring and view table are not shared between jobs
  if (rc) return rc;
  UploadJob job;
  job.n_views = n_views; job.dim = dim; job.esz = dtype == DT_F32 ? 4 : 1;
  job.slots.resize(n_views); job.descs.assign(descs, descs + n_views); job.counts.assign(counts, counts + n_views);
  job.bad->assign(n_views, 0);
  bool waited = false;
  for (int i = 0; i < n_views; ++i) {
    int slot;
    auto it = c->slot_of.find(view_ids[i]);
    if (it == c->slot_of.end()) {
      if (!c->free_slots.empty()) {
        slot = c->free_slots.back(); c->free_slots.pop_back();
      } else {
        slot = (int)c->views.size();
        if ((rc = ensure_view_capacity(c, slot + 1))) return rc;
        c->views.emplace_back();
      }
      c->slot_of[view_ids[i]] = slot;
    } else {
      slot = it->second;
      if (!waited) {       // no finishing task / copy / preparation kernel may still reference a view that is replaced
        c->pool->wait(); CK(cudaStreamSynchronize(c->up_stream)); waited = true;
      }
      free_view_buffers(c, c->views[slot]);
    }
    job.slots[i] = slot;
    ViewHost& v = c->views[slot];
    v = ViewHost();
    v.id = view_ids[i]; v.m = counts[i]; v.dim = dim; v.dtype = dtype;
    v.seq = ++c->next_seq;
    const int n = counts[i];
    if (xys && xys[i] && n > 0) v.xy.assign(xys[i], xys[i] + 2 * (size_t)n);   // general position: decided on the device (pos_rank_kernel)
    v.flags_known = !(v.tc_capable() || !v.xy.empty());
    if (c->u8_staging && dtype == DT_F32 && dim == 128 && n > 0) {
      // probe: integer-valued fp32 descriptors (the SIFT extractor's output) are staged and stored as uchar; real-valued data
      // fails on its first rows.  A later surprise is caught by the checked conversion of every chunk (run_upload).
      uint8_t tmp[4 * 128];
      v.stored_u8 = f32_to_u8_checked((const float*)descs[i], tmp, (size_t)std::min(n, 4) * 128);
    }
    if (n > 0 && (rc = alloc_view_buffers(c, v))) return rc;
    if ((rc = c->view_ev[slot].create(cudaEventDisableTiming))) return rc;
  }
  // device view table (tensor maps are encoded on the host from the device addresses; valid whatever the upload state)
  for (int i = 0; i < n_views; ++i) {
    const int slot = job.slots[i];
    if ((rc = make_view_dev(c, c->views[slot], c->h_views[slot]))) return rc;
    CK(cudaMemcpyAsync(c->d_views + slot, c->h_views + slot, sizeof(ViewDev), cudaMemcpyHostToDevice, c->stream));
  }
  CK(cudaEventRecord(c->ev_alloc, c->stream));
  // general position is decided on the device (pos_rank_kernel); without the device finishing stage the host checks it eagerly
  // (2 sorts per view) on the pool, in parallel; a finishing task that needs one earlier computes it itself
  if (!c->device_finish)
    for (int i = 0; i < n_views; ++i) {
      const ViewHost* vp = &c->views[job.slots[i]];        // deque element: stable address; replaced / removed only after pool->wait()
      if (!vp->xy.empty()) c->pool->submit([vp] { (void)vp->generic_pos(); });
    }
  {
    std::lock_guard<std::mutex> l(c->up_mu);
    if (!c->up_thread.joinable()) c->up_thread = std::thread(uploader_main, c);
    c->up_jobs.push_back(std::move(job));
    ++c->up_active;
  }
  c->up_cv.notify_all();
  if (timing) fprintf(stderr, "[b200m] upload_views_async n=%d: registration (slots, allocations, tensor maps, table copies) %.2f ms\n", n_views,
                      std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_reg0).count());
  return B200M_OK;
}

int b200m_upload_views(b200m_ctx* c, int n_views, const uint32_t* view_ids, const void* const* descs, const int* counts, int dim, int dtype,
                       const float* const* xys) {
  if (!c) return fail(B200M_ERR_ARG, "ctx is null");
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  int rc = b200m_upload_views_async(c, n_views, view_ids, descs, counts, dim, dtype, xys);
  if (rc) return rc;
  return wait_uploads(c);
}

int b200m_upload_view(b200m_ctx* c, uint32_t view_id, const void* desc, int n, int dim, int dtype, const float* xy) {
  if (n > 0 && !desc) return fail(B200M_ERR_ARG, "bad view arguments");
  return b200m_upload_views(c, 1, &view_id, &desc, &n, dim, dtype, xy ? &xy : nullptr);
}

int b200m_clear_views(b200m_ctx* c) {
  if (!c) return fail(B200M_ERR_ARG, "ctx is null");
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  CK(cudaSetDevice(c->device));
  const auto t0 = std::chrono::steady_clock::now();
  int rc = wait_uploads(c);
  if (rc) return rc;
  c->pool->wait();
  CK(cudaStreamSynchronize(c->up_stream));
  const size_t nv = c->views.size();
  for (auto& v : c->views) free_view_buffers(c, v);
  c->views.clear(); c->slot_of.clear(); c->free_slots.clear();
  CK(cudaStreamSynchronize(c->stream));
  if (getenv("B200M_TIMING")) fprintf(stderr, "[b200m] clear_views n=%zu: %.2f ms\n", nv, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
  return B200M_OK;
}

int b200m_remove_view(b200m_ctx* c, uint32_t view_id) {
  if (!c) return fail(B200M_ERR_ARG, "ctx is null");
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  auto it = c->slot_of.find(view_id);
  if (it == c->slot_of.end()) return fail(B200M_ERR_ARG, "unknown view id");
  CK(cudaSetDevice(c->device));
  int rc = wait_uploads(c);
  if (rc) return rc;
  c->pool->wait();                       // no finishing task may still reference the view
  CK(cudaStreamSynchronize(c->up_stream));   // its copies / preparation kernel are done before the stream-ordered free on the search stream
  const int slot = it->second;
  free_view_buffers(c, c->views[slot]);  // stream-ordered: kernels already enqueued on the context's stream still see the buffers
  c->views[slot] = ViewHost();
  c->slot_of.erase(it);
  c->free_slots.push_back(slot);
  return B200M_OK;
}

// ---- Surface 2: pairs -------------------------------------------------------------------------------------------
// The search-kernel class of a directed pair, decided once, when its batch is enqueued (pair_class).  The tensor-core classes come
// first, in the order of their work items in the batch's table; the kernels launch in class order.
enum : int { K_FP16, K_U8, K_NG, K_REAL, K_EXACT_F32, K_EXACT_U8, K_HAMMING, K_GENERIC_F32, K_GENERIC_U8, K_SKIP, K_COUNT };
constexpr int K_TC_COUNT = K_REAL + 1;
// PairDev::mode of each class (the fp16, u8 and norm-GEMM classes: PM_TC_FUSED when their kernel runs the exactness pass itself)
static const uint32_t kClassMode[K_COUNT] = {PM_TC, PM_TC, PM_TC, PM_TC_REAL, PM_EXACT_F32, PM_EXACT_U8, PM_HAMMING, PM_GENERIC_F32,
                                              PM_GENERIC_U8, PM_SKIP};

struct Directed { int slot_i, slot_j; bool skip; };   // slot_i = database, slot_j = query; skip: nothing to search (plan_pairs)
struct Batch { size_t begin, end; };                  // a range of the processing order

// The state of one b200m_match_pairs call, shared by its steps.  The destructor runs on every exit path (CUDA error, failed upload
// ...): the finishing tasks already submitted write into `arena` and `dir_len` and signal `groups`, so they are waited for first.
struct MatchCall {
  MatchCall(b200m_ctx* c_, int stage_, int cross, float dist_ratio_)
      : c(c_), stage(stage_), do_cross(cross != 0 && stage_ == B200M_STAGE_FULL), dev_fin(c_->device_finish && stage_ == B200M_STAGE_FULL),
        step(do_cross ? 2 : 1), tc_ctas_per_item((c_->tc_variant == 2 || c_->tc_variant == 4) ? 2 : 1), dist_ratio(dist_ratio_),
        ratio_sq(dist_ratio_ * dist_ratio_) {}   // Square(f_dist_ratio) in float, RegionsMatcher.hpp:150 / numeric.hpp:130
  ~MatchCall() { for (auto& g : groups) g->wait(); for (auto& b : arena) c->recycler->give(b); }

  b200m_ctx* c;
  int stage; bool do_cross, dev_fin;
  size_t step;                                  // directed pairs per pair: 2 when cross matching
  int tc_ctas_per_item;                         // CTAs per work item of the fp16 kernel
  float dist_ratio, ratio_sq;
  std::vector<std::pair<uint32_t, uint32_t>> fwd;   // the PairSet
  std::vector<Directed> dir;                    // fwd[k]: dir[k * step] = (i, j), then dir[k * step + 1] = (j, i) when cross matching
  std::vector<uint32_t> seqv;                   // directed-pair indices in processing order
  bool pending = false;                         // views still arriving: arrival order and short first batches
  std::vector<Batch> batches;
  std::vector<uint8_t> cls;                     // per directed pair: its class (K_*), set when its batch is enqueued
  // the batch being enqueued, per class: pairs, database rows, work items (tensor-core classes, from item0 in the table) or query
  // blocks of its largest pair (the grid of the exact, Hamming and generic kernels), and whether its kernel runs the exactness pass
  struct Tally { int n; long rows; int items, item0, qblk; bool fused; } tally[K_COUNT];
  // finishing output: one slot per directed pair in a flat arena per batch (capacity = its record count), filled by pool tasks
  std::vector<Recycler::Block> arena;
  std::vector<b200m_match*> dir_ptr; std::vector<int> dir_len;
  std::vector<std::unique_ptr<TaskGroup>> groups;   // per batch: its finishing tasks
  size_t tev_used = 0; std::vector<std::pair<cudaEvent_t, cudaEvent_t>> kernel_events;
  int launches = 0, tc_pairs = 0, u8_pairs = 0, ng_pairs = 0, real_pairs = 0;
  int64_t total_records = 0, fallback_rows = 0;
};

static double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// PairSet semantics (types.hpp:23): unique, lexicographically ordered; then the directed pairs of each pair and the argument errors.
static int plan_pairs(MatchCall& s, const uint32_t* pairs, int n_pairs) {
  b200m_ctx* c = s.c;
  s.fwd.resize((size_t)n_pairs);
  for (int k = 0; k < n_pairs; ++k) s.fwd[k] = {pairs[2 * k], pairs[2 * k + 1]};
  if (!std::is_sorted(s.fwd.begin(), s.fwd.end())) std::sort(s.fwd.begin(), s.fwd.end());
  s.fwd.erase(std::unique(s.fwd.begin(), s.fwd.end()), s.fwd.end());
  s.dir.reserve(s.fwd.size() * s.step);
  for (const auto& f : s.fwd) {
    auto si = c->slot_of.find(f.first), sj = c->slot_of.find(f.second);
    if (si == c->slot_of.end() || sj == c->slot_of.end())
      return fail(B200M_ERR_ARG, "pair references a view that was never uploaded (RegionsPerView::getRegions would throw std::out_of_range)");
    for (size_t rev = 0; rev < s.step; ++rev) {
      const int a = rev ? sj->second : si->second, b = rev ? si->second : sj->second;   // a = database, b = query
      const ViewHost& vi = c->views[a]; const ViewHost& vj = c->views[b];
      const bool skip = vi.m == 0 || vj.m == 0 || vi.dtype != vj.dtype || vi.dim != vj.dim     // generic.cpp:59-63,74-78
                        || vi.m < 2;                                                          // NN=2 > rows: bruteForce.hpp:105
      if (!skip && vi.dtype == DT_BIN && vi.dim != 64) return fail(B200M_ERR_UNSUPPORTED, "binary descriptors must be 64 bytes (AKAZE_BinaryRegions)");
      if (s.stage == B200M_STAGE_FULL && !skip && (vi.xy.empty() || vj.xy.empty()))
        return fail(B200M_ERR_ARG, "B200M_STAGE_FULL needs feature positions for every matched view");
      s.dir.push_back(Directed{a, b, skip});
    }
  }
  return B200M_OK;
}

// Processing order: PairSet order, or - while uploads are in flight - the order in which the pairs' views arrive.  Arrival order (with
// short first batches) only while copies are really in flight, not for views that are merely not yet marked ready after a completed
// upload.
static void order_pairs(MatchCall& s) {
  b200m_ctx* c = s.c;
  std::vector<uint32_t> ord(s.fwd.size());
  for (size_t k = 0; k < s.fwd.size(); ++k) ord[k] = (uint32_t)k;
  bool uploading;
  { std::lock_guard<std::mutex> l(c->up_mu); uploading = c->up_active > 0; }
  if (uploading) for (const Directed& d : s.dir) if (!d.skip) s.pending |= !c->views[d.slot_i].ready || !c->views[d.slot_j].ready;
  if (s.pending) {
    std::vector<uint64_t> key(s.fwd.size());
    for (size_t k = 0; k < s.fwd.size(); ++k) key[k] = std::max(c->views[s.dir[k * s.step].slot_i].seq, c->views[s.dir[k * s.step].slot_j].seq);
    std::stable_sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
  }
  s.seqv.reserve(s.dir.size());
  for (uint32_t k : ord) for (size_t u = 0; u < s.step; ++u) s.seqv.push_back((uint32_t)(k * s.step + u));
}

// Batches over the processing order, each within PAIR_CAP, CAND_CAP, ITEM_CAP and SLOT_CAP; both directions of a pair go into the
// same batch.  While views are still arriving the first batches are short (B200M_FIRST_BATCH pairs, doubled per batch) so the GPU
// starts early.
static int split_batches(MatchCall& s) {
  b200m_ctx* c = s.c;
  size_t b0 = 0; long cand = 0, items = 0, slots = 0;
  size_t pair_cap = s.pending ? (size_t)c->first_batch_pairs : (size_t)PAIR_CAP;
  for (size_t k = 0; k < s.seqv.size(); k += s.step) {
    long need_c = 0, need_i = 0, need_s = 0;
    for (size_t u = k; u < k + s.step; ++u) {
      const int mj = c->views[s.dir[s.seqv[u]].slot_j].m, mi = c->views[s.dir[s.seqv[u]].slot_i].m;
      if (mj > CAND_CAP || mi > SLOT_CAP / 2) return fail(B200M_ERR_UNSUPPORTED, "view too large for one batch");
      need_c += mj; need_i += (mj + tc::BM - 1) / tc::BM; need_s += mi;
    }
    if (k > b0 && (cand + need_c > CAND_CAP || items + need_i > ITEM_CAP || slots + need_s > SLOT_CAP || k - b0 + s.step > pair_cap)) {
      s.batches.push_back({b0, k}); b0 = k; cand = 0; items = 0; slots = 0;
      pair_cap = std::min<size_t>(PAIR_CAP, pair_cap * 2);
    }
    cand += need_c; items += need_i; slots += need_s;
  }
  if (s.seqv.size() > b0) s.batches.push_back({b0, s.seqv.size()});
  return B200M_OK;
}

// The class of a directed pair, from both views' exactness flags: they are known once the views are ready on the device.
static int pair_class(const b200m_ctx* c, const Directed& d) {
  if (d.skip) return K_SKIP;
  const ViewHost& vi = c->views[d.slot_i]; const ViewHost& vj = c->views[d.slot_j];
  if (vi.dtype == DT_BIN) return K_HAMMING;
  if (vi.dim != 128) return vi.dtype == DT_F32 ? K_GENERIC_F32 : K_GENERIC_U8;   // AKAZE float (64), LIOP (144), ...: generic exact path
  if (!c->force_exact && vi.tc_ok() && vj.tc_ok()) {
    // integer-valued pairs whose views are both stored as uchar run the u8 kernel (8-bit tensor cores, exact int32 distances) under
    // the default variant; the other tensor-core pairs run the fp16 kernel
    if (c->tc_variant != 4 || vi.store_dtype() != DT_U8 || vj.store_dtype() != DT_U8) return K_FP16;
    // ... and of those, the pairs whose query view has no component above 127 and whose database view's norms fit the limbs run the
    // u8 norm-GEMM kernel (the norms folded into the 8-bit GEMM)
    return c->u8_norm_gemm && vi.ng_db_ok() && vj.ng_query_ok() ? K_NG : K_U8;
  }
  // real-valued fp32: tensor-core filter + exact re-scoring
  if (!c->force_exact && c->real_tc && c->tc_variant == 4 && vi.real_ok() && vj.real_ok()) return K_REAL;
  return vi.dtype == DT_F32 ? K_EXACT_F32 : K_EXACT_U8;
}

// The search kernels of one batch on the search stream, in class order: each tensor-core kernel over its range of the work-item
// table, the real-valued path's re-scoring and fallbacks, then the exact, Hamming and generic kernels, each over all pairs of the
// batch (a kernel searches the pairs of its mode).
static void launch_search(MatchCall& s, const BatchBuf& bb, int np) {
  b200m_ctx* c = s.c;
  const MatchCall::Tally* t = s.tally;
  const cudaStream_t st = c->stream;
  const float r2 = s.ratio_sq;
  // the debug trace (one kernel's CTA 0) shows the norm-GEMM kernel when the batch has pairs on it, else the u8 kernel when it has u8
  // pairs, else the fp16 kernel
  const int traced = t[K_NG].n ? K_NG : t[K_U8].n ? K_U8 : K_FP16;
  auto trace = [&](int k) { return k == traced ? static_cast<long long*>(c->d_trace) : nullptr; };
  // one CTA per SM, whole work items per CTA group
  auto grid = [&](int k, int ctas) { return ctas * std::min(t[k].items, c->num_sms / ctas); };
  if (t[K_FP16].items) {
    const bool aug = c->tc_variant == 4;
    const int ctas = s.tc_ctas_per_item;
    auto* kernel = aug ? tc::l2_top2_tc_kernel<true> : tc::l2_top2_tc_kernel<false>;
    kernel<<<grid(K_FP16, ctas), tc::block_threads<tc::MODE_MATCH>(), aug ? tc::Lay<true>::SMEM_BYTES : tc::Lay<false>::SMEM_BYTES, st>>>(
        c->d_views, bb.d_pairs, bb.d_items + t[K_FP16].item0, t[K_FP16].items, ctas, bb.d_cands, bb.d_count, r2, trace(K_FP16), c->d_err,
        (int)t[K_FP16].fused, nullptr, FbSink{});
    ++s.launches;
  }
  if (t[K_U8].items) {
    tc::l2_top2_tc_u8_kernel<<<grid(K_U8, 2), tc::block_threads<tc::MODE_MATCH>(), tc::Lay<false, false, true>::SMEM_BYTES, st>>>(
        c->d_views, bb.d_pairs, bb.d_items + t[K_U8].item0, t[K_U8].items, 2, bb.d_cands, bb.d_count, r2, trace(K_U8), c->d_err,
        (int)t[K_U8].fused, nullptr, FbSink{});
    ++s.launches;
  }
  if (t[K_NG].items) {
    tc::l2_top2_tc_u8ng_kernel<<<grid(K_NG, 2), tc::block_threads<tc::MODE_MATCH>(), tc::Lay<false, false, true, true>::SMEM_BYTES, st>>>(
        c->d_views, bb.d_pairs, bb.d_items + t[K_NG].item0, t[K_NG].items, 2, bb.d_cands, bb.d_count, r2, trace(K_NG), c->d_err,
        (int)t[K_NG].fused, nullptr, FbSink{});
    ++s.launches;
  }
  if (t[K_REAL].items) {
    // real-valued pairs: filter kernel (re-scoring in-kernel when the items are long enough), stand-alone re-scoring otherwise, then the
    // exact search of the few queries the error bound could not decide; after that their candidates are final like everyone else's
    const FbSink fbs{bb.d_fb_pair, bb.d_fb_pair_cnt, bb.d_fb, bb.d_fb_count, (int)CAND_CAP, bb.d_fb_count + 1};
    tc::l2_top2_tc_kernel<true, tc::MODE_REAL><<<grid(K_REAL, 2), tc::block_threads<tc::MODE_REAL>(), tc::Lay<true, true>::SMEM_BYTES, st>>>(
        c->d_views, bb.d_pairs, bb.d_items + t[K_REAL].item0, t[K_REAL].items, 2, bb.d_cands, bb.d_count, r2, nullptr, c->d_err,
        (int)t[K_REAL].fused, bb.d_candx, fbs);
    ++s.launches;
    if (!t[K_REAL].fused) {
      rescore_real_kernel<<<dim3(np, 4), VERIFY_WARPS_REAL * 32, 0, st>>>(c->d_views, bb.d_pairs, bb.d_cands, bb.d_candx, bb.d_count, r2, c->d_err, fbs);
      ++s.launches;
    }
    exact_rows_pairs_kernel<<<dim3(np, FB_PER_PAIR / XP_MAXQ), XP_THREADS, XP_SMEM, st>>>(c->d_views, bb.d_pairs, bb.d_fb_pair, bb.d_fb_pair_cnt, bb.d_cands, bb.d_count, r2);
    exact_rows_kernel<<<c->num_sms, XR_THREADS, 0, st>>>(c->d_views, bb.d_pairs, bb.d_fb, bb.d_fb_count, (int)CAND_CAP, bb.d_cands, bb.d_count, r2);   // overflow list: normally empty
    s.launches += 2;
  }
  // the two exact kernels share one grid, as do the two generic ones
  const int qblk_exact = std::max(t[K_EXACT_F32].qblk, t[K_EXACT_U8].qblk), qblk_gen = std::max(t[K_GENERIC_F32].qblk, t[K_GENERIC_U8].qblk);
  if (t[K_EXACT_F32].n) {
    exact_top2_kernel<float, false><<<dim3(qblk_exact, np), 256, EX_SMEM, st>>>(c->d_views, bb.d_pairs, PM_EXACT_F32, bb.d_cands, bb.d_count, r2, nullptr, nullptr);
    ++s.launches;
  }
  if (t[K_EXACT_U8].n) {
    exact_top2_kernel<uint8_t, false><<<dim3(qblk_exact, np), 256, EX_SMEM, st>>>(c->d_views, bb.d_pairs, PM_EXACT_U8, bb.d_cands, bb.d_count, r2, nullptr, nullptr);
    ++s.launches;
  }
  if (t[K_HAMMING].n) {
    hamming_top2_kernel<false><<<dim3(t[K_HAMMING].qblk, np), HM_TQ, 0, st>>>(c->d_views, bb.d_pairs, bb.d_cands, bb.d_count, s.dist_ratio, nullptr, nullptr);
    ++s.launches;
  }
  if (t[K_GENERIC_F32].n) {
    generic_top2_pairs_kernel<float><<<dim3(qblk_gen, np), 128, 0, st>>>(c->d_views, bb.d_pairs, PM_GENERIC_F32, bb.d_cands, bb.d_count, r2);
    ++s.launches;
  }
  if (t[K_GENERIC_U8].n) {
    generic_top2_pairs_kernel<uint8_t><<<dim3(qblk_gen, np), 128, 0, st>>>(c->d_views, bb.d_pairs, PM_GENERIC_U8, bb.d_cands, bb.d_count, r2);
    ++s.launches;
  }
}

// Batch bi: the class of each pair, the per-class tally, the pair and work-item tables, the search, packing and finishing kernels and
// the meta read-back.  Three streams so that consecutive batches' search kernels run back to back: the tables of this batch travel on
// `tab_stream` (issued while the previous batch is still searching), the packing / finishing kernels and the meta read-back of this
// batch run on `pack_stream` beside the next batch's search kernel.  Buffer set (bi & 1) is free: the host has seen ev_meta of batch
// bi-2.
static int enqueue_batch(MatchCall& s, size_t bi) {
  b200m_ctx* c = s.c;
  const Batch& B = s.batches[bi];
  BatchBuf& bb = c->buf[bi & 1];
  const int np = (int)(B.end - B.begin);
  // queries per work item (tensor-core classes) or per block of the grid (the others)
  const int qrows[K_COUNT] = {s.tc_ctas_per_item * tc::BM, 2 * tc::BM, 2 * tc::BM, 2 * tc::BM, EX_TQ, EX_TQ, HM_TQ, 4, 4, 1};
  for (MatchCall::Tally& t : s.tally) t = MatchCall::Tally{};
  for (int p = 0; p < np; ++p) {
    const uint32_t di = s.seqv[B.begin + p];
    const Directed& d = s.dir[di];
    int rc;
    if (!d.skip && ((rc = ensure_view_ready(c, d.slot_i)) || (rc = ensure_view_ready(c, d.slot_j)))) return rc;
    const int k = s.cls[di] = (uint8_t)pair_class(c, d);
    const int blocks = (c->views[d.slot_j].m + qrows[k] - 1) / qrows[k];
    MatchCall::Tally& t = s.tally[k];
    ++t.n; t.rows += c->views[d.slot_i].m; t.items += blocks; t.qblk = std::max(t.qblk, blocks);
  }
  // In-kernel exactness pass only when a work item lasts long enough (>= 24 database tiles on average) for two warps to re-score the
  // previous item's candidates behind it; shorter images use the stand-alone exactness kernel.
  int n_items = 0, next[K_TC_COUNT];
  for (int k = 0; k < K_TC_COUNT; ++k) {
    MatchCall::Tally& t = s.tally[k];
    t.fused = t.n > 0 && t.rows / t.n >= (k == K_REAL ? c->real_fused_rows : 6144) && (k != K_FP16 || c->tc_variant >= 2);
    t.item0 = next[k] = n_items;
    n_items += t.items;
  }
  uint32_t cbase = 0, sbase = 0;
  for (int p = 0; p < np; ++p) {
    const uint32_t di = s.seqv[B.begin + p];
    const Directed& d = s.dir[di];
    const int k = s.cls[di];
    const ViewHost& vi = c->views[d.slot_i]; const ViewHost& vj = c->views[d.slot_j];
    const uint32_t mode = k < K_REAL && s.tally[k].fused ? (uint32_t)PM_TC_FUSED : kClassMode[k];
    bb.h_pairs[p] = PairDev{(uint32_t)d.slot_i, (uint32_t)d.slot_j, (uint32_t)vi.m, (uint32_t)vj.m, cbase, mode, sbase, k == K_U8 || k == K_NG ? 1u : 0u};
    cbase += (uint32_t)vj.m; sbase += (uint32_t)vi.m;
    if (k < K_TC_COUNT) for (int qt = 0; qt < (vj.m + qrows[k] - 1) / qrows[k]; ++qt) bb.h_items[next[k]++] = WorkItem{(uint32_t)p, (uint32_t)qt};
  }
  s.tc_pairs += s.tally[K_FP16].n + s.tally[K_U8].n + s.tally[K_NG].n;
  s.u8_pairs += s.tally[K_U8].n + s.tally[K_NG].n;
  s.ng_pairs += s.tally[K_NG].n;
  s.real_pairs += s.tally[K_REAL].n;

  cudaStream_t ts = c->pipe_streams ? c->tab_stream : c->stream, ps = c->pipe_streams ? c->pack_stream : c->stream;
  CK(cudaMemcpyAsync(bb.d_pairs, bb.h_pairs, sizeof(PairDev) * np, cudaMemcpyHostToDevice, ts));
  if (n_items) CK(cudaMemcpyAsync(bb.d_items, bb.h_items, sizeof(WorkItem) * n_items, cudaMemcpyHostToDevice, ts));
  CK(cudaMemsetAsync(bb.d_count, 0, sizeof(int) * np, ts));
  CK(cudaMemsetAsync(bb.d_fb_count, 0, 2 * sizeof(int), ts));
  if (s.tally[K_REAL].items) CK(cudaMemsetAsync(bb.d_fb_pair_cnt, 0, sizeof(int) * np, ts));
  if (c->pipe_streams) { CK(cudaEventRecord(bb.ev_tab, ts)); CK(cudaStreamWaitEvent(c->stream, bb.ev_tab, 0)); }
  cudaEvent_t k0 = timing_event(c, s.tev_used), k1 = timing_event(c, s.tev_used);
  CK(cudaEventRecord(k0, c->stream));
  launch_search(s, bb, np);
  CK(cudaEventRecord(k1, c->stream));
  if (c->pipe_streams) CK(cudaStreamWaitEvent(ps, k1, 0));
  s.kernel_events.push_back({k0, k1});
  scan_counts_kernel<<<1, 256, 0, ps>>>(bb.d_count, np, bb.d_off);
  verify_pack_kernel<<<dim3(np, VERIFY_BLOCKS_PER_PAIR), VERIFY_WARPS * 32, 0, ps>>>(c->d_views, bb.d_pairs, bb.d_cands, bb.d_count, bb.d_off, bb.d_out, s.ratio_sq, c->d_err);
  s.launches += 2;
  if (s.dev_fin) {
    finish_pairs_kernel<<<np, FIN_THREADS, 0, ps>>>(c->d_views, bb.d_pairs, c->d_flags, bb.d_out, bb.d_count, bb.d_off, bb.d_scratch, bb.d_fin, bb.d_fin_count);
    ++s.launches;
    CK(cudaMemcpyAsync(bb.meta_fin_counts(), bb.d_fin_count, sizeof(int) * np, cudaMemcpyDeviceToHost, ps));
  }
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(bb.meta_fallback_rows(), bb.d_fb_count + 1, sizeof(int), cudaMemcpyDeviceToHost, ps));
  CK(cudaMemcpyAsync(bb.meta_counts(), bb.d_count, sizeof(int) * np, cudaMemcpyDeviceToHost, ps));
  CK(cudaMemcpyAsync(bb.meta_offsets(), bb.d_off, sizeof(int) * (np + 1), cudaMemcpyDeviceToHost, ps));
  CK(cudaEventRecord(bb.ev_meta, ps));
  return B200M_OK;
}

// RAW / FULL: batch bi's records, copied to pinned memory once its meta block is in, and its finishing tasks.  The tasks run behind
// the GPU: they only have to be done before batch bi+2's records are copied into the same pinned buffer.  They take the per-pair
// counts and offsets out of the meta block here, because enqueue_batch(bi+2) overwrites it.
static int finish_batch(MatchCall& s, size_t bi) {
  b200m_ctx* c = s.c;
  const Batch& B = s.batches[bi];
  const BatchBuf& bb = c->buf[bi & 1];
  const int np = (int)(B.end - B.begin);
  const int total = bb.meta_offsets()[np];
  if (bi >= 2) s.groups[bi - 2]->wait();       // the tasks of batch bi-2 read this pinned record buffer
  if (total > 0) {
    CK(cudaStreamWaitEvent(c->copy_stream, bb.ev_meta, 0));
    CK(cudaMemcpyAsync(bb.h_out, s.dev_fin ? (const void*)bb.d_fin : (const void*)bb.d_out, sizeof(Rec) * (size_t)total, cudaMemcpyDeviceToHost, c->copy_stream));
    CK(cudaEventRecord(bb.ev_copy, c->copy_stream));
    CK(cudaEventSynchronize(bb.ev_copy));
  }
  if (bi + 1 == s.batches.size()) {
    // end of the device work of this call = the last match list has landed in pinned host memory (SURVEY 8d)
    CK(cudaStreamWaitEvent(c->copy_stream, bb.ev_meta, 0));
    CK(cudaEventRecord(c->ev_end, c->copy_stream));
  }
  s.arena[bi] = c->recycler->take((size_t)std::max(total, 1));
  TaskGroup* grp = s.groups[bi].get();
  // one pool task per ~4096 records (or 64 pairs): for small images the task hand-off would otherwise cost more than the work
  // cnt >= 0: raw records, finished here (finish_directed); done >= 0: `done` final matches from the device finishing stage, copied
  struct Job { const Rec* recs; int cnt; int done; b200m_match* dst; int* len; const ViewHost* vi; const ViewHost* vj; bool ham; };
  auto jobs = std::make_shared<std::vector<Job>>();
  long job_records = 0;
  const bool full = s.stage == B200M_STAGE_FULL;
  auto flush = [&] {
    if (jobs->empty()) return;
    grp->add(1);
    std::shared_ptr<std::vector<Job>> mine = std::move(jobs);
    c->pool->submit([mine, grp, full] {
      for (const Job& j : *mine) {
        if (j.done >= 0) { std::memcpy(j.dst, j.recs, sizeof(b200m_match) * (size_t)j.done); *j.len = j.done; }
        else *j.len = finish_directed(j.recs, j.cnt, j.ham, full, *j.vi, *j.vj, j.dst);
      }
      grp->done();
    });
    jobs = std::make_shared<std::vector<Job>>();
    job_records = 0;
  };
  for (int p = 0; p < np; ++p) {
    const size_t di = s.seqv[B.begin + p];
    const Directed& d = s.dir[di];
    s.dir_ptr[di] = s.arena[bi].p + bb.meta_offsets()[p];
    int cnt = bb.meta_counts()[p], done = -1;
    if (d.skip || cnt == 0) continue;
    if (s.dev_fin) {                                 // >= 0: final matches; < 0: -(records + 1) left for the host (view not in general position)
      const int f = bb.meta_fin_counts()[p];
      if (f >= 0) done = f; else cnt = -(f + 1);
      if (done == 0) continue;
    }
    jobs->push_back(Job{bb.h_out + bb.meta_offsets()[p], cnt, done, s.dir_ptr[di], &s.dir_len[di], &c->views[d.slot_i], &c->views[d.slot_j],
                        s.cls[di] == K_HAMMING});
    job_records += cnt;
    if (job_records >= 4096 || jobs->size() >= 64) flush();
  }
  flush();
  return B200M_OK;
}

// Every stage runs the same pipeline: batch j is enqueued while the host waits for the meta block of batch j-1 (which also frees
// buffer set j+1 & 1 for the next enqueue), then RAW / FULL copy batch j-1's records and submit its finishing tasks.  The device work
// of the call ends with the last batch's kernels (DEVICE) or with its records in pinned host memory (RAW / FULL, finish_batch).
static int batch_loop(MatchCall& s, bool timing) {
  b200m_ctx* c = s.c;
  const double t0 = now_ms();
  const size_t nb = s.batches.size();
  CK(cudaEventRecord(c->ev_start, c->stream));
  if (nb == 0) CK(cudaEventRecord(c->ev_end, c->stream));
  for (size_t j = 0; j <= nb; ++j) {
    int rc;
    if (j < nb) {
      if ((rc = enqueue_batch(s, j))) return rc;
      if (j + 1 == nb && s.stage == B200M_STAGE_DEVICE) CK(cudaEventRecord(c->ev_end, c->stream));
    }
    if (j == 0) continue;
    const size_t bi = j - 1;
    const BatchBuf& bb = c->buf[bi & 1];
    CK(cudaEventSynchronize(bb.ev_meta));
    s.total_records += bb.meta_offsets()[s.batches[bi].end - s.batches[bi].begin];
    s.fallback_rows += *bb.meta_fallback_rows();
    if (s.stage != B200M_STAGE_DEVICE && (rc = finish_batch(s, bi))) return rc;
  }
  const double t_loop = now_ms();
  for (auto& g : s.groups) g->wait();
  if (timing) fprintf(stderr, "[b200m] match_pairs: batch loop %.2f ms, last finishing groups +%.2f ms\n", t_loop - t0, now_ms() - t_loop);
  return B200M_OK;
}

// Cross matching: keep m iff (m.j, m.i) is in the reverse list (ImageCollectionMatcher_generic.cpp:92-109); filtered in place, in
// parallel.
static void cross_filter(MatchCall& s) {
  TaskGroup g; g.add((int)s.fwd.size());
  for (size_t k = 0; k < s.fwd.size(); ++k) {
    b200m_match* f = s.dir_ptr[k * s.step]; int* nf = &s.dir_len[k * s.step];
    const b200m_match* r = s.dir_ptr[k * s.step + 1]; const int nr = s.dir_len[k * s.step + 1];
    TaskGroup* gp = &g;
    s.c->pool->submit([=] {
      std::vector<std::pair<uint32_t, uint32_t>> rv; rv.reserve(nr);
      for (int e = 0; e < nr; ++e) rv.push_back({r[e].i, r[e].j});
      std::sort(rv.begin(), rv.end());
      int w = 0;
      for (int e = 0; e < *nf; ++e)
        if (std::binary_search(rv.begin(), rv.end(), std::make_pair(f[e].j, f[e].i))) f[w++] = f[e];
      *nf = w;
      gp->done();
    });
  }
  g.wait();
}

// The result: offsets first, then the per-pair copies into one contiguous block in parallel on the pool.
static b200m_result* assemble_result(MatchCall& s) {
  b200m_ctx* c = s.c;
  const size_t n = s.fwd.size(), step = s.step;
  std::unique_ptr<b200m_result> res(new b200m_result());
  res->pair_ids.reserve(2 * n);
  res->offsets.assign(n + 1, 0);
  for (size_t k = 0; k < n; ++k) {
    res->pair_ids.push_back(s.fwd[k].first); res->pair_ids.push_back(s.fwd[k].second);
    res->offsets[k + 1] = res->offsets[k] + (s.stage != B200M_STAGE_DEVICE ? s.dir_len[k * step] : 0);
  }
  const size_t total_matches = (size_t)res->offsets[n];
  res->recycler = c->recycler;
  res->matches = c->recycler->take(total_matches);
  if (total_matches) {
    const size_t CHUNK_PAIRS = 64;
    TaskGroup g; g.add((int)((n + CHUNK_PAIRS - 1) / CHUNK_PAIRS));
    for (size_t k0 = 0; k0 < n; k0 += CHUNK_PAIRS) {
      const size_t k1 = std::min(n, k0 + CHUNK_PAIRS);
      b200m_match* base = res->matches.p; const int64_t* offs = res->offsets.data();
      b200m_match* const* dp = s.dir_ptr.data(); const int* dl = s.dir_len.data(); TaskGroup* gp = &g;
      c->pool->submit([=] {
        for (size_t k = k0; k < k1; ++k) if (dl[k * step] > 0) std::memcpy(base + offs[k], dp[k * step], sizeof(b200m_match) * (size_t)dl[k * step]);
        gp->done();
      });
    }
    g.wait();
  }
  return res.release();
}

static int match_pairs_impl(b200m_ctx* c, const uint32_t* pairs, int n_pairs, float dist_ratio, int cross, int stage, b200m_result** out) {
  if (!c || !out || n_pairs < 0 || (n_pairs > 0 && !pairs) || stage < 0 || stage > 2) return fail(B200M_ERR_ARG, "bad arguments");
  *out = nullptr;
  CK(cudaSetDevice(c->device));
  int rc = ensure_batch_buffers(c);
  if (rc) return rc;
  const bool timing = getenv("B200M_TIMING") != nullptr;
  const double t_begin = now_ms();
  MatchCall s(c, stage, cross, dist_ratio);
  if ((rc = plan_pairs(s, pairs, n_pairs))) return rc;
  order_pairs(s);
  if ((rc = split_batches(s))) return rc;
  s.cls.assign(s.dir.size(), K_SKIP);
  s.dir_ptr.assign(s.dir.size(), nullptr);
  s.dir_len.assign(s.dir.size(), 0);
  s.arena.resize(s.batches.size());
  for (size_t b = 0; b < s.batches.size(); ++b) s.groups.emplace_back(new TaskGroup());

  const double t_setup = now_ms();
  if ((rc = batch_loop(s, timing))) return rc;
  const double t_gpu_done = now_ms();
  CK(cudaStreamSynchronize(c->stream));
  CK(cudaStreamSynchronize(c->pack_stream));
  float ms = 0.f;
  CK(cudaEventSynchronize(c->ev_end));
  CK(cudaEventElapsedTime(&ms, c->ev_start, c->ev_end));
  double sk = 0;
  const auto& kev = s.kernel_events;
  for (auto& e : kev) { float t = 0.f; CK(cudaEventElapsedTime(&t, e.first, e.second)); sk += t; }
  if (timing && !kev.empty()) {
    // device timeline of the call: search kernels back to back?  gap = end of one batch's search kernels -> start of the next one's
    // (packing / finishing kernels, meta copies, the next batch's pair-table copies, and any wait for the host)
    float lead = 0.f, gaps = 0.f, gmax = 0.f, tail = 0.f;
    CK(cudaEventElapsedTime(&lead, c->ev_start, kev.front().first));
    for (size_t k = 0; k + 1 < kev.size(); ++k) { float t = 0.f; CK(cudaEventElapsedTime(&t, kev[k].second, kev[k + 1].first)); gaps += t; gmax = std::max(gmax, t); }
    CK(cudaEventElapsedTime(&tail, kev.back().second, c->ev_end));
    fprintf(stderr, "[b200m] device timeline: %zu batches, search kernels %.2f ms, lead-in %.2f, gaps between batches %.2f (max %.2f), tail after the last search kernel %.2f ms\n",
            kev.size(), sk, lead, gaps, gmax, tail);
  }
  unsigned errs = 0;
  CK(cudaMemcpy(&errs, c->d_err, sizeof(unsigned), cudaMemcpyDeviceToHost));
  c->err_total = errs;

  if (s.do_cross) cross_filter(s);
  *out = assemble_result(s);
  if (timing) fprintf(stderr, "[b200m] match_pairs n=%d stage=%d: setup %.2f ms, batches %.2f ms (gpu %.2f), tail (cross+assemble) %.2f ms, total %.2f ms\n",
                      n_pairs, stage, t_setup - t_begin, t_gpu_done - t_setup, ms, now_ms() - t_gpu_done, now_ms() - t_begin);
  c->last = LastCall{ms, sk, s.launches, s.tc_pairs, s.real_pairs, s.u8_pairs, s.total_records, s.fallback_rows, (int)s.batches.size(), s.ng_pairs};
  return B200M_OK;
}

int b200m_match_pairs(b200m_ctx* c, const uint32_t* pairs, int n_pairs, float dist_ratio, int cross, int stage, b200m_result** out) {
  if (!c) return fail(B200M_ERR_ARG, "ctx is null");
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  const int rc = match_pairs_impl(c, pairs, n_pairs, dist_ratio, cross, stage, out);
  if (c) {
    // asynchronous uploads read caller memory until their copies are issued: that is guaranteed on return, error or not
    const std::string err = g_err;
    const int rcu = wait_uploads(c);
    if (rc) { g_err = err; return rc; }
    if (rcu) { if (out && *out) { b200m_result_free(*out); *out = nullptr; } return rcu; }
  }
  return rc;
}

int b200m_result_num_pairs(const b200m_result* r) { return r ? (int)(r->offsets.size() - 1) : 0; }
int b200m_result_get(const b200m_result* r, const uint32_t** pair_ids, const int64_t** offsets, const b200m_match** matches) {
  if (!r) return fail(B200M_ERR_ARG, "result is null");
  if (pair_ids) *pair_ids = r->pair_ids.data();
  if (offsets) *offsets = r->offsets.data();
  if (matches) *matches = r->matches.p;
  return B200M_OK;
}
void b200m_result_free(b200m_result* r) { delete r; }

static LastCall last_call(const b200m_ctx* c) {       // a concurrent call rewrites the record
  if (!c) return LastCall{};
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  return c->last;
}
double b200m_last_gpu_ms(const b200m_ctx* c) { return last_call(c).gpu_ms; }
double b200m_last_search_kernel_ms(const b200m_ctx* c) { return last_call(c).search_ms; }
int b200m_last_launches(const b200m_ctx* c) { return last_call(c).launches; }
int b200m_last_tc_pairs(const b200m_ctx* c) { return last_call(c).tc_pairs; }
unsigned b200m_exactness_errors(const b200m_ctx* c) { return c ? c->err_total : 0; }
int64_t b200m_last_records(const b200m_ctx* c) { return last_call(c).records; }
int b200m_last_real_tc_pairs(const b200m_ctx* c) { return last_call(c).real_pairs; }
int b200m_last_u8_tc_pairs(const b200m_ctx* c) { return last_call(c).u8_pairs; }
int b200m_last_u8_norm_gemm_pairs(const b200m_ctx* c) { return last_call(c).u8_norm_gemm_pairs; }
int64_t b200m_last_fallback_rows(const b200m_ctx* c) { return last_call(c).fallback_rows; }
int b200m_last_batches(const b200m_ctx* c) { return last_call(c).batches; }

// ---- guided matching (after the path: GeometricFilterMatrix_F_AC.hpp:363-390 -> matching/guidedMatching.hpp:206-268) ----------------
int b200m_guided_match(b200m_ctx* c, uint32_t view_left, uint32_t view_right, const double* F, double errorTh, double distRatio, b200m_result** out) {
  return b200m_guided_match_model(c, view_left, view_right, B200M_MODEL_FUNDAMENTAL, F, errorTh, distRatio, out);
}

int b200m_guided_match_model(b200m_ctx* c, uint32_t view_left, uint32_t view_right, int model, const double* F, double errorTh, double distRatio,
                             b200m_result** out) {
  const uint32_t pair[2] = {view_left, view_right};
  return b200m_guided_match_pairs(c, pair, 1, model, F, &errorTh, distRatio, out);
}

int b200m_set_view_geometry(b200m_ctx* c, uint32_t view_id, const double* xy, int n) {
  if (!c) return fail(B200M_ERR_ARG, "ctx is null");
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  auto it = c->slot_of.find(view_id);
  if (it == c->slot_of.end()) return fail(B200M_ERR_ARG, "unknown view id");
  ViewHost& v = c->views[it->second];
  CK(cudaSetDevice(c->device));
  if (xy && n != v.m) return fail(B200M_ERR_ARG, "geometry positions: n = " + std::to_string(n) + " but the view has " + std::to_string(v.m) + " features");
  if (v.d_geom) { CK(cudaFreeAsync(v.d_geom, c->stream)); v.d_geom = nullptr; }   // stream-ordered: kernels already enqueued still see it
  if (!xy || n == 0) return B200M_OK;
  CK(cudaMallocAsync((void**)&v.d_geom, sizeof(double2) * (size_t)n, c->stream));
  CK(cudaMemcpyAsync(v.d_geom, xy, sizeof(double2) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  CK(cudaStreamSynchronize(c->stream));    // the caller's array may go once this returns
  return B200M_OK;
}

}  // extern "C"

// ---- guided matching of a pair list: b200m_guided_match_fast_pairs (K9, guided_fast.cuh), b200m_guided_match_pairs (K7, guided.cuh)
// and b200m_guided_match_positions_pairs (position-only, guided.cuh).  The three calls share one path: guided_work checks the whole
// list before anything runs, run_batches groups it into batches (the rule is DESIGN.md K7), the call's own *_run_batch runs one batch
// and appends each pair's matches to its list, and guided_result returns one list per input pair, in input order. ---------------------
template <class T> static int exclusive_scan(DeviceBuffer<>& tmp, const T* in, T* out, size_t n, cudaStream_t st, int& launches) {
  size_t tb = 0;
  CK(cub::DeviceScan::ExclusiveSum(nullptr, tb, in, out, (int64_t)n, st));
  if (int rc = tmp.reserve(tb)) return rc;
  CK(cub::DeviceScan::ExclusiveSum(tmp, tb, in, out, (int64_t)n, st));
  launches += 2;
  return B200M_OK;
}

namespace {
struct GfPairHost { int index, slot_l, slot_r, kclass; };   // kclass: kernel dtype, or 3 = mixed (uchar-stored view expanded to fp32)
// One batch: pairs of one kernel class, and the uchar-stored views of its mixed pairs, each expanded to fp32 once
struct GuidedBatch { std::vector<GfPairHost> pairs; std::set<int> expand; };
// What a call measured, summed over its batches
struct GuidedTotals { double gpu_ms = 0, search_ms = 0; int launches = 0; int64_t cands = 0; };
using PairLists = std::vector<std::vector<b200m_match>>;
}

// The work list of pairs[0 .. n_pairs), checked whole before anything runs; check(k) runs first for each entry.  A pair with an empty
// view or no common descriptor type gets an empty list (guidedMatching.hpp:300-306).  `descriptors`: the call reads descriptors (128
// scalars or 64 bytes); `upload_xy`: it needs the upload positions of both views, geometry positions are not enough.
template <class Check>
static int guided_work(b200m_ctx* c, const uint32_t* pairs, int n_pairs, bool descriptors, bool upload_xy, Check check,
                       std::vector<GfPairHost>& work) {
  for (int k = 0; k < n_pairs; ++k) {
    if (int rc = check(k)) return rc;
    auto sl = c->slot_of.find(pairs[2 * k]), sr = c->slot_of.find(pairs[2 * k + 1]);
    if (sl == c->slot_of.end() || sr == c->slot_of.end()) return fail(B200M_ERR_ARG, "guided matching references a view that was never uploaded");
    const ViewHost& vl = c->views[sl->second]; const ViewHost& vr = c->views[sr->second];
    if (!(vl.m > 0 && vr.m > 0 && vl.dtype == vr.dtype && vl.dim == vr.dim)) continue;
    if (descriptors && !((vl.dtype == DT_BIN && vl.dim == 64) || (vl.dtype != DT_BIN && vl.dim == 128)))
      return fail(B200M_ERR_UNSUPPORTED, "guided matching takes 128-component scalar or 64-byte binary descriptors");
    if (upload_xy ? (vl.xy.empty() || vr.xy.empty()) : ((vl.xy.empty() && !vl.d_geom) || (vr.xy.empty() && !vr.d_geom)))
      return fail(B200M_ERR_ARG, upload_xy ? "the decorator needs the upload positions of both views"
                                           : "guided matching needs feature positions (or geometry positions) for both views");
    work.push_back({k, sl->second, sr->second, 0});
  }
  return B200M_OK;
}

// Walks the work list once in input order; each pair joins the open batch of its kernel class (uchar, fp32, mixed, binary; one class
// when `by_class` is false), and run(batch) runs a batch when one more pair would pass one of its bounds: 8192 pairs, left_cap left
// features (a larger pair runs alone), right_cap right features, bucket_cap buckets (buckets_of(index) per pair) or 64 Mi fp32
// expansion elements.  The open batches run at the end, class by class.  Each view is waited for when its first pair is reached.
template <class BucketsOf, class Run>
static int run_batches(b200m_ctx* c, const std::vector<GfPairHost>& work, bool by_class, long left_cap, long right_cap, long bucket_cap,
                       BucketsOf buckets_of, Run run) {
  const long pair_cap = 8192, exp_cap = 64l << 20;
  struct Open { GuidedBatch b; long l = 0, r = 0, nb = 0, e = 0; };
  Open open[4];
  auto flush = [&](Open& o) -> int {
    if (o.b.pairs.empty()) return B200M_OK;
    const int rc = run(o.b);
    o = Open();
    return rc;
  };
  for (GfPairHost p : work) {
    int rc;
    if ((rc = ensure_view_ready(c, p.slot_l)) || (rc = ensure_view_ready(c, p.slot_r))) return rc;
    // the stored type is final once the view is ready (a uchar-staged view that met a non-integer value was re-uploaded as fp32)
    const ViewHost& vl = c->views[p.slot_l]; const ViewHost& vr = c->views[p.slot_r];
    p.kclass = !by_class ? 0 : vl.store_dtype() == vr.store_dtype() ? vl.store_dtype() : 3;
    Open& o = open[p.kclass];
    const long nb = buckets_of(p.index);
    const int su = p.kclass == 3 ? (vl.stored_u8 ? p.slot_l : p.slot_r) : -1;
    auto expansion = [&] { return su >= 0 && !o.b.expand.count(su) ? (long)c->views[su].m * 128 : 0l; };   // elements the pair adds
    if (!o.b.pairs.empty() && ((long)o.b.pairs.size() + 1 > pair_cap || o.l + vl.m > left_cap || o.r + vr.m > right_cap ||
                               o.nb + nb > bucket_cap || o.e + expansion() > exp_cap))
      if ((rc = flush(o))) return rc;
    o.e += expansion();
    if (su >= 0) o.b.expand.insert(su);
    o.b.pairs.push_back(p);
    o.l += vl.m; o.r += vr.m; o.nb += nb;
  }
  for (Open& o : open)
    if (int rc = flush(o)) return rc;
  return B200M_OK;
}

// The fp32 copies of a batch's uchar-stored views in `buf`, one u8_to_f32_kernel each; x[slot] is the copy of view `slot`
static int expand_views(b200m_ctx* c, DeviceBuffer<>& buf, const std::set<int>& views, std::map<int, const float*>& x, int& launches) {
  size_t total = 0;
  for (int s : views) total += (size_t)c->views[s].m * 128;
  if (int rc = buf.reserve(sizeof(float) * total)) return rc;
  float* d = buf.as<float>();
  for (int s : views) {
    const ViewHost& vu = c->views[s];
    const size_t ne = (size_t)vu.m * 128;
    u8_to_f32_kernel<<<(unsigned)((ne + 255) / 256), 256, 0, c->stream>>>((const uint8_t*)vu.raw, d, ne);
    x[s] = d; d += ne; ++launches;
  }
  return B200M_OK;
}

// Adds the batch's GPU time (ev_start .. ev_end) and its search kernel's (k0 .. k1) to t, once the stream is synchronised
static int add_times(b200m_ctx* c, cudaEvent_t k0, cudaEvent_t k1, GuidedTotals& t) {
  float ms = 0.f, kms = 0.f;
  CK(cudaEventElapsedTime(&ms, c->ev_start, c->ev_end));
  CK(cudaEventElapsedTime(&kms, k0, k1));
  t.gpu_ms += ms; t.search_ms += kms;
  return B200M_OK;
}

// Appends the (i, j) of h[b .. e) to L as IndMatch(i, j): ratio and distance 0
static void append_matches(std::vector<b200m_match>& L, const uint2* h, int b, int e) {
  const size_t n0 = L.size();
  L.resize(n0 + (size_t)std::max(e - b, 0));
  for (b200m_match* m = L.data() + n0; b < e; ++b) *m++ = b200m_match{h[b].x, h[b].y, 0.f, 0.f};
}

// One result pair per input pair, in input order (empty lists included)
static b200m_result* guided_result(b200m_ctx* c, const uint32_t* pairs, int n_pairs, const PairLists& per_pair) {
  std::unique_ptr<b200m_result> res(new b200m_result());
  res->recycler = c->recycler;
  res->pair_ids.assign(pairs, pairs + 2 * (size_t)n_pairs);
  res->offsets.assign((size_t)n_pairs + 1, 0);
  for (int k = 0; k < n_pairs; ++k) res->offsets[k + 1] = res->offsets[k] + (int64_t)per_pair[k].size();
  res->matches = c->recycler->take((size_t)std::max<int64_t>(res->offsets[n_pairs], 1));
  for (int k = 0; k < n_pairs; ++k) std::copy(per_pair[k].begin(), per_pair[k].end(), res->matches.p + res->offsets[k]);
  return res.release();
}

// One K9 batch (guidedMatchingFundamentalFast, one kernel class)
static int gf_run_batch(b200m_ctx* c, const GuidedBatch& b, const double* F, const double* ep2, const int32_t* wh, double errorTh,
                        double distRatio, PairLists& per_pair, GuidedTotals& t) {
  GuidedFastScratch& g = c->gf;
  using G = GuidedFastScratch;
  cudaStream_t st = c->stream;
  const std::vector<GfPairHost>& batch = b.pairs;
  const int np = (int)batch.size();
  const int kclass = batch[0].kclass;
  int rc;
  if ((rc = g.h_pairs.reserve(sizeof(FastPair) * (size_t)np))) return rc;
  FastPair* hp = g.h_pairs;
  long sum_l = 0, sum_r = 0, sum_b = 0; int max_l = 0, max_r = 0;
  for (int k = 0; k < np; ++k) {
    const GfPairHost& q = batch[k];
    const ViewHost& vl = c->views[q.slot_l]; const ViewHost& vr = c->views[q.slot_r];
    FastPair& P = hp[k];
    std::memset(&P, 0, sizeof(P));
    P.rawl = vl.raw; P.rawr = vr.raw;
    P.gl = vl.d_geom; P.gr = vr.d_geom; P.fl = (const float2*)vl.d_xy; P.fr = (const float2*)vr.d_xy;
    // normalise once (guidedMatching.hpp:378-385): F and ep2 negated when ep2(2) > 0, then ep2 / ep2(2)
    const double* f = F + 9 * (size_t)q.index; const double* e = ep2 + 3 * (size_t)q.index;
    const bool neg = e[2] > 0.0;
    for (int u = 0; u < 9; ++u) P.F[u] = neg ? -f[u] : f[u];
    const double e0 = neg ? -e[0] : e[0], e1 = neg ? -e[1] : e[1], e2 = neg ? -e[2] : e[2];
    P.e0 = e0 / e2; P.e1 = e1 / e2; P.e2 = e2 / e2;
    P.ml = vl.m; P.mr = vr.m; P.W = wh[2 * q.index]; P.H = wh[2 * q.index + 1]; P.nb = 2 * (P.W + P.H - 2);
    P.left_base = (int)sum_l; P.right_base = (int)sum_r; P.bucket_base = (int)sum_b;
    sum_l += vl.m; sum_r += vr.m; sum_b += P.nb + 1;
    max_l = std::max(max_l, vl.m); max_r = std::max(max_r, vr.m);
  }
  const size_t i4 = sizeof(int), u8 = sizeof(unsigned long long);
  if ((rc = g.d[G::PAIRS].reserve(sizeof(FastPair) * np)) || (rc = g.d[G::LBUCKET].reserve(i4 * sum_l)) || (rc = g.d[G::BEST].reserve(u8 * sum_l)) ||
      (rc = g.d[G::SECOND].reserve(u8 * sum_l)) || (rc = g.d[G::BCOUNT].reserve(i4 * sum_b)) || (rc = g.d[G::BOFF].reserve(i4 * sum_b)) ||
      (rc = g.d[G::CSR].reserve(i4 * sum_l)) || (rc = g.d[G::RSTART].reserve(i4 * sum_r)) || (rc = g.d[G::RCOUNT].reserve(u8 * (sum_r + 1))) ||
      (rc = g.d[G::RCOFF].reserve(u8 * (sum_r + 1))) || (rc = g.d[G::RPAIR].reserve(i4 * sum_r)) || (rc = g.d[G::KEEP].reserve(i4 * (sum_l + 1))) ||
      (rc = g.d[G::KPOS].reserve(i4 * (sum_l + 1))) || (rc = g.d[G::OUT].reserve(sizeof(uint2) * sum_l)) || (rc = g.d[G::PSTART].reserve(i4 * (np + 1))))
    return rc;
  FastPair* d_pairs = g.d[G::PAIRS].as<FastPair>();
  int *d_lbucket = g.d[G::LBUCKET].as<int>(), *d_bcount = g.d[G::BCOUNT].as<int>(), *d_boff = g.d[G::BOFF].as<int>(), *d_csr = g.d[G::CSR].as<int>(),
      *d_rstart = g.d[G::RSTART].as<int>(), *d_rpair = g.d[G::RPAIR].as<int>(), *d_keep = g.d[G::KEEP].as<int>(), *d_kpos = g.d[G::KPOS].as<int>(),
      *d_pstart = g.d[G::PSTART].as<int>();
  unsigned long long *d_best = g.d[G::BEST].as<unsigned long long>(), *d_second = g.d[G::SECOND].as<unsigned long long>(),
                     *d_rcount = g.d[G::RCOUNT].as<unsigned long long>(), *d_rcoff = g.d[G::RCOFF].as<unsigned long long>();
  uint2* d_out = g.d[G::OUT].as<uint2>();
  // the temporary storage of the three scans is taken inside exclusive_scan; reserve it for the largest one first so that
  // no reallocation (a synchronising cudaFree) happens between launches
  { size_t tb = 0; CK(cub::DeviceScan::ExclusiveSum(nullptr, tb, d_rcount, d_rcoff, (int64_t)std::max(sum_r + 1, std::max(sum_b, sum_l + 1)), st));
    if ((rc = g.d[G::TEMP].reserve(tb))) return rc; }
  if ((rc = g.ev_c0.create()) || (rc = g.ev_c1.create())) return rc;
  CK(cudaEventRecord(c->ev_start, st));
  std::map<int, const float*> x;
  if ((rc = expand_views(c, g.d[G::EXPAND], b.expand, x, t.launches))) return rc;
  for (int k = 0; k < np && kclass == 3; ++k)      // mixed pairs read the fp32 copy of their uchar-stored view
    if (c->views[batch[k].slot_l].stored_u8) hp[k].rawl = x[batch[k].slot_l]; else hp[k].rawr = x[batch[k].slot_r];
  CK(cudaMemcpyAsync(d_pairs, hp, sizeof(FastPair) * (size_t)np, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(d_bcount, 0, sizeof(int) * (size_t)sum_b, st));
  CK(cudaMemsetAsync(d_rcount + sum_r, 0, sizeof(unsigned long long), st));
  CK(cudaMemsetAsync(d_keep + sum_l, 0, sizeof(int), st));
  const dim3 gl((max_l + GF_THREADS - 1) / GF_THREADS, np), gr((max_r + GF_THREADS - 1) / GF_THREADS, np);
  guided_fast_left_kernel<<<gl, GF_THREADS, 0, st>>>(d_pairs, d_lbucket, d_bcount, d_best, d_second);
  if ((rc = exclusive_scan(g.d[G::TEMP], d_bcount, d_boff, (size_t)sum_b, st, t.launches))) return rc;
  CK(cudaMemcpyAsync(d_bcount, d_boff, sizeof(int) * (size_t)sum_b, cudaMemcpyDeviceToDevice, st));   // scatter cursors
  guided_fast_scatter_kernel<<<gl, GF_THREADS, 0, st>>>(d_pairs, d_lbucket, d_bcount, d_csr);
  guided_fast_right_kernel<<<gr, GF_THREADS, 0, st>>>(d_pairs, std::sqrt(errorTh), d_boff, d_rstart, d_rcount, d_rpair);
  if ((rc = exclusive_scan(g.d[G::TEMP], d_rcount, d_rcoff, (size_t)sum_r + 1, st, t.launches))) return rc;
  CK(cudaEventRecord(g.ev_c0, st));
  const int cgrid = c->num_sms * 8;
  if (kclass == DT_U8) guided_fast_cand_kernel<DT_U8><<<cgrid, GF_THREADS, 0, st>>>(d_pairs, (int)sum_r, d_rcoff, d_rstart, d_rpair, d_csr, d_best, d_second);
  else if (kclass == DT_BIN) guided_fast_cand_kernel<DT_BIN><<<cgrid, GF_THREADS, 0, st>>>(d_pairs, (int)sum_r, d_rcoff, d_rstart, d_rpair, d_csr, d_best, d_second);
  else guided_fast_cand_kernel<DT_F32><<<cgrid, GF_THREADS, 0, st>>>(d_pairs, (int)sum_r, d_rcoff, d_rstart, d_rpair, d_csr, d_best, d_second);
  CK(cudaEventRecord(g.ev_c1, st));
  guided_fast_keep_kernel<<<gl, GF_THREADS, 0, st>>>(d_pairs, distRatio, d_best, d_second, d_keep);
  if ((rc = exclusive_scan(g.d[G::TEMP], d_keep, d_kpos, (size_t)sum_l + 1, st, t.launches))) return rc;
  guided_fast_emit_kernel<<<gl, GF_THREADS, 0, st>>>(d_pairs, np, (int)sum_l, d_keep, d_kpos, d_best, d_out, d_pstart);
  CK(cudaGetLastError());
  t.launches += 5;
  CK(cudaEventRecord(c->ev_end, st));
  // read-back: the candidate total + per-pair starts, then the matches
  if ((rc = g.h_meta.reserve(sizeof(unsigned long long) + sizeof(int) * (size_t)(np + 1)))) return rc;
  unsigned long long* h_total = g.h_meta.as<unsigned long long>();
  int* h_pstart = reinterpret_cast<int*>(h_total + 1);
  CK(cudaMemcpyAsync(h_pstart, d_pstart, sizeof(int) * (size_t)(np + 1), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h_total, d_rcoff + sum_r, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const int n_out = h_pstart[np];
  std::vector<int> starts(h_pstart, h_pstart + np + 1);
  t.cands += (int64_t)*h_total;
  if ((rc = add_times(c, g.ev_c0, g.ev_c1, t))) return rc;
  if (n_out > 0) {
    if ((rc = g.h_out.reserve(sizeof(uint2) * (size_t)n_out))) return rc;
    CK(cudaMemcpyAsync(g.h_out, d_out, sizeof(uint2) * (size_t)n_out, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int k = 0; k < np; ++k) append_matches(per_pair[batch[k].index], g.h_out, starts[k], starts[k + 1]);
  }
  return B200M_OK;
}

// One K7 batch (guidedMatching with descriptors, one kernel class)
static int gm_run_batch(b200m_ctx* c, const GuidedBatch& b, int model, const double* M, const double* errorTh, double distRatio,
                        PairLists& per_pair, GuidedTotals& t) {
  GuidedScratch& g = c->gm;
  using G = GuidedScratch;
  cudaStream_t st = c->stream;
  const std::vector<GfPairHost>& batch = b.pairs;
  const int np = (int)batch.size();
  const int kclass = batch[0].kclass;
  int rc;
  if ((rc = g.h_pairs.reserve(sizeof(GuidedPair) * (size_t)np))) return rc;
  GuidedPair* hp = g.h_pairs;
  long sum_l = 0, blocks = 0;
  for (int k = 0; k < np; ++k) {
    const GfPairHost& q = batch[k];
    const ViewHost& vl = c->views[q.slot_l]; const ViewHost& vr = c->views[q.slot_r];
    GuidedPair& P = hp[k];
    std::memset(&P, 0, sizeof(P));
    P.rawl = vl.raw; P.rawr = vr.raw;
    P.gl = vl.d_geom; P.gr = vr.d_geom; P.fl = (const float2*)vl.d_xy; P.fr = (const float2*)vr.d_xy;
    for (int u = 0; u < 9; ++u) P.M[u] = M[9 * (size_t)q.index + u];
    P.errorTh = errorTh[q.index];
    P.model = model == B200M_MODEL_HOMOGRAPHY ? GM_HOMOGRAPHY : GM_FUNDAMENTAL;
    P.ml = vl.m; P.mr = vr.m;
    P.block_base = (int)blocks; P.left_base = (int)sum_l;
    blocks += (vl.m + GM_WARPS - 1) / GM_WARPS; sum_l += vl.m;
  }
  const size_t i4 = sizeof(int), hdr = (size_t)(np + 2) / 2;      // hdr: uint2 words in front of the matches holding the np + 1 starts
  if ((rc = g.d[G::PAIRS].reserve(sizeof(GuidedPair) * np)) || (rc = g.d[G::BESTJ].reserve(i4 * sum_l)) || (rc = g.d[G::KEEP].reserve(i4 * (sum_l + 1))) ||
      (rc = g.d[G::KPOS].reserve(i4 * (sum_l + 1))) || (rc = g.d[G::OUT].reserve(sizeof(uint2) * (hdr + sum_l))) ||
      (rc = g.h_out.reserve(sizeof(uint2) * (hdr + sum_l))))
    return rc;
  GuidedPair* d_pairs = g.d[G::PAIRS].as<GuidedPair>();
  int *d_bestj = g.d[G::BESTJ].as<int>(), *d_keep = g.d[G::KEEP].as<int>(), *d_kpos = g.d[G::KPOS].as<int>();
  uint2* d_out = g.d[G::OUT].as<uint2>();
  // reserve the scan's temporary storage before the first launch: no reallocation (a synchronising cudaFree) between launches
  { size_t tb = 0; CK(cub::DeviceScan::ExclusiveSum(nullptr, tb, d_keep, d_kpos, (int64_t)(sum_l + 1), st));
    if ((rc = g.d[G::TEMP].reserve(tb))) return rc; }
  if ((rc = g.ev_k0.create()) || (rc = g.ev_k1.create())) return rc;
  CK(cudaEventRecord(c->ev_start, st));
  std::map<int, const float*> x;
  if ((rc = expand_views(c, g.d[G::EXPAND], b.expand, x, t.launches))) return rc;
  for (int k = 0; k < np && kclass == 3; ++k)      // mixed pairs read the fp32 copy of their uchar-stored view
    if (c->views[batch[k].slot_l].stored_u8) hp[k].rawl = x[batch[k].slot_l]; else hp[k].rawr = x[batch[k].slot_r];
  CK(cudaMemcpyAsync(d_pairs, hp, sizeof(GuidedPair) * (size_t)np, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(d_keep + sum_l, 0, sizeof(int), st));
  CK(cudaEventRecord(g.ev_k0, st));
  if (kclass == DT_U8) guided_pairs_kernel<DT_U8><<<(unsigned)blocks, GM_WARPS * 32, 0, st>>>(d_pairs, np, distRatio, d_bestj, d_keep);
  else if (kclass == DT_BIN) guided_pairs_kernel<DT_BIN><<<(unsigned)blocks, GM_WARPS * 32, 0, st>>>(d_pairs, np, distRatio, d_bestj, d_keep);
  else guided_pairs_kernel<DT_F32><<<(unsigned)blocks, GM_WARPS * 32, 0, st>>>(d_pairs, np, distRatio, d_bestj, d_keep);
  CK(cudaEventRecord(g.ev_k1, st));
  if ((rc = exclusive_scan(g.d[G::TEMP], d_keep, d_kpos, (size_t)sum_l + 1, st, t.launches))) return rc;
  const long emit_threads = std::max(sum_l, (long)np + 1);
  guided_pairs_emit_kernel<<<(unsigned)((emit_threads + 255) / 256), 256, 0, st>>>(d_pairs, np, (int)sum_l, d_bestj, d_keep, d_kpos, d_out + hdr,
                                                                                  reinterpret_cast<int*>(d_out));
  CK(cudaGetLastError());
  t.launches += 2;
  CK(cudaEventRecord(c->ev_end, st));
  // one read-back: the per-pair starts and every slot the matches may occupy
  CK(cudaMemcpyAsync(g.h_out, d_out, sizeof(uint2) * (hdr + sum_l), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if ((rc = add_times(c, g.ev_k0, g.ev_k1, t))) return rc;
  const int* h_pstart = g.h_out.as<int>();
  const uint2* h = g.h_out.as<uint2>() + hdr;
  for (int k = 0; k < np; ++k) append_matches(per_pair[batch[k].index], h, h_pstart[k], h_pstart[k + 1]);
  return B200M_OK;
}

// One position-only batch: each pair's guidedMatching list (the phantom (0, 0) included), decorated when `decorate`
static int gp_run_batch(b200m_ctx* c, const GuidedBatch& b, int model, const double* M, const double* errorTh, bool decorate,
                        PairLists& per_pair, GuidedTotals& t) {
  GuidedScratch& g = c->gm;
  using G = GuidedScratch;
  cudaStream_t st = c->stream;
  const std::vector<GfPairHost>& batch = b.pairs;
  const int np = (int)batch.size();
  int rc;
  if ((rc = g.h_pairs.reserve(sizeof(GuidedPair) * (size_t)np)) || (rc = g.h_yrank.reserve(sizeof(uint32_t*) * (size_t)np))) return rc;
  GuidedPair* hp = g.h_pairs;
  const uint32_t** hy = g.h_yrank;
  long sum_l = 0, blocks = 0;
  bool dev_deco = false;
  for (int k = 0; k < np; ++k) {
    const GfPairHost& q = batch[k];
    const ViewHost& vl = c->views[q.slot_l]; const ViewHost& vr = c->views[q.slot_r];
    GuidedPair& P = hp[k];
    std::memset(&P, 0, sizeof(P));
    P.gl = vl.d_geom; P.gr = vr.d_geom; P.fl = (const float2*)vl.d_xy; P.fr = (const float2*)vr.d_xy;
    for (int u = 0; u < 9; ++u) P.M[u] = M[9 * (size_t)q.index + u];
    P.errorTh = errorTh[q.index];
    P.model = model == B200M_MODEL_HOMOGRAPHY ? GM_HOMOGRAPHY : GM_FUNDAMENTAL;
    P.ml = vl.m; P.mr = vr.m;
    P.block_base = (int)blocks; P.left_base = (int)sum_l;
    blocks += (vl.m + GP_THREADS - 1) / GP_THREADS; sum_l += vl.m;
    // the decorator on the device: left view in general position (pos_rank_kernel's flag, read back with the view)
    hy[k] = decorate && c->device_finish && vl.d_yrank && !(vl.flags & VF_POS_NONGENERIC) ? vl.d_yrank : nullptr;
    dev_deco |= hy[k] != nullptr;
  }
  // d_out: np + 1 pair starts and np phantom flags (ints) in hdr uint2 words, then the matches
  const size_t i4 = sizeof(int), hdr = (size_t)np + 1;
  if ((rc = g.d[G::PAIRS].reserve(sizeof(GuidedPair) * np)) || (rc = g.d[G::BESTJ].reserve(i4 * sum_l)) || (rc = g.d[G::KEEP].reserve(i4 * (sum_l + 1))) ||
      (rc = g.d[G::KPOS].reserve(i4 * (sum_l + 1))) || (rc = g.d[G::OUT].reserve(sizeof(uint2) * (hdr + sum_l))) ||
      (rc = g.h_out.reserve(sizeof(uint2) * (hdr + sum_l))))
    return rc;
  if (dev_deco && ((rc = g.d[G::YRANK].reserve(sizeof(uint32_t*) * np)) || (rc = g.d[G::REC].reserve(sizeof(uint2) * sum_l)) ||
                   (rc = g.d[G::KEEP2].reserve(i4 * (sum_l + 1)))))
    return rc;
  GuidedPair* d_pairs = g.d[G::PAIRS].as<GuidedPair>();
  int *d_bestj = g.d[G::BESTJ].as<int>(), *d_keep = g.d[G::KEEP].as<int>(), *d_kpos = g.d[G::KPOS].as<int>();
  uint2* d_out = g.d[G::OUT].as<uint2>();
  int* d_pstart = reinterpret_cast<int*>(d_out);
  int* d_phantom = d_pstart + np + 1;
  int* d_scan_in = dev_deco ? g.d[G::KEEP2].as<int>() : d_keep;      // the slots the compaction reads
  { size_t tb = 0; CK(cub::DeviceScan::ExclusiveSum(nullptr, tb, d_scan_in, d_kpos, (int64_t)(sum_l + 1), st));
    if ((rc = g.d[G::TEMP].reserve(tb))) return rc; }
  if ((rc = g.ev_k0.create()) || (rc = g.ev_k1.create())) return rc;
  CK(cudaEventRecord(c->ev_start, st));
  CK(cudaMemcpyAsync(d_pairs, hp, sizeof(GuidedPair) * (size_t)np, cudaMemcpyHostToDevice, st));
  if (dev_deco) CK(cudaMemcpyAsync(g.d[G::YRANK], hy, sizeof(uint32_t*) * (size_t)np, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(d_phantom, 0, i4 * np, st));
  CK(cudaMemsetAsync(d_scan_in + sum_l, 0, sizeof(int), st));
  CK(cudaEventRecord(g.ev_k0, st));
  guided_positions_pairs_kernel<<<(unsigned)blocks, GP_THREADS, 0, st>>>(d_pairs, np, d_bestj, d_keep, d_phantom);
  CK(cudaEventRecord(g.ev_k1, st));
  ++t.launches;
  const long emit_threads = std::max(sum_l, (long)np + 1);
  const unsigned emit_blocks = (unsigned)((emit_threads + 255) / 256);
  if (dev_deco) {
    uint2* d_rec = g.d[G::REC].as<uint2>();
    guided_positions_deco_kernel<<<(unsigned)((sum_l + 255) / 256), 256, 0, st>>>(d_pairs, g.d[G::YRANK].as<const uint32_t*>(), np, (int)sum_l, d_bestj,
                                                                                 d_phantom, d_rec, d_scan_in);
    if ((rc = exclusive_scan(g.d[G::TEMP], d_scan_in, d_kpos, (size_t)sum_l + 1, st, t.launches))) return rc;
    guided_positions_emit_kernel<<<emit_blocks, 256, 0, st>>>(d_pairs, np, (int)sum_l, d_rec, d_scan_in, d_kpos, d_out + hdr, d_pstart);
  } else {
    if ((rc = exclusive_scan(g.d[G::TEMP], d_keep, d_kpos, (size_t)sum_l + 1, st, t.launches))) return rc;
    guided_pairs_emit_kernel<<<emit_blocks, 256, 0, st>>>(d_pairs, np, (int)sum_l, d_bestj, d_keep, d_kpos, d_out + hdr, d_pstart);
  }
  CK(cudaGetLastError());
  t.launches += dev_deco ? 2 : 1;
  CK(cudaEventRecord(c->ev_end, st));
  CK(cudaMemcpyAsync(g.h_out, d_out, sizeof(uint2) * (hdr + sum_l), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if ((rc = add_times(c, g.ev_k0, g.ev_k1, t))) return rc;
  const int* h_pstart = g.h_out.as<int>();
  const int* h_phantom = h_pstart + np + 1;
  const uint2* h = g.h_out.as<uint2>() + hdr;
  for (int k = 0; k < np; ++k) {
    std::vector<b200m_match>& L = per_pair[batch[k].index];
    if (h_phantom[k] && !hy[k] && !(h_pstart[k + 1] > h_pstart[k] && h[h_pstart[k]].x == 0 && h[h_pstart[k]].y == 0))
      L.push_back(b200m_match{0, 0, 0.f, 0.f});                       // IndMatch() sorts first; a real (0, 0) is the same match
    append_matches(L, h, h_pstart[k], h_pstart[k + 1]);
    if (decorate && !hy[k] && !L.empty()) {
      const ViewHost& vl = c->views[batch[k].slot_l]; const ViewHost& vr = c->views[batch[k].slot_r];
      L.resize((size_t)decorator_dedup(L.data(), (int)L.size(), vl.xy.data(), vr.xy.data()));
    }
  }
  return B200M_OK;
}

extern "C" {

int b200m_guided_match_fast_pairs(b200m_ctx* c, const uint32_t* pairs, int n_pairs, const double* F, const double* epipole2, const int32_t* wh,
                                  double errorTh, double distRatio, b200m_result** out) {
  if (!c || !out || n_pairs < 0 || (n_pairs > 0 && (!pairs || !F || !epipole2 || !wh))) return fail(B200M_ERR_ARG, "bad arguments");
  *out = nullptr;
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  CK(cudaSetDevice(c->device));
  auto check_wh = [wh](int k) {
    const int W = wh[2 * k], H = wh[2 * k + 1];
    if (W < 2 || H < 2 || W > (1 << 24) || H > (1 << 24))
      return fail(B200M_ERR_ARG, "pair " + std::to_string(k) + ": the right image must be at least 2 x 2 pixels (and at most 2^24 on a side)");
    return (int)B200M_OK;
  };
  std::vector<GfPairHost> work;
  if (int rc = guided_work(c, pairs, n_pairs, true, false, check_wh, work)) return rc;
  PairLists per_pair((size_t)n_pairs);
  GuidedTotals t;
  auto buckets = [wh](int k) { return 2l * (wh[2 * k] + wh[2 * k + 1] - 2) + 1; };
  auto run = [&](const GuidedBatch& b) { return gf_run_batch(c, b, F, epipole2, wh, errorTh, distRatio, per_pair, t); };
  if (int rc = run_batches(c, work, true, c->gf_left_cap, std::max(c->gf_left_cap, 1l << 20), 16l << 20, buckets, run)) return rc;
  if (int rc = wait_uploads(c)) return rc;
  c->last = LastCall{t.gpu_ms, t.search_ms, t.launches, 0, 0, 0, t.cands, 0};
  *out = guided_result(c, pairs, n_pairs, per_pair);
  return B200M_OK;
}

int b200m_guided_match_pairs(b200m_ctx* c, const uint32_t* pairs, int n_pairs, int model, const double* M, const double* errorTh, double distRatio,
                             b200m_result** out) {
  if (!c || !out || n_pairs < 0 || (model != B200M_MODEL_FUNDAMENTAL && model != B200M_MODEL_HOMOGRAPHY) ||
      (n_pairs > 0 && (!pairs || !M || !errorTh)))
    return fail(B200M_ERR_ARG, "bad arguments");
  *out = nullptr;
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  CK(cudaSetDevice(c->device));
  std::vector<GfPairHost> work;
  if (int rc = guided_work(c, pairs, n_pairs, true, false, [](int) { return 0; }, work)) return rc;
  PairLists per_pair((size_t)n_pairs);
  GuidedTotals t;
  auto run = [&](const GuidedBatch& b) { return gm_run_batch(c, b, model, M, errorTh, distRatio, per_pair, t); };
  if (int rc = run_batches(c, work, true, c->gm_left_cap, LONG_MAX, LONG_MAX, [](int) { return 0l; }, run)) return rc;
  if (int rc = wait_uploads(c)) return rc;
  *out = guided_result(c, pairs, n_pairs, per_pair);
  c->last = LastCall{t.gpu_ms, t.search_ms, t.launches, 0, 0, 0, (*out)->offsets[n_pairs], 0};
  return B200M_OK;
}

int b200m_guided_match_positions_pairs(b200m_ctx* c, const uint32_t* pairs, int n_pairs, int model, const double* M, const double* errorTh,
                                       int decorate, b200m_result** out) {
  if (!c || !out || n_pairs < 0 || (model != B200M_MODEL_FUNDAMENTAL && model != B200M_MODEL_HOMOGRAPHY) || (decorate != 0 && decorate != 1) ||
      (n_pairs > 0 && (!pairs || !M || !errorTh)))
    return fail(B200M_ERR_ARG, "bad arguments");
  *out = nullptr;
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  CK(cudaSetDevice(c->device));
  std::vector<GfPairHost> work;
  if (int rc = guided_work(c, pairs, n_pairs, false, decorate != 0, [](int) { return 0; }, work)) return rc;
  PairLists per_pair((size_t)n_pairs);
  GuidedTotals t;
  auto run = [&](const GuidedBatch& b) { return gp_run_batch(c, b, model, M, errorTh, decorate != 0, per_pair, t); };
  if (int rc = run_batches(c, work, false, c->gm_left_cap, LONG_MAX, LONG_MAX, [](int) { return 0l; }, run)) return rc;
  if (int rc = wait_uploads(c)) return rc;
  *out = guided_result(c, pairs, n_pairs, per_pair);
  c->last = LastCall{t.gpu_ms, t.search_ms, t.launches, 0, 0, 0, (*out)->offsets[n_pairs], 0};
  return B200M_OK;
}

}  // extern "C"

// ---- K12: homography growing for a list of work items (hgrowing.cuh) ----
// Items go in batches, in input order: a batch holds at most kHgBatchPutatives putatives and kHgBatchSeeds / window items.  Per batch
// and round: for each window w < ceil(n_max / window), one grow and one replay launch over the whole batch; then one finish launch.
// The call's features and outputs stay on the device throughout, and the outputs come back in one copy at the end.
constexpr long long kHgBatchPutatives = 1ll << 24;
constexpr long long kHgBatchSeeds = 1ll << 21;

static int hgrowing_pairs(b200m_ctx* c, int n_items, const int64_t* offsets, const float* feat, const hg::Param& p, int32_t* n_h_out,
                          double* H_out, int32_t* counts_out, int32_t* inl_out, int32_t* trace_out, int32_t* rounds_out) {
  const int mh = p.max_nb_homographies;
  const long long N = n_items ? offsets[n_items] : 0;
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  CK(cudaSetDevice(c->device));
  HgrowingScratch& S = c->hgr;
  S.last_ms = 0; S.stats[0] = S.stats[1] = S.stats[2] = 0;
  if (n_items == 0) return B200M_OK;
  const int W = S.window;
  // batches: [first item, last item + 1)
  std::vector<std::pair<int, int>> batches;
  for (int k = 0; k < n_items;) {
    int e = k;
    long long put = 0;
    while (e < n_items && (e == k || (put + (offsets[e + 1] - offsets[e]) <= kHgBatchPutatives && (long long)(e - k + 1) * W <= kHgBatchSeeds))) {
      put += offsets[e + 1] - offsets[e];
      ++e;
    }
    batches.emplace_back(k, e);
    k = e;
  }
  // the largest batch sizes the batch region
  long long b_put = 0, b_words = 0, b_items = 0, n_max = 0;
  for (auto& b : batches) {
    long long put = 0, words = 0;
    for (int k = b.first; k < b.second; ++k) {
      const long long n = offsets[k + 1] - offsets[k];
      put += n; words += (n + 31) / 32; n_max = std::max(n_max, n);
    }
    b_put = std::max(b_put, put); b_words = std::max(b_words, words); b_items = std::max(b_items, (long long)(b.second - b.first));
  }
  const int grow_blocks = (int)std::min<long long>((b_items * W + hgk::kWarps - 1) / hgk::kWarps, (long long)c->num_sms * 8);
  const long long scratch_words = std::max<long long>(1, (n_max + 31) / 32);
  const size_t rows = (size_t)n_items * std::max(mh, 1);
  size_t at = 0;
  auto take = [&](size_t bytes) { const size_t o = at; at += (bytes + 255) & ~(size_t)255; return o; };
  // output region first: one contiguous read-back
  const size_t o_H = take(sizeof(double) * 9 * rows), o_stats = take(sizeof(unsigned long long) * 2), o_cnt = take(sizeof(int) * rows),
               o_tr = take(sizeof(int) * 3 * rows), o_nh = take(sizeof(int) * n_items), o_rounds = take(sizeof(int) * n_items),
               o_inl = take(sizeof(int) * std::max<long long>(N, 1));
  const size_t out_bytes = at;
  const size_t o_feat = take(sizeof(float) * hg::kFeat * std::max<long long>(N, 1)), o_items = take(sizeof(hgk::Item) * b_items),
               o_rem = take(sizeof(int) * std::max<long long>(b_put, 1)), o_used = take(sizeof(uint32_t) * std::max<long long>(b_words, 1)),
               o_seeds = take(sizeof(hgk::Seed) * b_items * W),
               o_scr = take(sizeof(uint32_t) * (size_t)scratch_words * grow_blocks * hgk::kWarps);
  int rc;
  if ((rc = S.d.reserve(at)) || (rc = S.ev0.create()) || (rc = S.ev1.create())) return rc;
  char* d = S.d;
  cudaStream_t st = c->stream;
  CK(cudaMemsetAsync(d, 0, out_bytes, st));
  if (N) CK(cudaMemcpyAsync(d + o_feat, feat, sizeof(float) * hg::kFeat * N, cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(S.ev0, st));
  hgk::Ctl ctl{};
  ctl.feat = (const float*)(d + o_feat);
  ctl.items = (hgk::Item*)(d + o_items);
  ctl.rem = (int*)(d + o_rem); ctl.used = (uint32_t*)(d + o_used); ctl.seeds = (hgk::Seed*)(d + o_seeds);
  ctl.window = W; ctl.scratch = (uint32_t*)(d + o_scr); ctl.scratch_words = (int)scratch_words; ctl.p = p;
  ctl.H = (double*)(d + o_H); ctl.counts = (int*)(d + o_cnt); ctl.trace = (int*)(d + o_tr); ctl.inl = (int*)(d + o_inl);
  ctl.n_h = (int*)(d + o_nh); ctl.rounds = (int*)(d + o_rounds); ctl.stats = (unsigned long long*)(d + o_stats);
  std::vector<hgk::Item> items;
  std::vector<int> rem;
  for (auto& b : batches) {
    items.clear(); rem.clear();
    long long words = 0, bmax = 0;
    for (int k = b.first; k < b.second; ++k) {
      hgk::Item it{};
      it.off = offsets[k]; it.n = it.n_r = (int)(offsets[k + 1] - offsets[k]);
      it.rem_off = (long long)rem.size(); it.used_off = words;
      it.done = mh == 0; it.best_seed = -1; it.row = k;
      for (int j = 0; j < it.n; ++j) rem.push_back(j);
      words += (it.n + 31) / 32; bmax = std::max(bmax, (long long)it.n);
      items.push_back(it);
    }
    const int nb = (int)items.size();
    ctl.n_items = nb;
    // the host vectors stay alive until the synchronise below (the copies read pageable memory when they run)
    CK(cudaMemcpyAsync(ctl.items, items.data(), sizeof(hgk::Item) * nb, cudaMemcpyHostToDevice, st));
    if (!rem.empty()) CK(cudaMemcpyAsync(ctl.rem, rem.data(), sizeof(int) * rem.size(), cudaMemcpyHostToDevice, st));
    if (words) CK(cudaMemsetAsync(ctl.used, 0, sizeof(uint32_t) * words, st));
    const int n_win = (int)((bmax + W - 1) / W);
    const int item_blocks = (nb + hgk::kWarps - 1) / hgk::kWarps;
    const int gb = (int)std::min<long long>(((long long)nb * W + hgk::kWarps - 1) / hgk::kWarps, grow_blocks);
    for (int r = 0; r < mh; ++r) {
      for (int w = 0; w < n_win; ++w) {
        hgk::hg_grow_kernel<<<gb, 32 * hgk::kWarps, 0, st>>>(ctl, w);
        hgk::hg_replay_kernel<<<item_blocks, 32 * hgk::kWarps, 0, st>>>(ctl, w);
      }
      hgk::hg_finish_kernel<<<item_blocks, 32 * hgk::kWarps, 0, st>>>(ctl);
    }
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));   // `items` and `rem` are rewritten for the next batch
  }
  CK(cudaEventRecord(S.ev1, st));
  std::vector<char> out(out_bytes);
  CK(cudaMemcpyAsync(out.data(), d, out_bytes, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, S.ev0, S.ev1));
  S.last_ms = ms;
  const unsigned long long* stats = (const unsigned long long*)(out.data() + o_stats);
  const int* nh = (const int*)(out.data() + o_nh);
  const int* rounds = (const int*)(out.data() + o_rounds);
  const int* cnt = (const int*)(out.data() + o_cnt);
  const int* inl = (const int*)(out.data() + o_inl);
  S.stats[0] = (int64_t)stats[0]; S.stats[1] = (int64_t)stats[1];
  for (int k = 0; k < n_items; ++k) {
    n_h_out[k] = nh[k];
    S.stats[2] += rounds[k];
    if (rounds_out) rounds_out[k] = rounds[k];
    long long stored = 0;
    for (int h = 0; h < nh[k]; ++h) stored += cnt[(size_t)k * mh + h];
    if (stored) std::memcpy(inl_out + offsets[k], inl + offsets[k], sizeof(int) * stored);
  }
  if (mh) {
    std::memcpy(H_out, out.data() + o_H, sizeof(double) * 9 * rows);
    std::memcpy(counts_out, cnt, sizeof(int) * rows);
    if (trace_out) std::memcpy(trace_out, out.data() + o_tr, sizeof(int) * 3 * rows);
  }
  return B200M_OK;
}

extern "C" {

int b200m_hgrowing_pairs(b200m_ctx* c, int n_items, const int64_t* offsets, const float* feat, double similarity_tolerance,
                         double affinity_tolerance, double homography_tolerance, int min_inliers_to_refine, int nb_refining_iterations,
                         int max_nb_homographies, int min_nb_matches_per_h, int32_t* n_homographies, double* H, int32_t* counts,
                         int32_t* inliers, int32_t* trace, int32_t* rounds) {
  auto tol_ok = [](double t) { return t >= 0 && t <= 1e150; };
  if (!c || n_items < 0 || (n_items > 0 && (!offsets || !n_homographies || (max_nb_homographies > 0 && (!H || !counts)))))
    return fail(B200M_ERR_ARG, "bad arguments");
  if (!tol_ok(similarity_tolerance) || !tol_ok(affinity_tolerance) || !tol_ok(homography_tolerance))
    return fail(B200M_ERR_ARG, "tolerances must be finite and non-negative");
  if (min_inliers_to_refine < 1 || nb_refining_iterations < 0 || nb_refining_iterations > 64 || max_nb_homographies < 0 ||
      max_nb_homographies > hgk::kMaxH || min_nb_matches_per_h < 0)
    return fail(B200M_ERR_ARG, "parameters out of range: min_inliers_to_refine >= 1, nb_refining_iterations 0..64, max_nb_homographies 0..64, "
                               "min_nb_matches_per_h >= 0");
  if (n_items > 0 && offsets[0] != 0) return fail(B200M_ERR_ARG, "offsets[0] must be 0");
  for (int k = 0; k < n_items; ++k) {
    const int64_t n = offsets[k + 1] - offsets[k];
    if (n < 0 || n > hgk::kMaxItem)
      return fail(B200M_ERR_ARG, "item " + std::to_string(k) + ": offsets must ascend, at most " + std::to_string(hgk::kMaxItem) +
                                     " putatives an item");
  }
  if (n_items > 0 && offsets[n_items] > 0 && (!feat || !inliers)) return fail(B200M_ERR_ARG, "bad arguments");
  hg::Param p;
  p.tol_similarity = similarity_tolerance; p.tol_affinity = affinity_tolerance; p.tol_homography = homography_tolerance;
  p.min_inliers_to_refine = min_inliers_to_refine; p.nb_refining_iterations = nb_refining_iterations;
  p.max_nb_homographies = max_nb_homographies; p.min_nb_matches_per_h = min_nb_matches_per_h;
  return hgrowing_pairs(c, n_items, offsets, feat, p, n_homographies, H, counts, inliers, trace, rounds);
}

double b200m_hgrowing_last_stats(const b200m_ctx* c, int64_t stats[3]) {
  if (!c) return 0;
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  if (stats) for (int t = 0; t < 3; ++t) stats[t] = c->hgr.stats[t];
  return c->hgr.last_ms;
}

int b200m_ctx_set_hgrowing_window(b200m_ctx* c, int window) {
  if (!c || window < 1 || window > 4096) return fail(B200M_ERR_ARG, "bad arguments: window 1..4096");
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  c->hgr.window = window;
  return B200M_OK;
}

}  // extern "C"

// ---- K10: a-contrario RANSAC for a pair list: fundamental matrix, homography, spherical fundamental matrix, essential matrix,
// fundamental matrix with radial distortion (acransac.cuh) ----
// One launch of acransac_kernel<Policy> over the list; the entry points differ in the model, the correspondence width
// (Policy::kWidth doubles; 4 pixel doubles in for the calibrated policy) and the generator contract.  wh: image sizes of the planar
// and calibrated policies (unused, may be NULL, for bearings).  K: n_pairs x 18 (K_I, K_J row-major) for the calibrated policy, else
// unused.  mt_per_pair: 0 = mt_state is one 625-word state for every pair, 1 = n_pairs x 625.  mt_out: NULL or n_pairs x 625.
// L: n_pairs x 2, the winners' radial distortion, for the distortion policy (required there), else unused.
template <class Policy>
static int acransac_pairs(b200m_ctx* c, int n_pairs, const int64_t* offsets, const double* corr, const int32_t* wh, const double* K,
                          const uint32_t* mt_state, int mt_per_pair, int64_t max_iteration, double precision, uint8_t* valid, int32_t* n_inliers,
                          uint32_t* inliers, double* model, double* error_max, double* min_nfa, int32_t* iterations, uint32_t* mt_out,
                          double* L = nullptr) {
  using OutT = std::conditional_t<Policy::kDistortion, acrk::OutL, acrk::Out>;
  constexpr bool kSized = Policy::kPlanar || Policy::kCalibrated;
  if (!c || n_pairs < 0 || max_iteration < 0 || max_iteration > INT32_MAX || !(precision > 0) || (mt_per_pair != 0 && mt_per_pair != 1) ||
      (n_pairs > 0 && (!offsets || (kSized && !wh) || (Policy::kCalibrated && !K) || !mt_state || !valid || !n_inliers || !model ||
                       !error_max || !min_nfa || !iterations || (Policy::kDistortion && !L))))
    return fail(B200M_ERR_ARG, "bad arguments");
  if (n_pairs > 0 && offsets[0] != 0) return fail(B200M_ERR_ARG, "offsets[0] must be 0");
  std::vector<acrk::Pair> pairs((size_t)n_pairs);
  std::vector<acrk::PairE> pairs_e(Policy::kCalibrated ? (size_t)n_pairs : 0);
  int64_t sort_total = 0; int max_n = 0;
  for (int k = 0; k < n_pairs; ++k) {
    const int64_t n = offsets[k + 1] - offsets[k];
    if (n < 0 || n > (1 << 24)) return fail(B200M_ERR_ARG, "pair " + std::to_string(k) + ": offsets must ascend, at most 2^24 correspondences a pair");
    int32_t s[4] = {0, 0, 0, 0};
    if (kSized)
      for (int t = 0; t < 4; ++t)
        if ((s[t] = wh[4 * k + t]) < 1) return fail(B200M_ERR_ARG, "pair " + std::to_string(k) + ": image sizes must be positive");
    if (Policy::kPlanar && ((int64_t)s[0] * s[1] > INT32_MAX || (int64_t)s[2] * s[3] > INT32_MAX))
      return fail(B200M_ERR_ARG, "pair " + std::to_string(k) + ": width * height must fit an int, as in the reference");
    if (Policy::kCalibrated) {   // K^-1 as RelativePoseKernel_K's constructor takes it; a singular K gives a non-finite inverse
      bool ok = true;
      for (int t = 0; t < 18; ++t) ok &= std::isfinite(K[18 * k + t]);
      if (ok) {
        acr::inverse3(K + 18 * k, pairs_e[k].kinv);
        acr::inverse3(K + 18 * k + 9, pairs_e[k].kinv + 9);
        for (int t = 0; t < 18; ++t) ok &= std::isfinite(pairs_e[k].kinv[t]);
      }
      if (!ok) return fail(B200M_ERR_ARG, "pair " + std::to_string(k) + ": K must be finite and invertible");
    }
    int64_t n2 = 1;
    while (n2 < n) n2 <<= 1;
    pairs[k] = acrk::Pair{offsets[k], n2 > acrk::kSmemSort ? sort_total : 0, (int)n, s[0], s[1], s[2], s[3]};
    if (n2 > acrk::kSmemSort) sort_total += n2;
    if (Policy::kCalibrated) pairs_e[k].q = pairs[k];
    max_n = std::max(max_n, (int)n);
  }
  const int64_t N = n_pairs ? offsets[n_pairs] : 0;
  if (N > 0 && (!corr || !inliers)) return fail(B200M_ERR_ARG, "bad arguments");
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  CK(cudaSetDevice(c->device));
  c->acr.trace.assign((size_t)n_pairs * acrk::kTraceCap, 0); c->acr.trace_nfa.assign((size_t)n_pairs * acrk::kTraceCap, 0);
  c->acr.n_trace.assign((size_t)n_pairs, 0);
  for (int t = 0; t < 4; ++t) c->acr.stats[t] = 0;
  c->acr.last_ms = 0;
  if (n_pairs == 0) return B200M_OK;
  // float log10 table of makelogcombi: log10 on the double k, rounded to float (pinned against the compiled reference's tables)
  std::vector<float> l10((size_t)max_n + 2);
  for (size_t k = 0; k < l10.size(); ++k) l10[k] = (float)log10((double)k);
  const size_t n_states = mt_per_pair ? (size_t)n_pairs : 1;
  // one grow-only device buffer, shared by every model
  constexpr int W = Policy::kWidth, W_in = Policy::kCalibrated ? 4 : W;
  const size_t pair_bytes = Policy::kCalibrated ? sizeof(acrk::PairE) : sizeof(acrk::Pair);
  const void* pair_src = Policy::kCalibrated ? (const void*)pairs_e.data() : (const void*)pairs.data();
  size_t at = 0;
  auto take = [&](size_t bytes) { const size_t o = at; at += (bytes + 255) & ~(size_t)255; return o; };
  const size_t o_pairs = take(pair_bytes * n_pairs), o_corr = take(sizeof(double) * W_in * N), o_l10 = take(sizeof(float) * l10.size()),
               o_mt = take(sizeof(uint32_t) * 625 * n_states), o_pts = take(sizeof(double) * W * N), o_idx = take(sizeof(uint32_t) * N),
               o_logc = take(sizeof(float) * 2 * (N + n_pairs)), o_gk = take(sizeof(unsigned long long) * sort_total),
               o_gv = take(sizeof(uint32_t) * sort_total), o_inl = take(sizeof(uint32_t) * N),
               o_tr = take(sizeof(int32_t) * acrk::kTraceCap * n_pairs),
               o_trn = take(sizeof(double) * acrk::kTraceCap * n_pairs), o_out = take(sizeof(OutT) * n_pairs),
               o_mto = take(mt_out ? sizeof(uint32_t) * 625 * n_pairs : 0);
  int rc;
  if ((rc = c->acr.d.reserve(at)) || (rc = c->acr.ev0.create()) || (rc = c->acr.ev1.create())) return rc;
  char* d = c->acr.d;
  cudaStream_t st = c->stream;
  CK(cudaMemcpyAsync(d + o_pairs, pair_src, pair_bytes * n_pairs, cudaMemcpyHostToDevice, st));
  if (N) CK(cudaMemcpyAsync(d + o_corr, corr, sizeof(double) * W_in * N, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d + o_l10, l10.data(), sizeof(float) * l10.size(), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(d + o_mt, mt_state, sizeof(uint32_t) * 625 * n_states, cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(c->acr.ev0, st));
  acrk::launch<Policy>(
      n_pairs, st, (const acrk::Pair*)(d + o_pairs), (const double*)(d + o_corr), (const float*)(d + o_l10), (const uint32_t*)(d + o_mt),
      mt_per_pair ? 625 : 0, (long long)max_iteration, precision, c->acr.skip ? 1 : 0, (double*)(d + o_pts), (uint32_t*)(d + o_idx),
      (float*)(d + o_logc), (unsigned long long*)(d + o_gk), (uint32_t*)(d + o_gv), (uint32_t*)(d + o_inl), (int*)(d + o_tr),
      (double*)(d + o_trn), (acrk::Out*)(d + o_out), mt_out ? (uint32_t*)(d + o_mto) : nullptr);
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->acr.ev1, st));
  std::vector<OutT> outs((size_t)n_pairs);
  CK(cudaMemcpyAsync(outs.data(), d + o_out, sizeof(OutT) * n_pairs, cudaMemcpyDeviceToHost, st));
  if (N) CK(cudaMemcpyAsync(inliers, d + o_inl, sizeof(uint32_t) * N, cudaMemcpyDeviceToHost, st));
  if (mt_out) CK(cudaMemcpyAsync(mt_out, d + o_mto, sizeof(uint32_t) * 625 * n_pairs, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(c->acr.trace.data(), d + o_tr, sizeof(int32_t) * acrk::kTraceCap * n_pairs, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(c->acr.trace_nfa.data(), d + o_trn, sizeof(double) * acrk::kTraceCap * n_pairs, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, c->acr.ev0, c->acr.ev1));
  c->acr.last_ms = ms;
  c->acr.stats[3] = 1;
  for (int k = 0; k < n_pairs; ++k) {
    const acrk::Out& o = reinterpret_cast<const acrk::Out&>(outs[k]);   // an OutL begins with its Out
    if constexpr (Policy::kDistortion) { L[2 * k] = outs[k].L[0]; L[2 * k + 1] = outs[k].L[1]; }
    valid[k] = (uint8_t)o.valid; n_inliers[k] = o.n_inl;
    for (int t = 0; t < 9; ++t) model[9 * k + t] = o.model[t];
    error_max[k] = o.error_max; min_nfa[k] = o.min_nfa; iterations[k] = o.iterations;
    c->acr.n_trace[k] = o.n_trace;
    c->acr.stats[0] += o.evaluated; c->acr.stats[1] += o.skipped; c->acr.stats[2] += o.exact;
  }
  return B200M_OK;
}

extern "C" {

int b200m_acransac_fundamental_pairs(b200m_ctx* c, int n_pairs, const int64_t* offsets, const double* corr, const int32_t* wh,
                                     const uint32_t* mt_state, int64_t max_iteration, double precision, uint8_t* valid,
                                     int32_t* n_inliers, uint32_t* inliers, double* F, double* error_max, double* min_nfa,
                                     int32_t* iterations) {
  return acransac_pairs<acrk::FPolicy>(c, n_pairs, offsets, corr, wh, nullptr, mt_state, 0, max_iteration, precision, valid, n_inliers, inliers, F,
                                       error_max, min_nfa, iterations, nullptr);
}

int b200m_acransac_homography_pairs(b200m_ctx* c, int n_pairs, const int64_t* offsets, const double* corr, const int32_t* wh,
                                    const uint32_t* mt_state, int mt_state_per_pair, int64_t max_iteration, double precision, uint8_t* valid,
                                    int32_t* n_inliers, uint32_t* inliers, double* H, double* error_max, double* min_nfa, int32_t* iterations,
                                    uint32_t* mt_state_out) {
  return acransac_pairs<acrk::HPolicy>(c, n_pairs, offsets, corr, wh, nullptr, mt_state, mt_state_per_pair, max_iteration, precision, valid, n_inliers,
                                       inliers, H, error_max, min_nfa, iterations, mt_state_out);
}

int b200m_acransac_fundamental_spherical_pairs(b200m_ctx* c, int n_pairs, const int64_t* offsets, const double* bearings,
                                               const uint32_t* mt_state, int mt_state_per_pair, int64_t max_iteration, double precision,
                                               uint8_t* valid, int32_t* n_inliers, uint32_t* inliers, double* F, double* error_max,
                                               double* min_nfa, int32_t* iterations, uint32_t* mt_state_out) {
  return acransac_pairs<acrk::SPolicy>(c, n_pairs, offsets, bearings, nullptr, nullptr, mt_state, mt_state_per_pair, max_iteration, precision, valid,
                                       n_inliers, inliers, F, error_max, min_nfa, iterations, mt_state_out);
}

int b200m_acransac_essential_pairs(b200m_ctx* c, int n_pairs, const int64_t* offsets, const double* corr, const int32_t* wh, const double* K,
                                   const uint32_t* mt_state, int mt_state_per_pair, int64_t max_iteration, double precision, uint8_t* valid,
                                   int32_t* n_inliers, uint32_t* inliers, double* E, double* error_max, double* min_nfa, int32_t* iterations,
                                   uint32_t* mt_state_out) {
  return acransac_pairs<acrk::EPolicy>(c, n_pairs, offsets, corr, wh, K, mt_state, mt_state_per_pair, max_iteration, precision, valid,
                                       n_inliers, inliers, E, error_max, min_nfa, iterations, mt_state_out);
}

int b200m_acransac_fundamental_distortion_pairs(b200m_ctx* c, int n_pairs, const int64_t* offsets, const double* corr, const int32_t* wh,
                                                const uint32_t* mt_state, int64_t max_iteration, double precision, uint8_t* valid,
                                                int32_t* n_inliers, uint32_t* inliers, double* F, double* L, double* error_max, double* min_nfa,
                                                int32_t* iterations) {
  return acransac_pairs<acrk::F10Policy>(c, n_pairs, offsets, corr, wh, nullptr, mt_state, 0, max_iteration, precision, valid, n_inliers, inliers,
                                         F, error_max, min_nfa, iterations, nullptr, L);
}

double b200m_acransac_last_stats(const b200m_ctx* c, int64_t stats[4]) {
  if (!c) return 0;
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);   // a concurrent call rewrites them
  if (stats) for (int t = 0; t < 4; ++t) stats[t] = c->acr.stats[t];
  return c->acr.last_ms;
}

int b200m_acransac_last_trace(const b200m_ctx* c, int pair, int32_t* iters, double* nfa, int cap) {
  if (!c) return 0;
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  if (pair < 0 || pair >= (int)c->acr.n_trace.size()) return 0;
  const int n = c->acr.n_trace[pair];
  for (int i = 0; i < std::min({n, cap, acrk::kTraceCap}); ++i) {
    if (iters) iters[i] = c->acr.trace[(size_t)pair * acrk::kTraceCap + i];
    if (nfa) nfa[i] = c->acr.trace_nfa[(size_t)pair * acrk::kTraceCap + i];
  }
  return n;
}

int b200m_ctx_set_acransac_skip(b200m_ctx* c, int on) {
  if (!c) return fail(B200M_ERR_ARG, "bad arguments");
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  c->acr.skip = on != 0;
  return B200M_OK;
}

void b200m_mt19937_seed(uint32_t seed, uint32_t state[625]) {
  acr::Mt19937 g;
  acr::mt_seed(g, seed);
  std::memcpy(state, g.x, sizeof g.x);
  state[624] = (uint32_t)g.p;
}

int b200m_debug_rand_sample_k(const uint32_t state[625], int sample_size, int range, int draws, uint32_t* out, uint32_t* states) {
  if (!state || (sample_size != 4 && sample_size != 7) || range <= sample_size || draws < 0 || (draws > 0 && !out) ||
      state[624] > (uint32_t)acr::kMtN)
    return fail(B200M_ERR_ARG, "bad arguments");
  acr::Mt19937 g;
  std::memcpy(g.x, state, sizeof g.x);
  g.p = (int)state[624];
  for (int d = 0; d < draws; ++d) {
    if (sample_size == 7) acr::rand_sample<7>(g, (uint32_t)range, out + 7 * (size_t)d);
    else acr::rand_sample<4>(g, (uint32_t)range, out + 4 * (size_t)d);
    if (states) { std::memcpy(states + 625 * (size_t)d, g.x, sizeof g.x); states[625 * (size_t)d + 624] = (uint32_t)g.p; }
  }
  return B200M_OK;
}

int b200m_debug_rand_sample(const uint32_t state[625], int range, int draws, uint32_t* out, uint32_t* states) {
  return b200m_debug_rand_sample_k(state, 7, range, draws, out, states);
}

// ---- Surface 2 on several GPUs from ONE process ----------------------------------------------------------------------
// The reference binary is a single process (main_featureMatching.cpp): to use every GPU of the node behind the same
// IImageCollectionMatcher::Match call, the pair list is dealt by database image over one engine context per device
// (SURVEY 8e: independent units, no exchange step, no collective), each driven by its own host thread; only the views
// a shard references are uploaded to its GPU, and the per-device results are merged back in PairSet order.
int b200m_shard_pairs(const uint32_t* pairs, int n_pairs, int n_shards, int32_t* shard_of) {
  if (n_pairs < 0 || n_shards < 1 || (n_pairs > 0 && (!pairs || !shard_of))) return fail(B200M_ERR_ARG, "bad arguments");
  // database images (first index, as ImageCollectionMatcher_generic groups them, .cpp:45-50) in ascending order, dealt round-robin,
  // direction alternating every round so the triangular row lengths of an exhaustive list balance
  std::set<uint32_t> firsts;
  for (int k = 0; k < n_pairs; ++k) firsts.insert(pairs[2 * k]);
  std::unordered_map<uint32_t, int> owner;
  int k = 0;
  for (uint32_t f : firsts) {
    const int rnd = k / n_shards, pos = k % n_shards;
    owner[f] = (rnd % 2 == 0) ? pos : n_shards - 1 - pos;
    ++k;
  }
  for (int p = 0; p < n_pairs; ++p) shard_of[p] = owner[pairs[2 * p]];
  return B200M_OK;
}

// 2-D sharding: what a shard must UPLOAD shrinks with the number of shards.  The view ids (sorted) are dealt cyclically into g
// classes; a pair belongs to the folded block {class(I), class(J)} (g(g+1)/2 blocks: the pair matrix is symmetric in what it needs,
// both views); blocks go to shards heaviest first, each to the least loaded shard, ties to the shard that already holds most of
// the block's classes.  g is chosen per call: the smallest maximum number of classes per shard among the g whose load imbalance is
// within 3 % (else the best balance).  8 shards -> g = 4: six shards own one off-diagonal block (2 of 4 classes = half of the views),
// two own two diagonal blocks each; 4 shards -> 3 of 4 classes at most; 2 shards need every view whatever the split.
int b200m_shard_pairs_2d(const uint32_t* pairs, int n_pairs, int n_shards, int32_t* shard_of) {
  if (n_pairs < 0 || n_shards < 1 || (n_pairs > 0 && (!pairs || !shard_of))) return fail(B200M_ERR_ARG, "bad arguments");
  if (n_pairs == 0) return B200M_OK;
  if (n_shards == 1) { std::fill(shard_of, shard_of + n_pairs, 0); return B200M_OK; }
  std::vector<uint32_t> ids(pairs, pairs + 2 * (size_t)n_pairs);
  std::sort(ids.begin(), ids.end());
  ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
  std::unordered_map<uint32_t, int> pos; pos.reserve(ids.size() * 2);
  for (size_t k = 0; k < ids.size(); ++k) pos[ids[k]] = (int)k;
  struct Plan { int g = 0; double imbalance = 1e30; int max_classes = 1 << 30; std::vector<int> owner; };
  Plan best;
  const int g_max = (int)std::min<size_t>(ids.size(), (size_t)std::max(2, 2 * n_shards));
  for (int g = 1; g <= g_max; ++g) {
    const int nb = g * (g + 1) / 2;
    auto block_of = [&](int a, int b) { if (a > b) std::swap(a, b); return a * g - a * (a - 1) / 2 + (b - a); };
    std::vector<long> weight(nb, 0);
    for (int k = 0; k < n_pairs; ++k) ++weight[block_of(pos[pairs[2 * k]] % g, pos[pairs[2 * k + 1]] % g)];
    std::vector<int> order(nb);
    for (int b = 0; b < nb; ++b) order[b] = b;
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return weight[x] > weight[y]; });
    std::vector<std::pair<int, int>> cls(nb);
    for (int a = 0; a < g; ++a) for (int b = a; b < g; ++b) cls[block_of(a, b)] = {a, b};
    std::vector<long> load(n_shards, 0);
    std::vector<std::vector<char>> has(n_shards, std::vector<char>(g, 0));
    Plan plan; plan.g = g; plan.owner.assign(nb, 0);
    for (int b : order) {
      if (weight[b] == 0) continue;
      int pick = 0; long pl = -1; int padd = 0;
      for (int r = 0; r < n_shards; ++r) {
        const int add = (has[r][cls[b].first] ? 0 : 1) + ((cls[b].second != cls[b].first && !has[r][cls[b].second]) ? 1 : 0);
        // least loaded first (2 % slack so that near-ties are decided by the views a shard already holds)
        const bool better = pl < 0 || load[r] * 100 < pl * 98 || (load[r] * 98 <= pl * 100 && add < padd);
        if (better) { pick = r; pl = load[r]; padd = add; }
      }
      plan.owner[b] = pick; load[pick] += weight[b];
      has[pick][cls[b].first] = 1; has[pick][cls[b].second] = 1;
    }
    long mx = 0, sum = 0; int mc = 0;
    for (int r = 0; r < n_shards; ++r) { mx = std::max(mx, load[r]); sum += load[r]; int cc = 0; for (char h : has[r]) cc += h; mc = std::max(mc, cc); }
    plan.imbalance = (double)mx * n_shards / (double)std::max<long>(sum, 1) - 1.0;
    plan.max_classes = mc;
    // compare on the FRACTION of views a shard needs (max_classes / g), among acceptably balanced plans
    auto frac = [](const Plan& p) { return (double)p.max_classes / p.g; };
    const bool ok = plan.imbalance <= 0.03, best_ok = best.imbalance <= 0.03;
    bool take;
    if (best.g == 0) take = true;
    else if (ok != best_ok) take = ok;
    else if (ok) take = frac(plan) < frac(best) - 1e-9;
    else take = plan.imbalance < best.imbalance - 1e-9;
    if (take) best = plan;
  }
  const int g = best.g;
  auto block_of = [&](int a, int b) { if (a > b) std::swap(a, b); return a * g - a * (a - 1) / 2 + (b - a); };
  for (int k = 0; k < n_pairs; ++k) shard_of[k] = best.owner[block_of(pos[pairs[2 * k]] % g, pos[pairs[2 * k + 1]] % g)];
  return B200M_OK;
}

struct b200m_multi {
  std::vector<b200m_ctx*> ctx;      // owned
  double last_gpu_ms_max = 0;
  ~b200m_multi() { for (auto* c : ctx) b200m_ctx_destroy(c); }
};

int b200m_multi_create(const int* devices, int n_devices, b200m_multi** out) {
  if (!out || n_devices < 1 || !devices) return fail(B200M_ERR_ARG, "bad arguments");
  *out = nullptr;
  std::unique_ptr<b200m_multi> m(new b200m_multi());
  for (int d = 0; d < n_devices; ++d) {
    b200m_ctx* c = nullptr;
    const int rc = b200m_ctx_create(devices[d], nullptr, &c);
    if (rc) return rc;
    m->ctx.push_back(c);
  }
  // the finishing pools share the host: split the threads
  const int ht = std::max(2, (int)std::thread::hardware_concurrency() / n_devices);
  for (auto* c : m->ctx) b200m_ctx_set_host_threads(c, std::min(ht, 32));
  *out = m.release();
  return B200M_OK;
}

void b200m_multi_destroy(b200m_multi* m) { delete m; }

int b200m_multi_num_devices(const b200m_multi* m) { return m ? (int)m->ctx.size() : 0; }
b200m_ctx* b200m_multi_ctx(b200m_multi* m, int k) { return (m && k >= 0 && k < (int)m->ctx.size()) ? m->ctx[k] : nullptr; }
double b200m_multi_last_gpu_ms(const b200m_multi* m) { return m ? m->last_gpu_ms_max : 0; }

int b200m_multi_match(b200m_multi* m, int n_views, const uint32_t* view_ids, const void* const* descs, const int* counts, int dim, int dtype,
                      const float* const* xys, const uint32_t* pairs, int n_pairs, float dist_ratio, int cross, b200m_result** out) {
  if (!m || !out || n_views < 0 || n_pairs < 0 || (n_views > 0 && (!view_ids || !descs || !counts)) || (n_pairs > 0 && !pairs))
    return fail(B200M_ERR_ARG, "bad arguments");
  *out = nullptr;
  const int nd = (int)m->ctx.size();
  std::unordered_map<uint32_t, int> index_of;
  for (int v = 0; v < n_views; ++v) index_of[view_ids[v]] = v;
  for (int p = 0; p < 2 * n_pairs; ++p)
    if (!index_of.count(pairs[p]))
      return fail(B200M_ERR_ARG, "pair references a view that was not given (RegionsPerView::getRegions would throw std::out_of_range)");
  std::vector<int32_t> shard_of(std::max(n_pairs, 1));
  int rc = b200m_shard_pairs_2d(pairs, n_pairs, nd, shard_of.data());
  if (rc) return rc;
  struct Shard { std::vector<uint32_t> pairs; b200m_result* res = nullptr; int rc = B200M_OK; std::string err; };
  std::vector<Shard> sh(nd);
  for (int p = 0; p < n_pairs; ++p) { sh[shard_of[p]].pairs.push_back(pairs[2 * p]); sh[shard_of[p]].pairs.push_back(pairs[2 * p + 1]); }
  auto run = [&](int d) {
    Shard& s = sh[d];
    b200m_ctx* c = m->ctx[d];
    std::vector<uint32_t> ids; std::vector<const void*> dp; std::vector<int> cnt; std::vector<const float*> xp;
    {
      std::set<uint32_t> used(s.pairs.begin(), s.pairs.end());
      for (uint32_t id : used) { const int v = index_of[id]; ids.push_back(id); dp.push_back(descs[v]); cnt.push_back(counts[v]); xp.push_back(xys ? xys[v] : nullptr); }
    }
    s.rc = b200m_clear_views(c);
    if (!s.rc) s.rc = b200m_upload_views_async(c, (int)ids.size(), ids.data(), dp.data(), cnt.data(), dim, dtype, xys ? xp.data() : nullptr);
    if (!s.rc) s.rc = b200m_match_pairs(c, s.pairs.data(), (int)(s.pairs.size() / 2), dist_ratio, cross, B200M_STAGE_FULL, &s.res);
    if (s.rc) s.err = g_err;       // thread-local message of this worker
  };
  std::vector<std::thread> th;
  for (int d = 1; d < nd; ++d) th.emplace_back(run, d);
  run(0);
  for (auto& t : th) t.join();
  m->last_gpu_ms_max = 0;
  for (int d = 0; d < nd; ++d) {
    m->last_gpu_ms_max = std::max(m->last_gpu_ms_max, b200m_last_gpu_ms(m->ctx[d]));
    if (sh[d].rc) {
      const int code = sh[d].rc; const std::string msg = sh[d].err;
      for (auto& s : sh) if (s.res) b200m_result_free(s.res);
      return fail(code, "device " + std::to_string(m->ctx[d]->device) + ": " + msg);
    }
  }
  // merge in PairSet (lexicographic) order: every shard's result is already sorted, and a pair lives in exactly one shard
  struct Ref { uint32_t i, j; int shard; int64_t k; };
  std::vector<Ref> order;
  for (int d = 0; d < nd; ++d) {
    const b200m_result* r = sh[d].res;
    for (size_t k = 0; k + 1 < r->offsets.size(); ++k) order.push_back(Ref{r->pair_ids[2 * k], r->pair_ids[2 * k + 1], d, (int64_t)k});
  }
  std::sort(order.begin(), order.end(), [](const Ref& a, const Ref& b) { return a.i < b.i || (a.i == b.i && a.j < b.j); });
  std::unique_ptr<b200m_result> res(new b200m_result());
  res->offsets.assign(order.size() + 1, 0);
  res->pair_ids.reserve(2 * order.size());
  for (size_t k = 0; k < order.size(); ++k) {
    const b200m_result* r = sh[order[k].shard].res;
    res->pair_ids.push_back(order[k].i); res->pair_ids.push_back(order[k].j);
    res->offsets[k + 1] = res->offsets[k] + (r->offsets[order[k].k + 1] - r->offsets[order[k].k]);
  }
  const size_t total = (size_t)res->offsets[order.size()];
  res->matches.cap = std::max<size_t>(total, 1);
  res->matches.p = static_cast<b200m_match*>(::operator new(res->matches.cap * sizeof(b200m_match)));
  {
    const int nt = (int)std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    auto copy = [&](int t) {
      for (size_t k = (size_t)t; k < order.size(); k += (size_t)nt) {
        const b200m_result* r = sh[order[k].shard].res;
        const int64_t a = r->offsets[order[k].k], b = r->offsets[order[k].k + 1];
        if (b > a) std::memcpy(res->matches.p + res->offsets[k], r->matches.p + a, sizeof(b200m_match) * (size_t)(b - a));
      }
    };
    std::vector<std::thread> ct;
    for (int t = 1; t < nt; ++t) ct.emplace_back(copy, t);
    copy(0);
    for (auto& t : ct) t.join();
  }
  for (auto& s : sh) b200m_result_free(s.res);
  *out = res.release();
  return B200M_OK;
}

// ---- Surface 1: ArrayMatcher ------------------------------------------------------------------------------------
// Build keeps the dataset RESIDENT in the form the tensor-core kernel reads (fp16 copy, half-norm limbs, tensor maps: the same
// preparation as an uploaded view), so SearchNeighbours with NN = 2 on 128-D integer-valued descriptors - what RegionsMatcher<ArrayMatcherT>
// ::Match calls, matching/RegionsMatcher.hpp:140-146 - is one query copy, the preparation kernel, the tensor-core kernel in its MODE_KNN
// (both neighbours' chunks kept, every query emitted) and knn_finalize_kernel, out of grow-only scratch: no allocation, one synchronisation.
int b200m_db_create(b200m_ctx* c, const void* data, int rows, int dim, int dtype, int metric, b200m_db** out) {
  if (!c || !out) return fail(B200M_ERR_ARG, "bad arguments");
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  *out = nullptr;
  if (rows < 1) return fail(B200M_ERR_EMPTY, "Build: nbRows < 1 (ArrayMatcher_bruteForce.hpp:44-48)");
  if (!data || dim < 1 || dtype < 0 || dtype > 2 || metric < 0 || metric > 2) return fail(B200M_ERR_ARG, "bad database arguments");
  if ((metric == B200M_HAMMING) != (dtype == B200M_BIN)) return fail(B200M_ERR_ARG, "Hamming metric needs binary descriptors and vice versa");
  CK(cudaSetDevice(c->device));
  int rc = ensure_batch_buffers(c);
  if (rc) return rc;
  std::unique_ptr<b200m_db> db(new b200m_db());
  db->ctx = c; db->metric = metric;
  ViewHost& v = db->v;
  v.m = rows; v.dim = dim; v.dtype = dtype;
  const size_t esz = dtype == DT_F32 ? 4 : 1;
  if ((rc = alloc_view_buffers(c, v, false))) return rc;
  CK(cudaMemcpyAsync(v.raw, data, (size_t)rows * dim * esz, cudaMemcpyHostToDevice, c->stream));
  if (v.tc_capable()) {
    uint32_t* d_flag = nullptr;
    CK(cudaMallocAsync((void**)&d_flag, 4, c->stream));
    CK(cudaMemsetAsync(d_flag, 0, 4, c->stream));
    if ((rc = run_prep(c, v, d_flag, c->stream))) return rc;
    CK(cudaMemcpyAsync(&v.flags, d_flag, 4, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    cudaFreeAsync(d_flag, c->stream);
    if ((rc = make_view_dev(c, v, db->dev))) return rc;
  } else {
    CK(cudaStreamSynchronize(c->stream));         // `data` is the caller's (pageable) memory
    std::memset(&db->dev, 0, sizeof(db->dev));
    db->dev.raw = v.raw; db->dev.m = v.m; db->dev.dim = v.dim; db->dev.dtype = v.dtype;
  }
  *out = db.release();
  return B200M_OK;
}
void b200m_db_destroy(b200m_db* db) {
  if (!db) return;
  b200m_ctx* c = db->ctx;
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  cudaSetDevice(c->device);
  free_view_buffers(c, db->v);
  cudaStreamSynchronize(c->stream);
  delete db;
}

// grow-only scratch of b200m_knn: the query batch as a prepared view + the small tables and outputs of one call
// (each call ends with a synchronisation: nothing enqueued still uses a buffer that grows)
static int ensure_knn_scratch(b200m_ctx* c, int nq, int dim, size_t esz) {
  KnnScratch& k = c->knn;
  const size_t pad = (size_t)(nq + tc::ROW_PAD - 1) / tc::ROW_PAD * tc::ROW_PAD;
  int rc;
  if ((rc = k.raw.reserve(std::max<size_t>((size_t)nq * dim * esz, 256))) || (rc = k.h16.reserve(pad * 256)) || (rc = k.nbh.reserve(pad * 4)) ||
      (rc = k.nrm.reserve(pad * 4)) || (rc = k.aug16.reserve(pad * 32)) || (rc = k.augq16.reserve(pad * 32)) || (rc = k.err.reserve(pad * 4)) ||
      (rc = k.cands.reserve(sizeof(Cand) * pad)) ||
      (rc = k.idx.reserve(sizeof(int32_t) * 16 * (size_t)nq)) || (rc = k.dist.reserve(sizeof(uint32_t) * 16 * (size_t)nq)) ||   // NN <= 16 on the generic path
      (rc = k.items.reserve(sizeof(WorkItem) * (pad / 256 + 1))) ||
      (rc = k.small.reserve(4096)))                  // stats (16 B) | flag (4 B) | PairDev | 2 x ViewDev (aligned 128)
    return rc;
  return B200M_OK;
}

int b200m_knn(b200m_ctx* c, const b200m_db* db, const void* query, int nq, int nn, int32_t* idx, void* dist) {
  if (!c || !db) return fail(B200M_ERR_ARG, "matcher not built (ArrayMatcher_bruteForce.hpp:100-103)");
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  if (nn < 1 || nn > db->v.m || nq < 1) return fail(B200M_ERR_ARG, "NN > rows or nbQuery < 1 (ArrayMatcher_bruteForce.hpp:105-108)");
  if (nn > GEN_MAX_NN) return fail(B200M_ERR_UNSUPPORTED, "NN > 16 is not supported");
  if (!query || !idx || !dist) return fail(B200M_ERR_ARG, "null buffers");
  CK(cudaSetDevice(c->device));
  int rc = ensure_batch_buffers(c);
  if (rc) return rc;
  const ViewHost& v = db->v;
  const size_t esz = v.dtype == DT_F32 ? 4 : 1;
  if ((rc = ensure_knn_scratch(c, nq, v.dim, esz))) return rc;
  KnnScratch& k = c->knn;
  cudaStream_t st = c->stream;
  CK(cudaMemcpyAsync(k.raw, query, (size_t)nq * v.dim * esz, cudaMemcpyHostToDevice, st));
  uint32_t* d_stats = k.small.as<uint32_t>();
  uint32_t* d_flag = d_stats + 4;
  PairDev* d_pair = reinterpret_cast<PairDev*>(k.small + 64);
  ViewDev* d_views = reinterpret_cast<ViewDev*>(k.small + 128);

  // ---- tensor-core path: the two nearest neighbours of 128-D integer-valued descriptors (any L2 metric: every sum is exact)
  bool done = false;
  if (nn == 2 && v.tc_ok() && !c->force_exact && c->tc_variant == 4 && v.m <= 16 * 0xFFFF) {
    ViewHost qv;
    qv.m = nq; qv.dim = v.dim; qv.dtype = v.dtype; qv.m_pad = (nq + tc::ROW_PAD - 1) / tc::ROW_PAD * tc::ROW_PAD;
    qv.raw = k.raw; qv.h16 = k.h16; qv.nbh = k.nbh; qv.nrm = k.nrm; qv.aug16 = k.aug16; qv.augq16 = k.augq16; qv.err = k.err; qv.stats = d_stats;
    ViewDev hv[2];
    hv[0] = db->dev;
    if ((rc = make_view_dev(c, qv, hv[1]))) return rc;
    CK(cudaMemsetAsync(d_flag, 0, 4, st));
    if ((rc = run_prep(c, qv, d_flag, st))) return rc;
    const int n_items = (nq + 2 * tc::BM - 1) / (2 * tc::BM);
    std::vector<WorkItem> items(n_items);
    for (int t = 0; t < n_items; ++t) items[t] = WorkItem{0u, (uint32_t)t};
    const PairDev hp{0u, 1u, (uint32_t)v.m, (uint32_t)nq, 0u, (uint32_t)PM_TC, 0u};
    CK(cudaMemcpyAsync(d_views, hv, sizeof(hv), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_pair, &hp, sizeof(hp), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(k.items, items.data(), sizeof(WorkItem) * n_items, cudaMemcpyHostToDevice, st));
    const int grid = 2 * std::min(n_items, c->num_sms / 2);
    tc::l2_top2_tc_kernel<true, tc::MODE_KNN><<<grid, tc::block_threads<tc::MODE_KNN>(), tc::Lay<true>::SMEM_BYTES, st>>>(
        d_views, d_pair, k.items, n_items, 2, k.cands, nullptr, 0.f, nullptr, c->d_err, 0, nullptr, FbSink{});
    knn_finalize_kernel<<<(nq + 7) / 8, 256, 0, st>>>(d_views, d_pair, k.cands, k.idx, k.dist.as<float>(), c->d_err);
    CK(cudaGetLastError());
    uint32_t qflags = 0;
    CK(cudaMemcpyAsync(idx, k.idx, sizeof(int32_t) * (size_t)nq * 2, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(dist, k.dist, sizeof(float) * (size_t)nq * 2, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&qflags, d_flag, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&c->err_total, c->d_err, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));               // items / hv / hp are stack objects; results are in the caller's buffers
    done = (qflags & VF_EXACT_MASK) == 0;        // a query batch outside the exact domain (non-integer, huge values): redo on the exact kernels
  }
  if (done) { c->last = LastCall{0, 0, 0, 1, 0, 0, 0, 0}; return B200M_OK; }

  const bool tiled_l2 = nn == 2 && v.dim == 128 && v.dtype != DT_BIN && (v.dtype == DT_U8 || db->metric == B200M_L2_VECTORIZED);
  const bool tiled_ham = nn == 2 && v.dim == 64 && v.dtype == DT_BIN;
  if (tiled_l2 || tiled_ham) {
    ViewDev hv[2]; std::memset(hv, 0, sizeof(hv));
    hv[0].raw = v.raw; hv[0].m = v.m; hv[0].dim = v.dim; hv[0].dtype = v.dtype;
    hv[1].raw = k.raw; hv[1].m = nq; hv[1].dim = v.dim; hv[1].dtype = v.dtype;
    const uint32_t mode = tiled_ham ? PM_HAMMING : (v.dtype == DT_F32 ? PM_EXACT_F32 : PM_EXACT_U8);
    const PairDev hp{0u, 1u, (uint32_t)v.m, (uint32_t)nq, 0u, mode, 0u};
    CK(cudaMemcpyAsync(d_views, hv, sizeof(hv), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_pair, &hp, sizeof(hp), cudaMemcpyHostToDevice, st));
    if (tiled_ham) hamming_top2_kernel<true><<<dim3((nq + HM_TQ - 1) / HM_TQ, 1), HM_TQ, 0, st>>>(d_views, d_pair, nullptr, nullptr, 0.f, k.idx, k.dist);
    else if (v.dtype == DT_F32) exact_top2_kernel<float, true><<<dim3((nq + EX_TQ - 1) / EX_TQ, 1), 256, EX_SMEM, st>>>(d_views, d_pair, mode, nullptr, nullptr, 0.f, k.idx, k.dist.as<float>());
    else exact_top2_kernel<uint8_t, true><<<dim3((nq + EX_TQ - 1) / EX_TQ, 1), 256, EX_SMEM, st>>>(d_views, d_pair, mode, nullptr, nullptr, 0.f, k.idx, k.dist.as<float>());
    CK(cudaGetLastError());
  } else {
    const int grid = (nq + 3) / 4;
    if (v.dtype == DT_F32) generic_knn_kernel<float><<<grid, 128, 0, st>>>((const float*)v.raw, v.m, k.raw.as<const float>(), nq, v.dim, nn, db->metric, k.idx, k.dist);
    else generic_knn_kernel<uint8_t><<<grid, 128, 0, st>>>((const uint8_t*)v.raw, v.m, k.raw.as<const uint8_t>(), nq, v.dim, nn, db->metric, k.idx, k.dist);
    CK(cudaGetLastError());
  }
  CK(cudaMemcpyAsync(idx, k.idx, sizeof(int32_t) * (size_t)nq * nn, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(dist, k.dist, sizeof(uint32_t) * (size_t)nq * nn, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  c->last = LastCall{};
  return B200M_OK;
}

}  // extern "C"

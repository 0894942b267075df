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
#include "hamming.cuh"
#include "l2_exact.cuh"
#include "l2_tc.cuh"
#include "prep.cuh"
#include "verify.cuh"
#include "hostconv.hpp"

#include <pthread.h>
#include <sched.h>

#include <algorithm>
#include <chrono>
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
namespace b200m { int set_error(int code, const std::string& msg) { return fail(code, msg); } }   // for the other translation units of the library
#define CK(call)                                                                                          \
  do {                                                                                                    \
    cudaError_t e_ = (call);                                                                              \
    if (e_ != cudaSuccess) return fail(B200M_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
  } while (0)

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
  float* d_xy = nullptr; uint32_t* d_yrank = nullptr;   // positions + rank of y on the device (device finishing stage, finish.cuh)
  bool failed = false;        // its upload job failed: the device buffers were never filled
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
};

struct UploadJob {
  int n_views = 0, dim = 0; size_t esz = 1;
  std::vector<int> slots; std::vector<const void*> descs; std::vector<int> counts;
  std::shared_ptr<std::vector<int>> bad = std::make_shared<std::vector<int>>();   // per view: the checked f32 -> u8 conversion hit a value it cannot hold
};

struct BatchBuf {
  PairDev* d_pairs = nullptr; WorkItem* d_items = nullptr; Cand* d_cands = nullptr; int* d_count = nullptr; int* d_off = nullptr;
  Rec* d_out = nullptr;
  FinMatch* d_fin = nullptr; int* d_fin_count = nullptr; uint32_t* d_scratch = nullptr;   // device finishing stage (finish.cuh)
  WorkItem* d_items_real = nullptr; WorkItem* h_items_real = nullptr;                     // work items of the real-valued pairs (own launch)
  uint32_t* d_candx = nullptr; uint4* d_fb = nullptr; int* d_fb_count = nullptr;          // fallback lists: d_fb_count = [overflow count, total]
  uint4* d_fb_pair = nullptr; int* d_fb_pair_cnt = nullptr;          // real-valued path: 5th candidate word, fallback list (pair, query)
  PairDev* h_pairs = nullptr; WorkItem* h_items = nullptr; int* h_meta = nullptr; Rec* h_out = nullptr;   // pinned
  cudaEvent_t ev_meta = nullptr, ev_copy = nullptr, ev_tab = nullptr;
};

constexpr int PAIR_CAP = 4096;            // directed pairs per batch
constexpr long CAND_CAP = 4l << 20;       // candidate slots per batch (sum of m_j)
constexpr long ITEM_CAP = CAND_CAP / 64 + PAIR_CAP;
constexpr long SLOT_CAP = 8l << 20;       // database rows per batch (sum of m_i): scratch of the device finishing stage
constexpr int META_INTS = 3 * PAIR_CAP + 3;   // pinned per-batch read-back: counts | offsets (+1) | finishing counts | fallback rows of the real-valued path

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// grow-only device scratch of b200m_knn (Surface 1)
struct KnnScratch {
  int cap = 0; size_t raw_bytes = 0;
  void* raw = nullptr; __half* h16 = nullptr; float* nbh = nullptr; float* nrm = nullptr; __half* aug16 = nullptr; __half* augq16 = nullptr; float* err = nullptr;
  Cand* cands = nullptr; int32_t* idx = nullptr; uint32_t* dist = nullptr; WorkItem* items = nullptr; uint8_t* small = nullptr;
};

struct b200m_ctx {
  int device = 0, num_sms = 148;
  KnnScratch knn;
  cudaStream_t stream = nullptr, copy_stream = nullptr, up_stream = nullptr, tab_stream = nullptr, pack_stream = nullptr;
  bool pipe_streams = true;       // tables / packing+finishing on their own streams (B200M_PIPE_STREAMS=0: everything on the search stream)
  bool own_stream = false;
  EncodeTiledFn encode = nullptr;
  std::deque<ViewHost> views;     // deque: references stay valid while pool tasks (position checks) run
  std::unordered_map<uint32_t, int> slot_of;
  std::vector<int> free_slots;    // slots of removed views (b200m_remove_view), reused by later uploads
  ViewDev* d_views = nullptr; uint32_t* d_flags = nullptr; int view_cap = 0;
  BatchBuf buf[2]; bool bufs_ready = false;
  // upload staging: pageable caller memory -> pinned ring (parallel memcpy on the pool) -> async H2D
  static constexpr int NSTG = 24;
  void* stg[NSTG] = {}; size_t stg_bytes[NSTG] = {}; cudaEvent_t stg_ev[NSTG] = {};
  ViewDev* h_views = nullptr;     // pinned mirror of the device view table (source of the async table updates)
  uint32_t* h_flags = nullptr;    // pinned: per-slot exactness flags, copied back behind each view's preparation kernel
  std::vector<cudaEvent_t> view_ev;   // per slot: recorded on up_stream when the view is complete on the device
  cudaEvent_t ev_alloc = nullptr;     // search stream -> upload stream: the view buffers of the current job are allocated
  // uploader thread (one job at a time, FIFO)
  std::thread up_thread; std::mutex up_mu; std::condition_variable up_cv;
  std::deque<UploadJob> up_jobs; bool up_quit = false; int up_active = 0;
  uint64_t up_issued_seq = 0, next_seq = 0;   // last view whose ready event was recorded / last sequence number handed out
  int up_rc = 0; std::string up_err;
  // the entry points that touch views, batch buffers or the stream serialise on this lock: one context may be shared by
  // several host threads (e.g. IRegionsMatcher adaptors created from an OpenMP region); calls simply queue up
  std::recursive_mutex api_mu;
  unsigned int* d_err = nullptr;
  long long* d_trace = nullptr;   // optional pipeline trace of CTA 0 (debug)
  std::vector<cudaEvent_t> tev;   // search-kernel timing events, reused across calls
  cudaEvent_t ev_start = nullptr, ev_end = nullptr;
  std::unique_ptr<Pool> pool;
  CpuSet cpus;                    // CPUs of the GPU's NUMA node (pool, uploader thread); empty = not pinned
  bool u8_staging = true;         // stage integer-valued fp32 descriptors as uchar (B200M_U8_STAGING=0 disables)
  bool device_finish = true;      // finishing stage on the device for views in general position (B200M_DEVICE_FINISH=0 disables)
  std::shared_ptr<Recycler> recycler = std::make_shared<Recycler>();
  bool force_exact = false;
  bool real_tc = true;            // real-valued fp32 pairs on the tensor-core filter kernel (B200M_REAL_TC=0: exact CUDA-core kernel as in round 1)
  int first_batch_pairs = 16;     // while uploads are in flight: pairs of the first batch (then 2x per batch): how soon the GPU starts (B200M_FIRST_BATCH)
  long real_fused_rows = 6144;    // average database rows per item from which the real-valued re-scoring runs inside the filter kernel
  int tc_variant = 4;             // tensor-core kernel (l2_tc.cuh): 4 (default) = half-norms folded into the GEMM (AUG), 256-query work items;
                                  // half-norms added in the epilogue: 2 = 256-query items, 3 = 128-query items, 1 = 128-query items and
                                  // the stand-alone exactness pass (2-4 re-score in the kernel when the database images are long)
  // last-call instrumentation
  double last_gpu_ms = 0, last_search_ms = 0; int last_launches = 0, last_tc_pairs = 0; int64_t last_records = 0;
  int last_real_pairs = 0; int64_t last_fallback_rows = 0;      // real-valued pairs on the tensor-core filter kernel; queries left to the exact_rows fallback
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
// frees than for its copy): raw | h16 | nbh | nrm | aug16 | augq16 | err | stats | yrank | xy, each 256-byte aligned; stats and yrank are
// adjacent so that one memset zeroes both.
static int alloc_view_buffers(b200m_ctx* c, ViewHost& v) {
  const size_t esz = v.store_dtype() == DT_F32 ? 4 : 1;
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  const bool tcv = v.tc_capable(), pos = !v.xy.empty();
  if (tcv) v.m_pad = (v.m + tc::ROW_PAD - 1) / tc::ROW_PAD * tc::ROW_PAD;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += al(std::max<size_t>(bytes, 1)); return o; };
  const size_t o_raw = take(std::max<size_t>((size_t)v.m * v.dim * esz, 256));
  const size_t o_h16 = tcv ? take((size_t)v.m * 128 * 2) : 0, o_nbh = tcv ? take((size_t)v.m_pad * 4) : 0, o_nrm = tcv ? take((size_t)v.m_pad * 4) : 0;
  const size_t o_aug = tcv ? take((size_t)v.m_pad * 32) : 0, o_augq = tcv ? take((size_t)v.m_pad * 32) : 0, o_err = tcv ? take((size_t)v.m_pad * 4) : 0;
  const size_t o_stats = tcv ? take(16) : 0;
  const size_t o_yrank = pos ? take((size_t)v.m * 4) : 0, o_xy = pos ? take((size_t)v.m * 8) : 0;
  char* base = nullptr;
  CK(cudaMallocAsync((void**)&base, off, c->stream));
  v.arena = base;
  v.raw = base + o_raw;
  if (tcv) {
    v.h16 = (__half*)(base + o_h16); v.nbh = (float*)(base + o_nbh); v.nrm = (float*)(base + o_nrm); v.aug16 = (__half*)(base + o_aug);
    v.augq16 = (__half*)(base + o_augq); v.err = (float*)(base + o_err); v.stats = (uint32_t*)(base + o_stats);
  }
  if (pos) { v.d_yrank = (uint32_t*)(base + o_yrank); v.d_xy = (float*)(base + o_xy); }
  return B200M_OK;
}
static void free_view_buffers(b200m_ctx* c, ViewHost& v) {
  if (v.arena) cudaFreeAsync(v.arena, c->stream);
  if (v.raw_own) cudaFreeAsync(v.raw_own, c->stream);      // fp32 re-upload of a view whose uchar staging failed late
  v.arena = nullptr; v.raw_own = nullptr;
  v.raw = nullptr; v.h16 = nullptr; v.nbh = nullptr; v.nrm = nullptr; v.aug16 = nullptr; v.d_xy = nullptr; v.d_yrank = nullptr;
  v.augq16 = nullptr; v.err = nullptr; v.stats = nullptr;
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
  }
  return B200M_OK;
}

static int run_prep(b200m_ctx* c, const ViewHost& v, uint32_t* d_flag, cudaStream_t st, bool zero_stats = true) {
  (void)c;
  if (!v.tc_capable()) return B200M_OK;
  const int grid = (v.m_pad + 7) / 8;
  if (zero_stats) CK(cudaMemsetAsync(v.stats, 0, 16, st));
  if (v.store_dtype() == DT_F32) prep_view_kernel<float><<<grid, 256, 0, st>>>((const float*)v.raw, v.m, v.h16, v.nbh, v.nrm, v.m_pad, d_flag, v.aug16, v.augq16, v.err, v.stats);
  else prep_view_kernel<uint8_t><<<grid, 256, 0, st>>>((const uint8_t*)v.raw, v.m, v.h16, v.nbh, v.nrm, v.m_pad, d_flag, v.aug16, v.augq16, v.err, v.stats);
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
  ViewDev* nv = nullptr; uint32_t* nf = nullptr; ViewDev* nh = nullptr; uint32_t* nhf = nullptr;
  CK(cudaStreamSynchronize(c->stream));
  CK(cudaStreamSynchronize(c->up_stream));
  CK(cudaMallocHost((void**)&nh, sizeof(ViewDev) * cap));
  if (c->h_views) { std::memcpy(nh, c->h_views, sizeof(ViewDev) * c->view_cap); cudaFreeHost(c->h_views); }
  c->h_views = nh;
  CK(cudaMallocHost((void**)&nhf, sizeof(uint32_t) * cap));
  std::memset(nhf, 0, sizeof(uint32_t) * cap);
  if (c->h_flags) { std::memcpy(nhf, c->h_flags, sizeof(uint32_t) * c->view_cap); cudaFreeHost(c->h_flags); }
  c->h_flags = nhf;
  c->view_ev.resize(cap, nullptr);
  CK(cudaMalloc((void**)&nv, sizeof(ViewDev) * cap));
  CK(cudaMalloc((void**)&nf, sizeof(uint32_t) * cap));
  CK(cudaMemset(nf, 0, sizeof(uint32_t) * cap));
  if (c->d_views) {
    CK(cudaMemcpy(nv, c->d_views, sizeof(ViewDev) * c->view_cap, cudaMemcpyDeviceToDevice));
    CK(cudaMemcpy(nf, c->d_flags, sizeof(uint32_t) * c->view_cap, cudaMemcpyDeviceToDevice));
    cudaFree(c->d_views); cudaFree(c->d_flags);
  }
  c->d_views = nv; c->d_flags = nf; c->view_cap = cap;
  return B200M_OK;
}

static int ensure_batch_buffers(b200m_ctx* c) {
  if (c->bufs_ready) return B200M_OK;
  for (int s = 0; s < 2; ++s) {
    BatchBuf& b = c->buf[s];
    CK(cudaMalloc((void**)&b.d_pairs, sizeof(PairDev) * PAIR_CAP));
    CK(cudaMalloc((void**)&b.d_items, sizeof(WorkItem) * ITEM_CAP));
    CK(cudaMalloc((void**)&b.d_cands, sizeof(Cand) * CAND_CAP));
    CK(cudaMalloc((void**)&b.d_count, sizeof(int) * PAIR_CAP));
    CK(cudaMalloc((void**)&b.d_off, sizeof(int) * (PAIR_CAP + 1)));
    CK(cudaMalloc((void**)&b.d_out, sizeof(Rec) * CAND_CAP));
    CK(cudaMalloc((void**)&b.d_fin, sizeof(FinMatch) * CAND_CAP));
    CK(cudaMalloc((void**)&b.d_fin_count, sizeof(int) * PAIR_CAP));
    CK(cudaMalloc((void**)&b.d_scratch, sizeof(uint32_t) * 2 * SLOT_CAP));
    CK(cudaMalloc((void**)&b.d_items_real, sizeof(WorkItem) * ITEM_CAP));
    CK(cudaMalloc((void**)&b.d_candx, sizeof(uint32_t) * CAND_CAP));
    CK(cudaMalloc((void**)&b.d_fb, sizeof(uint4) * CAND_CAP));
    CK(cudaMalloc((void**)&b.d_fb_count, 2 * sizeof(int)));
    CK(cudaMalloc((void**)&b.d_fb_pair, sizeof(uint4) * (size_t)PAIR_CAP * FB_PER_PAIR));
    CK(cudaMalloc((void**)&b.d_fb_pair_cnt, sizeof(int) * PAIR_CAP));
    CK(cudaMallocHost((void**)&b.h_items_real, sizeof(WorkItem) * ITEM_CAP));
    CK(cudaMallocHost((void**)&b.h_pairs, sizeof(PairDev) * PAIR_CAP));
    CK(cudaMallocHost((void**)&b.h_items, sizeof(WorkItem) * ITEM_CAP));
    CK(cudaMallocHost((void**)&b.h_meta, sizeof(int) * META_INTS));
    CK(cudaMallocHost((void**)&b.h_out, sizeof(Rec) * CAND_CAP));
    CK(cudaEventCreateWithFlags(&b.ev_meta, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&b.ev_copy, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&b.ev_tab, cudaEventDisableTiming));
  }
  CK(cudaFuncSetAttribute(tc::l2_top2_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::Lay<false>::SMEM_BYTES));
  CK(cudaFuncSetAttribute(tc::l2_top2_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::Lay<true>::SMEM_BYTES));
  CK(cudaFuncSetAttribute(tc::l2_top2_tc_kernel<true, tc::MODE_REAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::Lay<true, true>::SMEM_BYTES));
  CK(cudaFuncSetAttribute(tc::l2_top2_tc_kernel<true, tc::MODE_KNN>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::Lay<true>::SMEM_BYTES));
  CK(cudaFuncSetAttribute(exact_rows_pairs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, XP_SMEM));
  CK(cudaFuncSetAttribute(exact_top2_kernel<float, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, EX_SMEM));
  CK(cudaFuncSetAttribute(exact_top2_kernel<uint8_t, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, EX_SMEM));
  CK(cudaFuncSetAttribute(exact_top2_kernel<float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, EX_SMEM));
  CK(cudaFuncSetAttribute(exact_top2_kernel<uint8_t, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, EX_SMEM));
  c->bufs_ready = true;
  return B200M_OK;
}

static cudaEvent_t timing_event(b200m_ctx* c, size_t& used) {
  if (used == c->tev.size()) { cudaEvent_t e; cudaEventCreate(&e); c->tev.push_back(e); }
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
    std::vector<DecoKey> keys; keys.reserve(cnt);
    for (int k = 0; k < cnt; ++k) { const b200m_match& m = out[k]; keys.push_back(DecoKey{xi[2 * m.i], xi[2 * m.i + 1], xj[2 * m.j], xj[2 * m.j + 1], m}); }
    std::set<DecoKey, DecoBefore> st(keys.begin(), keys.end());
    cnt = 0;
    for (const auto& k : st) out[cnt++] = k.m;
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
  if (stream) { c->stream = (cudaStream_t)stream; }
  else { CK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking)); c->own_stream = true; }
  CK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&c->up_stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&c->tab_stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&c->pack_stream, cudaStreamNonBlocking));
  if (const char* e = getenv("B200M_PIPE_STREAMS")) c->pipe_streams = atoi(e) != 0;
  CK(cudaEventCreateWithFlags(&c->ev_alloc, cudaEventDisableTiming));
  cudaDriverEntryPointQueryResult qres;
  void* fn = nullptr;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (!fn || qres != cudaDriverEntryPointSuccess) return fail(B200M_ERR_CUDA, "cuTensorMapEncodeTiled not available in this driver");
  c->encode = (EncodeTiledFn)fn;
  cudaMemPool_t mp;
  CK(cudaDeviceGetDefaultMemPool(&mp, device));
  uint64_t thr = ~0ull;
  CK(cudaMemPoolSetAttribute(mp, cudaMemPoolAttrReleaseThreshold, &thr));
  CK(cudaMalloc((void**)&c->d_err, sizeof(unsigned int)));
  CK(cudaMemset(c->d_err, 0, sizeof(unsigned int)));
  CK(cudaEventCreate(&c->ev_start));
  CK(cudaEventCreate(&c->ev_end));
  c->cpus = numa_cpus_of_device(device);
  int ht = c->cpus.count > 0 ? c->cpus.count : (int)std::thread::hardware_concurrency();
  if (const char* e = getenv("B200M_HOST_THREADS")) ht = std::max(1, atoi(e));     // several engine processes sharing one host (one per GPU)
  c->pool.reset(new Pool(std::min(std::max(ht, 1), 32), c->cpus));
  if (const char* e = getenv("B200M_U8_STAGING")) c->u8_staging = atoi(e) != 0;
  if (const char* e = getenv("B200M_DEVICE_FINISH")) c->device_finish = atoi(e) != 0;
  if (const char* e = getenv("B200M_FIRST_BATCH")) c->first_batch_pairs = std::max(1, atoi(e));
  if (const char* e = getenv("B200M_REAL_TC")) c->real_tc = atoi(e) != 0;
  if (const char* e = getenv("B200M_REAL_FUSED_ROWS")) c->real_fused_rows = std::max(0l, atol(e));
  *out = c.release();
  return B200M_OK;
}

void b200m_ctx_destroy(b200m_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  {
    std::unique_lock<std::mutex> l(c->up_mu);
    c->up_cv.wait(l, [c] { return c->up_active == 0; });
    c->up_quit = true;
  }
  c->up_cv.notify_all();
  if (c->up_thread.joinable()) c->up_thread.join();
  c->pool->wait();
  cudaStreamSynchronize(c->up_stream);
  cudaStreamSynchronize(c->stream);
  for (auto& v : c->views) free_view_buffers(c, v);
  cudaStreamSynchronize(c->stream);
  for (int s = 0; s < 2; ++s) {
    BatchBuf& b = c->buf[s];
    cudaFree(b.d_pairs); cudaFree(b.d_items); cudaFree(b.d_cands); cudaFree(b.d_count); cudaFree(b.d_off); cudaFree(b.d_out);
    cudaFree(b.d_fin); cudaFree(b.d_fin_count); cudaFree(b.d_scratch);
    cudaFree(b.d_items_real); cudaFree(b.d_candx); cudaFree(b.d_fb); cudaFree(b.d_fb_count); cudaFreeHost(b.h_items_real);
    cudaFree(b.d_fb_pair); cudaFree(b.d_fb_pair_cnt);
    cudaFreeHost(b.h_pairs); cudaFreeHost(b.h_items); cudaFreeHost(b.h_meta); cudaFreeHost(b.h_out);
    if (b.ev_meta) cudaEventDestroy(b.ev_meta);
    if (b.ev_copy) cudaEventDestroy(b.ev_copy);
    if (b.ev_tab) cudaEventDestroy(b.ev_tab);
  }
  for (auto& e : c->tev) cudaEventDestroy(e);
  for (int k = 0; k < b200m_ctx::NSTG; ++k) { if (c->stg[k]) cudaFreeHost(c->stg[k]); if (c->stg_ev[k]) cudaEventDestroy(c->stg_ev[k]); }
  if (c->h_views) cudaFreeHost(c->h_views);
  if (c->h_flags) cudaFreeHost(c->h_flags);
  for (auto& e : c->view_ev) if (e) cudaEventDestroy(e);
  cudaEventDestroy(c->ev_alloc);
  cudaStreamDestroy(c->up_stream);
  cudaStreamDestroy(c->tab_stream); cudaStreamDestroy(c->pack_stream);
  if (c->d_trace) cudaFree(c->d_trace);
  cudaFree(c->d_views); cudaFree(c->d_flags); cudaFree(c->d_err);
  {
    KnnScratch& k = c->knn;
    for (void* q : {(void*)k.raw, (void*)k.h16, (void*)k.nbh, (void*)k.nrm, (void*)k.aug16, (void*)k.augq16, (void*)k.err, (void*)k.cands, (void*)k.idx, (void*)k.dist, (void*)k.items, (void*)k.small}) if (q) cudaFree(q);
  }
  cudaEventDestroy(c->ev_start); cudaEventDestroy(c->ev_end);
  cudaStreamDestroy(c->copy_stream);
  if (c->own_stream) cudaStreamDestroy(c->stream);
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
  if (enable && !c->d_trace) { CK(cudaMalloc((void**)&c->d_trace, total * 8)); CK(cudaMemset(c->d_trace, 0, total * 8)); }
  if (out && c->d_trace) { CK(cudaStreamSynchronize(c->stream)); CK(cudaMemcpy(out, c->d_trace, std::min<size_t>(total, (size_t)n) * 8, cudaMemcpyDeviceToHost)); }
  if (!enable && c->d_trace) { cudaFree(c->d_trace); c->d_trace = nullptr; }
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
    if (c->stg_bytes[k] < CH) {
      if (c->stg[k]) { CK(cudaEventSynchronize(c->stg_ev[k])); CK(cudaFreeHost(c->stg[k])); c->stg[k] = nullptr; }
      CK(cudaMallocHost(&c->stg[k], CH)); c->stg_bytes[k] = CH;
    }
    if (!c->stg_ev[k]) CK(cudaEventCreateWithFlags(&c->stg_ev[k], cudaEventDisableTiming));
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
    if (!c->view_ev[slot]) CK(cudaEventCreateWithFlags(&c->view_ev[slot], cudaEventDisableTiming));
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
struct Directed { int slot_i, slot_j; uint32_t mode; int fwd_index; bool reverse; };

static int match_pairs_impl(b200m_ctx* c, const uint32_t* pairs, int n_pairs, float dist_ratio, int cross, int stage, b200m_result** out);

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

static int match_pairs_impl(b200m_ctx* c, const uint32_t* pairs, int n_pairs, float dist_ratio, int cross, int stage, b200m_result** out) {
  if (!c || !out || n_pairs < 0 || (n_pairs > 0 && !pairs) || stage < 0 || stage > 2) return fail(B200M_ERR_ARG, "bad arguments");
  *out = nullptr;
  CK(cudaSetDevice(c->device));
  int rc = ensure_batch_buffers(c);
  if (rc) return rc;
  const bool timing = getenv("B200M_TIMING") != nullptr;
  auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  const double t_begin = now();

  // PairSet semantics (types.hpp:23): unique, lexicographically ordered.
  std::vector<std::pair<uint32_t, uint32_t>> fwd((size_t)n_pairs);
  for (int k = 0; k < n_pairs; ++k) fwd[k] = {pairs[2 * k], pairs[2 * k + 1]};
  if (!std::is_sorted(fwd.begin(), fwd.end())) std::sort(fwd.begin(), fwd.end());
  fwd.erase(std::unique(fwd.begin(), fwd.end()), fwd.end());

  const bool do_cross = cross != 0 && stage == B200M_STAGE_FULL;
  std::vector<Directed> dir;
  dir.reserve(fwd.size() * (do_cross ? 2 : 1));
  int tc_pairs = 0;
  for (size_t k = 0; k < fwd.size(); ++k) {
    auto si = c->slot_of.find(fwd[k].first), sj = c->slot_of.find(fwd[k].second);
    if (si == c->slot_of.end() || sj == c->slot_of.end())
      return fail(B200M_ERR_ARG, "pair references a view that was never uploaded (RegionsPerView::getRegions would throw std::out_of_range)");
    for (int rev = 0; rev < (do_cross ? 2 : 1); ++rev) {
      const int a = rev ? sj->second : si->second, b = rev ? si->second : sj->second;   // a = database, b = query
      const ViewHost& vi = c->views[a]; const ViewHost& vj = c->views[b];
      uint32_t mode;
      if (vi.m == 0 || vj.m == 0 || vi.dtype != vj.dtype || vi.dim != vj.dim) mode = PM_SKIP;           // generic.cpp:59-63,74-78
      else if (vi.m < 2) mode = PM_SKIP;                                                                 // NN=2 > rows: bruteForce.hpp:105
      else if (vi.dtype == DT_BIN) {
        if (vi.dim != 64) return fail(B200M_ERR_UNSUPPORTED, "binary descriptors must be 64 bytes (AKAZE_BinaryRegions)");
        mode = PM_HAMMING;
      } else {
        if (vi.dim != 128) mode = vi.dtype == DT_F32 ? PM_GENERIC_F32 : PM_GENERIC_U8;   // AKAZE float (64), LIOP (144), ...: generic exact path
        else mode = PM_TC;      // provisional: resolved to the tensor-core or an exact kernel once both views' exactness flags are known (enqueue)
      }
      if (stage == B200M_STAGE_FULL && mode != PM_SKIP && (vi.xy.empty() || vj.xy.empty()))
        return fail(B200M_ERR_ARG, "B200M_STAGE_FULL needs feature positions for every matched view");
      dir.push_back(Directed{a, b, mode, (int)k, rev != 0});
    }
  }

  // ---- processing order: PairSet order, or - while uploads are in flight - the order in which the pairs' views arrive
  const size_t step = do_cross ? 2 : 1;
  std::vector<uint32_t> seqv;                      // directed-pair indices in processing order
  bool pending = false;
  {
    std::vector<uint32_t> ord(fwd.size());
    for (size_t k = 0; k < fwd.size(); ++k) ord[k] = (uint32_t)k;
    bool uploading;
    { std::lock_guard<std::mutex> l(c->up_mu); uploading = c->up_active > 0; }
    // arrival-order processing with short first batches only while copies are really in flight (not for views that are merely not yet
    // marked ready after a completed upload)
    if (uploading) for (const Directed& d : dir) if (d.mode != PM_SKIP) pending |= !c->views[d.slot_i].ready || !c->views[d.slot_j].ready;
    if (pending) {
      std::vector<uint64_t> key(fwd.size());
      for (size_t k = 0; k < fwd.size(); ++k) key[k] = std::max(c->views[dir[k * step].slot_i].seq, c->views[dir[k * step].slot_j].seq);
      std::stable_sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
    }
    seqv.reserve(dir.size());
    for (uint32_t k : ord) for (size_t u = 0; u < step; ++u) seqv.push_back((uint32_t)(k * step + u));
  }

  // ---- batching (over the processing order); while views are still arriving the first batches are short so the GPU starts early
  struct Batch { size_t begin, end; };
  std::vector<Batch> batches;
  {
    size_t b0 = 0; long cand = 0, items = 0, slots = 0;
    size_t pair_cap = pending ? (size_t)c->first_batch_pairs : (size_t)PAIR_CAP;
    for (size_t k = 0; k < seqv.size(); k += step) {
      long need_c = 0, need_i = 0, need_s = 0;
      for (size_t u = k; u < k + step; ++u) {
        const int mj = c->views[dir[seqv[u]].slot_j].m, mi = c->views[dir[seqv[u]].slot_i].m;
        if (mj > CAND_CAP || mi > SLOT_CAP / 2) return fail(B200M_ERR_UNSUPPORTED, "view too large for one batch");
        need_c += mj; need_i += (mj + tc::BM - 1) / tc::BM; need_s += mi;
      }
      if (k > b0 && (cand + need_c > CAND_CAP || items + need_i > ITEM_CAP || slots + need_s > SLOT_CAP || k - b0 + step > pair_cap)) {
        batches.push_back({b0, k}); b0 = k; cand = 0; items = 0; slots = 0;
        pair_cap = std::min<size_t>(PAIR_CAP, pair_cap * 2);
      }
      cand += need_c; items += need_i; slots += need_s;
    }
    if (seqv.size() > b0) batches.push_back({b0, seqv.size()});
  }

  const float ratio_sq = dist_ratio * dist_ratio;   // Square(f_dist_ratio) in float, RegionsMatcher.hpp:150 / numeric.hpp:130
  // finishing output: one slot per directed pair in a flat arena (capacity = its record count), filled by pool tasks
  struct ArenaSet {                                                     // uninitialised blocks, one per batch, recycled on exit
    std::vector<Recycler::Block> b; Recycler* r;
    ~ArenaSet() { for (auto& x : b) r->give(x); }
  } arena{std::vector<Recycler::Block>(batches.size()), c->recycler.get()};
  std::vector<b200m_match*> dir_ptr(dir.size(), nullptr);
  std::vector<int> dir_len(dir.size(), 0);
  std::vector<std::unique_ptr<TaskGroup>> groups;
  for (size_t b = 0; b < batches.size(); ++b) groups.emplace_back(new TaskGroup());
  struct WaitGroups {       // every exit path (CUDA error, failed upload ...): the finishing tasks already submitted write into `arena`, `dir_len`
    std::vector<std::unique_ptr<TaskGroup>>& g;             // and signal `groups`; they must be done before those locals are destroyed
    ~WaitGroups() { for (auto& x : g) x->wait(); }
  } wait_groups{groups};
  const bool dev_fin = c->device_finish && stage == B200M_STAGE_FULL;
  size_t tev_used = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> kernel_events;
  int launches = 0;
  int64_t total_records = 0, fallback_rows = 0;
  int real_pairs = 0;
  const bool real_tc = !c->force_exact && c->real_tc && c->tc_variant == 4;

  auto enqueue = [&](size_t bi) -> int {
    const Batch& B = batches[bi];
    BatchBuf& bb = c->buf[bi & 1];
    const int np = (int)(B.end - B.begin);
    uint32_t cbase = 0, sbase = 0; int n_items = 0, n_items_real = 0; int max_qblk_exact = 0, max_qblk_ham = 0;
    // In-kernel exactness pass only when a work item lasts long enough (>= 24 database tiles on average) for two warps to
    // re-score the previous item's candidates behind it; shorter images use the stand-alone exactness kernel.
    // the views of this batch must be complete on the device; their exactness flags decide tensor-core vs exact kernel
    for (int p = 0; p < np; ++p) {
      Directed& d = dir[seqv[B.begin + p]];
      if (d.mode == PM_SKIP) continue;
      int r2;
      if ((r2 = ensure_view_ready(c, d.slot_i)) || (r2 = ensure_view_ready(c, d.slot_j))) return r2;
      if (d.mode == PM_TC) {
        const ViewHost& vi = c->views[d.slot_i]; const ViewHost& vj = c->views[d.slot_j];
        if (!c->force_exact && vi.tc_ok() && vj.tc_ok()) ++tc_pairs;
        else if (real_tc && vi.real_ok() && vj.real_ok()) { d.mode = PM_TC_REAL; ++real_pairs; }   // real-valued fp32: tensor-core filter + exact re-scoring
        else d.mode = vi.dtype == DT_F32 ? PM_EXACT_F32 : PM_EXACT_U8;
      }
    }
    long tc_rows = 0, tc_n = 0, real_rows = 0, real_n = 0;
    for (int p = 0; p < np; ++p) {
      const Directed& d = dir[seqv[B.begin + p]];
      if (d.mode == PM_TC) { tc_rows += c->views[d.slot_i].m; ++tc_n; }
      if (d.mode == PM_TC_REAL) { real_rows += c->views[d.slot_i].m; ++real_n; }
    }
    const bool fused = c->tc_variant >= 2 && tc_n > 0 && tc_rows / tc_n >= 6144;
    const int tc_ctas_per_item = (c->tc_variant == 2 || c->tc_variant == 4) ? 2 : 1;
    const bool fused_real = real_n > 0 && real_rows / real_n >= c->real_fused_rows;
    bool any_f32 = false, any_u8 = false, any_ham = false, any_gf32 = false, any_gu8 = false; int max_qblk_gen = 0;
    for (int p = 0; p < np; ++p) {
      const Directed& d = dir[seqv[B.begin + p]];
      const ViewHost& vi = c->views[d.slot_i]; const ViewHost& vj = c->views[d.slot_j];
      // the CTA-pair kernel runs the exactness pass itself: its candidates are final records
      const uint32_t dev_mode = (d.mode == PM_TC && fused) ? (uint32_t)PM_TC_FUSED : d.mode;
      bb.h_pairs[p] = PairDev{(uint32_t)d.slot_i, (uint32_t)d.slot_j, (uint32_t)vi.m, (uint32_t)vj.m, cbase, dev_mode, sbase};
      cbase += (uint32_t)vj.m; sbase += (uint32_t)vi.m;
      const int qrows = tc_ctas_per_item * tc::BM;   // queries per work item
      if (d.mode == PM_TC) for (int qt = 0; qt < (vj.m + qrows - 1) / qrows; ++qt) bb.h_items[n_items++] = WorkItem{(uint32_t)p, (uint32_t)qt};
      if (d.mode == PM_TC_REAL) for (int qt = 0; qt < (vj.m + 2 * tc::BM - 1) / (2 * tc::BM); ++qt) bb.h_items_real[n_items_real++] = WorkItem{(uint32_t)p, (uint32_t)qt};
      if (d.mode == PM_EXACT_F32) { any_f32 = true; max_qblk_exact = std::max(max_qblk_exact, (vj.m + EX_TQ - 1) / EX_TQ); }
      if (d.mode == PM_EXACT_U8) { any_u8 = true; max_qblk_exact = std::max(max_qblk_exact, (vj.m + EX_TQ - 1) / EX_TQ); }
      if (d.mode == PM_HAMMING) { any_ham = true; max_qblk_ham = std::max(max_qblk_ham, (vj.m + HM_TQ - 1) / HM_TQ); }
      if (d.mode == PM_GENERIC_F32 || d.mode == PM_GENERIC_U8) { (d.mode == PM_GENERIC_F32 ? any_gf32 : any_gu8) = true; max_qblk_gen = std::max(max_qblk_gen, (vj.m + 3) / 4); }
    }
    // Three streams so that consecutive batches' search kernels run back to back: the pair / work-item tables of this batch travel on
    // `tab_stream` (issued while the previous batch is still searching), the packing / finishing kernels and the meta read-back of this
    // batch run on `pack_stream` beside the next batch's search kernel.  Buffer set (bi & 1) is free: the host has seen ev_meta of batch bi-2.
    cudaStream_t ts = c->pipe_streams ? c->tab_stream : c->stream, ps = c->pipe_streams ? c->pack_stream : c->stream;
    CK(cudaMemcpyAsync(bb.d_pairs, bb.h_pairs, sizeof(PairDev) * np, cudaMemcpyHostToDevice, ts));
    if (n_items) CK(cudaMemcpyAsync(bb.d_items, bb.h_items, sizeof(WorkItem) * n_items, cudaMemcpyHostToDevice, ts));
    if (n_items_real) CK(cudaMemcpyAsync(bb.d_items_real, bb.h_items_real, sizeof(WorkItem) * n_items_real, cudaMemcpyHostToDevice, ts));
    CK(cudaMemsetAsync(bb.d_count, 0, sizeof(int) * np, ts));
    CK(cudaMemsetAsync(bb.d_fb_count, 0, 2 * sizeof(int), ts));
    if (n_items_real) CK(cudaMemsetAsync(bb.d_fb_pair_cnt, 0, sizeof(int) * np, ts));
    if (c->pipe_streams) { CK(cudaEventRecord(bb.ev_tab, ts)); CK(cudaStreamWaitEvent(c->stream, bb.ev_tab, 0)); }
    cudaEvent_t k0 = timing_event(c, tev_used), k1 = timing_event(c, tev_used);
    CK(cudaEventRecord(k0, c->stream));
    if (n_items) {
      const int grid = tc_ctas_per_item * std::min(n_items, c->num_sms / tc_ctas_per_item);   // one CTA per SM, whole work items per CTA group
      if (c->tc_variant == 4)
        tc::l2_top2_tc_kernel<true><<<grid, tc::block_threads<tc::MODE_MATCH>(), tc::Lay<true>::SMEM_BYTES, c->stream>>>(c->d_views, bb.d_pairs, bb.d_items, n_items, tc_ctas_per_item, bb.d_cands, bb.d_count, ratio_sq, c->d_trace, c->d_err, (int)fused, nullptr, FbSink{});
      else
        tc::l2_top2_tc_kernel<false><<<grid, tc::block_threads<tc::MODE_MATCH>(), tc::Lay<false>::SMEM_BYTES, c->stream>>>(c->d_views, bb.d_pairs, bb.d_items, n_items, tc_ctas_per_item, bb.d_cands, bb.d_count, ratio_sq, c->d_trace, c->d_err, (int)fused, nullptr, FbSink{});
      ++launches;
    }
    if (n_items_real) {
      // real-valued pairs: filter kernel (re-scoring in-kernel when the items are long enough), stand-alone re-scoring otherwise, then the
      // exact search of the few queries the error bound could not decide; after that their candidates are final like everyone else's
      const int grid = 2 * std::min(n_items_real, c->num_sms / 2);
      const FbSink fbs{bb.d_fb_pair, bb.d_fb_pair_cnt, bb.d_fb, bb.d_fb_count, (int)CAND_CAP, bb.d_fb_count + 1};
      tc::l2_top2_tc_kernel<true, tc::MODE_REAL><<<grid, tc::block_threads<tc::MODE_REAL>(), tc::Lay<true, true>::SMEM_BYTES, c->stream>>>(
          c->d_views, bb.d_pairs, bb.d_items_real, n_items_real, 2, bb.d_cands, bb.d_count, ratio_sq, nullptr, c->d_err, (int)fused_real, bb.d_candx, fbs);
      ++launches;
      if (!fused_real) {
        rescore_real_kernel<<<dim3(np, 4), VERIFY_WARPS_REAL * 32, 0, c->stream>>>(c->d_views, bb.d_pairs, bb.d_cands, bb.d_candx, bb.d_count, ratio_sq, c->d_err, fbs);
        ++launches;
      }
      exact_rows_pairs_kernel<<<dim3(np, FB_PER_PAIR / XP_MAXQ), XP_THREADS, XP_SMEM, c->stream>>>(c->d_views, bb.d_pairs, bb.d_fb_pair, bb.d_fb_pair_cnt, bb.d_cands, bb.d_count, ratio_sq);
      exact_rows_kernel<<<c->num_sms, XR_THREADS, 0, c->stream>>>(c->d_views, bb.d_pairs, bb.d_fb, bb.d_fb_count, (int)CAND_CAP, bb.d_cands, bb.d_count, ratio_sq);   // overflow list: normally empty
      launches += 2;
    }
    if (any_f32) {
      exact_top2_kernel<float, false><<<dim3(max_qblk_exact, np), 256, EX_SMEM, c->stream>>>(c->d_views, bb.d_pairs, PM_EXACT_F32, bb.d_cands, bb.d_count, ratio_sq, nullptr, nullptr);
      ++launches;
    }
    if (any_u8) {
      exact_top2_kernel<uint8_t, false><<<dim3(max_qblk_exact, np), 256, EX_SMEM, c->stream>>>(c->d_views, bb.d_pairs, PM_EXACT_U8, bb.d_cands, bb.d_count, ratio_sq, nullptr, nullptr);
      ++launches;
    }
    if (any_ham) {
      hamming_top2_kernel<false><<<dim3(max_qblk_ham, np), HM_TQ, 0, c->stream>>>(c->d_views, bb.d_pairs, bb.d_cands, bb.d_count, dist_ratio, nullptr, nullptr);
      ++launches;
    }
    if (any_gf32) {
      generic_top2_pairs_kernel<float><<<dim3(max_qblk_gen, np), 128, 0, c->stream>>>(c->d_views, bb.d_pairs, PM_GENERIC_F32, bb.d_cands, bb.d_count, ratio_sq);
      ++launches;
    }
    if (any_gu8) {
      generic_top2_pairs_kernel<uint8_t><<<dim3(max_qblk_gen, np), 128, 0, c->stream>>>(c->d_views, bb.d_pairs, PM_GENERIC_U8, bb.d_cands, bb.d_count, ratio_sq);
      ++launches;
    }
    CK(cudaEventRecord(k1, c->stream));
    if (c->pipe_streams) CK(cudaStreamWaitEvent(ps, k1, 0));
    kernel_events.push_back({k0, k1});
    scan_counts_kernel<<<1, 256, 0, ps>>>(bb.d_count, np, bb.d_off);
    verify_pack_kernel<<<dim3(np, VERIFY_BLOCKS_PER_PAIR), VERIFY_WARPS * 32, 0, ps>>>(c->d_views, bb.d_pairs, bb.d_cands, bb.d_count, bb.d_off, bb.d_out, ratio_sq, c->d_err);
    launches += 2;
    if (dev_fin) {
      finish_pairs_kernel<<<np, FIN_THREADS, 0, ps>>>(c->d_views, bb.d_pairs, c->d_flags, bb.d_out, bb.d_count, bb.d_off, bb.d_scratch, bb.d_fin, bb.d_fin_count);
      ++launches;
      CK(cudaMemcpyAsync(bb.h_meta + 2 * PAIR_CAP + 2, bb.d_fin_count, sizeof(int) * np, cudaMemcpyDeviceToHost, ps));
    }
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(bb.h_meta + 3 * PAIR_CAP + 2, bb.d_fb_count + 1, sizeof(int), cudaMemcpyDeviceToHost, ps));
    CK(cudaMemcpyAsync(bb.h_meta, bb.d_count, sizeof(int) * np, cudaMemcpyDeviceToHost, ps));
    CK(cudaMemcpyAsync(bb.h_meta + PAIR_CAP, bb.d_off, sizeof(int) * (np + 1), cudaMemcpyDeviceToHost, ps));
    CK(cudaEventRecord(bb.ev_meta, ps));
    return B200M_OK;
  };

  const double t_setup = now();
  CK(cudaEventRecord(c->ev_start, c->stream));
  if (stage == B200M_STAGE_DEVICE) {
    for (size_t bi = 0; bi < batches.size(); ++bi) {
      if (bi >= 2) CK(cudaEventSynchronize(c->buf[bi & 1].ev_meta));   // pinned staging of batch bi-2 consumed by its H2D copies
      if ((rc = enqueue(bi))) return rc;
      // totals are read from the pinned meta buffer once the batch is done; accumulate lazily below
      if (bi >= 1) { CK(cudaEventSynchronize(c->buf[(bi - 1) & 1].ev_meta)); const Batch& P = batches[bi - 1]; total_records += c->buf[(bi - 1) & 1].h_meta[PAIR_CAP + (P.end - P.begin)]; fallback_rows += c->buf[(bi - 1) & 1].h_meta[3 * PAIR_CAP + 2]; }
    }
    CK(cudaEventRecord(c->ev_end, c->stream));
    if (!batches.empty()) { const size_t l = batches.size() - 1; CK(cudaEventSynchronize(c->buf[l & 1].ev_meta)); total_records += c->buf[l & 1].h_meta[PAIR_CAP + (batches[l].end - batches[l].begin)]; fallback_rows += c->buf[l & 1].h_meta[3 * PAIR_CAP + 2]; }
  } else {
    if (!batches.empty() && (rc = enqueue(0))) return rc;
    for (size_t bi = 0; bi < batches.size(); ++bi) {
      const Batch& B = batches[bi];
      BatchBuf& bb = c->buf[bi & 1];
      const int np = (int)(B.end - B.begin);
      if (bi + 1 < batches.size()) {
        // buffer set (bi+1)&1 was last used by batch bi-1: its records have been consumed (pool wait below)
        if ((rc = enqueue(bi + 1))) return rc;
      }
      CK(cudaEventSynchronize(bb.ev_meta));
      const int total = bb.h_meta[PAIR_CAP + np];
      fallback_rows += bb.h_meta[3 * PAIR_CAP + 2];
      if (bi >= 2) groups[bi - 2]->wait();       // the tasks of batch bi-2 read this pinned record buffer
      if (total > 0) {
        CK(cudaStreamWaitEvent(c->copy_stream, bb.ev_meta, 0));
        CK(cudaMemcpyAsync(bb.h_out, dev_fin ? (const void*)bb.d_fin : (const void*)bb.d_out, sizeof(Rec) * (size_t)total, cudaMemcpyDeviceToHost, c->copy_stream));
        CK(cudaEventRecord(bb.ev_copy, c->copy_stream));
        CK(cudaEventSynchronize(bb.ev_copy));
      }
      if (bi + 1 == batches.size()) {
        // end of the device work of this call = the last match list has landed in pinned host memory (SURVEY 8d)
        CK(cudaStreamWaitEvent(c->copy_stream, bb.ev_meta, 0));
        CK(cudaEventRecord(c->ev_end, c->copy_stream));
      }
      total_records += total;
      // finishing tasks (one per directed pair) run behind the GPU: they only have to be done before batch bi+2's records
      // are copied into the same pinned buffer.  The per-pair counts/offsets are copied out of the pinned meta block first,
      // because enqueue(bi+2) overwrites it.
      arena.b[bi] = c->recycler->take((size_t)std::max(total, 1));
      TaskGroup* grp = groups[bi].get();
      // one pool task per ~4096 records (or 64 pairs): for small images the task hand-off would otherwise cost more than the work
      // cnt >= 0: raw records, finished here (finish_directed); done >= 0: `done` final matches from the device finishing stage, copied
      struct Job { const Rec* recs; int cnt; int done; b200m_match* dst; int* len; const ViewHost* vi; const ViewHost* vj; bool ham; };
      auto jobs = std::make_shared<std::vector<Job>>();
      long job_records = 0;
      const bool full = stage == B200M_STAGE_FULL;
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
        const size_t di = seqv[B.begin + p];
        const Directed d = dir[di];
        dir_ptr[di] = arena.b[bi].p + bb.h_meta[PAIR_CAP + p];
        int cnt = bb.h_meta[p], done = -1;
        if (d.mode == PM_SKIP || cnt == 0) continue;
        if (dev_fin) {                                   // >= 0: final matches; < 0: -(records + 1) left for the host (view not in general position)
          const int f = bb.h_meta[2 * PAIR_CAP + 2 + p];
          if (f >= 0) done = f; else cnt = -(f + 1);
          if (done == 0) continue;
        }
        jobs->push_back(Job{bb.h_out + bb.h_meta[PAIR_CAP + p], cnt, done, dir_ptr[di], &dir_len[di], &c->views[d.slot_i], &c->views[d.slot_j], d.mode == PM_HAMMING});
        job_records += cnt;
        if (job_records >= 4096 || jobs->size() >= 64) flush();
      }
      flush();
    }
    const double t_loop = now();
    for (auto& g : groups) g->wait();
    if (timing) fprintf(stderr, "[b200m] match_pairs: batch loop %.2f ms, last finishing groups +%.2f ms\n", t_loop - t_setup, now() - t_loop);
    if (batches.empty()) CK(cudaEventRecord(c->ev_end, c->stream));
  }
  const double t_gpu_done = now();
  CK(cudaStreamSynchronize(c->stream));
  CK(cudaStreamSynchronize(c->pack_stream));
  float ms = 0.f;
  CK(cudaEventSynchronize(c->ev_end));
  CK(cudaEventElapsedTime(&ms, c->ev_start, c->ev_end));
  c->last_gpu_ms = ms;
  double sk = 0;
  for (auto& e : kernel_events) { float t = 0.f; CK(cudaEventElapsedTime(&t, e.first, e.second)); sk += t; }
  if (timing && !kernel_events.empty()) {
    // device timeline of the call: search kernels back to back?  gap = end of one batch's search kernels -> start of the next one's
    // (packing / finishing kernels, meta copies, the next batch's pair-table copies, and any wait for the host)
    float lead = 0.f, gaps = 0.f, gmax = 0.f, tail = 0.f;
    CK(cudaEventElapsedTime(&lead, c->ev_start, kernel_events.front().first));
    for (size_t k = 0; k + 1 < kernel_events.size(); ++k) { float t = 0.f; CK(cudaEventElapsedTime(&t, kernel_events[k].second, kernel_events[k + 1].first)); gaps += t; gmax = std::max(gmax, t); }
    CK(cudaEventElapsedTime(&tail, kernel_events.back().second, c->ev_end));
    fprintf(stderr, "[b200m] device timeline: %zu batches, search kernels %.2f ms, lead-in %.2f, gaps between batches %.2f (max %.2f), tail after the last search kernel %.2f ms\n",
            kernel_events.size(), sk, lead, gaps, gmax, tail);
  }
  c->last_search_ms = sk; c->last_launches = launches; c->last_tc_pairs = tc_pairs; c->last_records = total_records;
  c->last_real_pairs = real_pairs; c->last_fallback_rows = fallback_rows;
  unsigned errs = 0;
  CK(cudaMemcpy(&errs, c->d_err, sizeof(unsigned), cudaMemcpyDeviceToHost));
  c->err_total = errs;

  // ---- assemble: offsets first, then the per-pair copies into one contiguous block in parallel on the pool
  std::unique_ptr<b200m_result> res(new b200m_result());
  res->pair_ids.reserve(2 * fwd.size());
  res->offsets.assign(fwd.size() + 1, 0);
  if (stage != B200M_STAGE_DEVICE && do_cross) {
    // keep m iff (m.j, m.i) is in the reverse list (ImageCollectionMatcher_generic.cpp:92-109); filtered in place, in parallel
    TaskGroup g; g.add((int)fwd.size());
    for (size_t k = 0; k < fwd.size(); ++k) {
      b200m_match* f = dir_ptr[k * step]; int* nf = &dir_len[k * step];
      const b200m_match* r = dir_ptr[k * step + 1]; const int nr = dir_len[k * step + 1];
      TaskGroup* gp = &g;
      c->pool->submit([=] {
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
  for (size_t k = 0; k < fwd.size(); ++k) {
    res->pair_ids.push_back(fwd[k].first); res->pair_ids.push_back(fwd[k].second);
    res->offsets[k + 1] = res->offsets[k] + (stage != B200M_STAGE_DEVICE ? dir_len[k * step] : 0);
  }
  const size_t total_matches = (size_t)res->offsets[fwd.size()];
  res->recycler = c->recycler;
  res->matches = c->recycler->take(total_matches);
  if (total_matches) {
    const size_t CHUNK_PAIRS = 64;
    TaskGroup g; g.add((int)((fwd.size() + CHUNK_PAIRS - 1) / CHUNK_PAIRS));
    for (size_t k0 = 0; k0 < fwd.size(); k0 += CHUNK_PAIRS) {
      const size_t k1 = std::min(fwd.size(), k0 + CHUNK_PAIRS);
      b200m_match* base = res->matches.p; const int64_t* offs = res->offsets.data();
      b200m_match* const* dp = dir_ptr.data(); const int* dl = dir_len.data(); TaskGroup* gp = &g;
      c->pool->submit([=] {
        for (size_t k = k0; k < k1; ++k) if (dl[k * step] > 0) std::memcpy(base + offs[k], dp[k * step], sizeof(b200m_match) * (size_t)dl[k * step]);
        gp->done();
      });
    }
    g.wait();
  }
  if (timing) fprintf(stderr, "[b200m] match_pairs n=%d stage=%d: setup %.2f ms, batches %.2f ms (gpu %.2f), tail (cross+assemble) %.2f ms, total %.2f ms\n",
                      n_pairs, stage, t_setup - t_begin, t_gpu_done - t_setup, c->last_gpu_ms, now() - t_gpu_done, now() - t_begin);
  *out = res.release();
  return B200M_OK;
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

double b200m_last_gpu_ms(const b200m_ctx* c) { return c ? c->last_gpu_ms : 0; }
double b200m_last_search_kernel_ms(const b200m_ctx* c) { return c ? c->last_search_ms : 0; }
int b200m_last_launches(const b200m_ctx* c) { return c ? c->last_launches : 0; }
int b200m_last_tc_pairs(const b200m_ctx* c) { return c ? c->last_tc_pairs : 0; }
unsigned b200m_exactness_errors(const b200m_ctx* c) { return c ? c->err_total : 0; }
int64_t b200m_last_records(const b200m_ctx* c) { return c ? c->last_records : 0; }
int b200m_last_real_tc_pairs(const b200m_ctx* c) { return c ? c->last_real_pairs : 0; }
int64_t b200m_last_fallback_rows(const b200m_ctx* c) { return c ? c->last_fallback_rows : 0; }

// ---- guided matching (after the path: GeometricFilterMatrix_F_AC.hpp:363-390 -> matching/guidedMatching.hpp:206-268) ----------------
int b200m_guided_match(b200m_ctx* c, uint32_t view_left, uint32_t view_right, const double* F, double errorTh, double distRatio, b200m_result** out) {
  return b200m_guided_match_model(c, view_left, view_right, B200M_MODEL_FUNDAMENTAL, F, errorTh, distRatio, out);
}

int b200m_guided_match_model(b200m_ctx* c, uint32_t view_left, uint32_t view_right, int model, const double* F, double errorTh, double distRatio,
                             b200m_result** out) {
  if (!c || !out || !F || (model != B200M_MODEL_FUNDAMENTAL && model != B200M_MODEL_HOMOGRAPHY)) return fail(B200M_ERR_ARG, "bad arguments");
  *out = nullptr;
  std::lock_guard<std::recursive_mutex> api_lock(c->api_mu);
  CK(cudaSetDevice(c->device));
  auto sl = c->slot_of.find(view_left), sr = c->slot_of.find(view_right);
  if (sl == c->slot_of.end() || sr == c->slot_of.end()) return fail(B200M_ERR_ARG, "guided matching references a view that was never uploaded");
  int rc;
  if ((rc = ensure_view_ready(c, sl->second)) || (rc = ensure_view_ready(c, sr->second))) return rc;
  if ((rc = wait_uploads(c))) return rc;
  const ViewHost& vl = c->views[sl->second]; const ViewHost& vr = c->views[sr->second];
  std::unique_ptr<b200m_result> res(new b200m_result());
  res->pair_ids = {view_left, view_right};
  res->offsets = {0, 0};
  res->recycler = c->recycler;
  const bool usable = vl.m > 0 && vr.m > 0 && vl.dtype == vr.dtype && vl.dim == vr.dim;      // common descriptor type, :300-306
  if (usable) {
    if (!((vl.dtype == DT_BIN && vl.dim == 64) || (vl.dtype != DT_BIN && vl.dim == 128)))
      return fail(B200M_ERR_UNSUPPORTED, "guided matching takes 128-component scalar or 64-byte binary descriptors");
    if (vl.xy.empty() || vr.xy.empty()) return fail(B200M_ERR_ARG, "guided matching needs feature positions for both views");
    float* d_xy = nullptr; double2* d_xl = nullptr; double2* d_xr = nullptr; Rec* d_out = nullptr; int* d_cnt = nullptr;
    cudaStream_t st = c->stream;
    CK(cudaMallocAsync((void**)&d_xy, sizeof(float) * 2 * (size_t)std::max(vl.m, vr.m), st));
    CK(cudaMallocAsync((void**)&d_xl, sizeof(double2) * (size_t)vl.m, st));
    CK(cudaMallocAsync((void**)&d_xr, sizeof(double2) * (size_t)vr.m, st));
    CK(cudaMallocAsync((void**)&d_out, sizeof(Rec) * (size_t)vl.m, st));
    CK(cudaMallocAsync((void**)&d_cnt, sizeof(int), st));
    CK(cudaMemsetAsync(d_cnt, 0, sizeof(int), st));
    CK(cudaMemcpyAsync(d_xy, vl.xy.data(), sizeof(float) * 2 * (size_t)vl.m, cudaMemcpyHostToDevice, st));
    positions_to_double_kernel<<<(vl.m + 255) / 256, 256, 0, st>>>(d_xy, vl.m, d_xl);
    CK(cudaStreamSynchronize(st));                     // d_xy is reused for the right view
    CK(cudaMemcpyAsync(d_xy, vr.xy.data(), sizeof(float) * 2 * (size_t)vr.m, cudaMemcpyHostToDevice, st));
    positions_to_double_kernel<<<(vr.m + 255) / 256, 256, 0, st>>>(d_xy, vr.m, d_xr);
    GuidedParams P;
    P.model = model == B200M_MODEL_HOMOGRAPHY ? GM_HOMOGRAPHY : GM_FUNDAMENTAL;
    for (int k = 0; k < 9; ++k) P.F[k] = F[k];
    P.errorTh = errorTh; P.distRatio = distRatio;
    const int grid = (vl.m + GM_WARPS - 1) / GM_WARPS;
    CK(cudaEventRecord(c->ev_start, st));
    // integer-valued fp32 views are stored as uchar (same distances: exact integers); a pair of one such view and one real-valued
    // fp32 view gets a temporary fp32 expansion of the former
    const void* rawl = vl.raw; const void* rawr = vr.raw; float* tmp32 = nullptr;
    int kdt = vl.store_dtype();
    if (vl.store_dtype() != vr.store_dtype()) {
      const ViewHost& vu = vl.stored_u8 ? vl : vr;
      const size_t ne = (size_t)vu.m * 128;
      CK(cudaMallocAsync((void**)&tmp32, ne * 4, st));
      u8_to_f32_kernel<<<(unsigned)((ne + 255) / 256), 256, 0, st>>>((const uint8_t*)vu.raw, tmp32, ne);
      (vl.stored_u8 ? rawl : rawr) = tmp32;
      kdt = DT_F32;
    }
    if (kdt == DT_F32) guided_top2_kernel<DT_F32><<<grid, GM_WARPS * 32, 0, st>>>(rawl, rawr, d_xl, d_xr, vl.m, vr.m, P, d_out, d_cnt);
    else if (kdt == DT_U8) guided_top2_kernel<DT_U8><<<grid, GM_WARPS * 32, 0, st>>>(rawl, rawr, d_xl, d_xr, vl.m, vr.m, P, d_out, d_cnt);
    else guided_top2_kernel<DT_BIN><<<grid, GM_WARPS * 32, 0, st>>>(rawl, rawr, d_xl, d_xr, vl.m, vr.m, P, d_out, d_cnt);
    if (tmp32) cudaFreeAsync(tmp32, st);
    CK(cudaGetLastError());
    CK(cudaEventRecord(c->ev_end, st));
    int n = 0;
    CK(cudaMemcpyAsync(&n, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    std::vector<Rec> recs((size_t)n);
    if (n) CK(cudaMemcpy(recs.data(), d_out, sizeof(Rec) * (size_t)n, cudaMemcpyDeviceToHost));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, c->ev_start, c->ev_end));
    c->last_gpu_ms = ms; c->last_search_ms = ms; c->last_launches = 3; c->last_records = n; c->last_tc_pairs = 0;
    cudaFreeAsync(d_xy, st); cudaFreeAsync(d_xl, st); cudaFreeAsync(d_xr, st); cudaFreeAsync(d_out, st); cudaFreeAsync(d_cnt, st);
    // IndMatch::getDeduplicated (guidedMatching.hpp:267): one record per left feature, so this is a sort by (i, j)
    std::sort(recs.begin(), recs.end(), [](const Rec& a, const Rec& b) { return a.i < b.i || (a.i == b.i && a.j < b.j); });
    res->matches = c->recycler->take((size_t)std::max(n, 1));
    for (int k = 0; k < n; ++k) res->matches.p[k] = b200m_match{recs[k].i, recs[k].j, 0.f, 0.f};    // IndMatch(i, j): ratio and distance default to 0
    res->offsets[1] = n;
  } else {
    res->matches = c->recycler->take(1);
  }
  *out = res.release();
  return B200M_OK;
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
  std::vector<b200m_ctx*> ctx;
  double last_gpu_ms_max = 0;
};

int b200m_multi_create(const int* devices, int n_devices, b200m_multi** out) {
  if (!out || n_devices < 1 || !devices) return fail(B200M_ERR_ARG, "bad arguments");
  *out = nullptr;
  std::unique_ptr<b200m_multi> m(new b200m_multi());
  for (int d = 0; d < n_devices; ++d) {
    b200m_ctx* c = nullptr;
    const int rc = b200m_ctx_create(devices[d], nullptr, &c);
    if (rc) { for (auto* x : m->ctx) b200m_ctx_destroy(x); return rc; }
    m->ctx.push_back(c);
  }
  // the finishing pools share the host: split the threads
  const int ht = std::max(2, (int)std::thread::hardware_concurrency() / n_devices);
  for (auto* c : m->ctx) b200m_ctx_set_host_threads(c, std::min(ht, 32));
  *out = m.release();
  return B200M_OK;
}

void b200m_multi_destroy(b200m_multi* m) {
  if (!m) return;
  for (auto* c : m->ctx) b200m_ctx_destroy(c);
  delete m;
}

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
    m->last_gpu_ms_max = std::max(m->last_gpu_ms_max, m->ctx[d]->last_gpu_ms);
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
  if ((rc = alloc_view_buffers(c, v))) return rc;
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
static int ensure_knn_scratch(b200m_ctx* c, int nq, int dim, size_t esz) {
  KnnScratch& k = c->knn;
  const size_t raw_bytes = std::max<size_t>((size_t)nq * dim * esz, 256);
  if (nq <= k.cap && raw_bytes <= k.raw_bytes) return B200M_OK;
  CK(cudaStreamSynchronize(c->stream));
  const int cap = std::max(nq, k.cap * 2);
  const int cap_pad = (cap + tc::ROW_PAD - 1) / tc::ROW_PAD * tc::ROW_PAD;
  const size_t rb = std::max(raw_bytes, (size_t)cap * dim * esz);
  for (void* q : {(void*)k.raw, (void*)k.h16, (void*)k.nbh, (void*)k.nrm, (void*)k.aug16, (void*)k.augq16, (void*)k.err, (void*)k.cands, (void*)k.idx, (void*)k.dist, (void*)k.items}) if (q) cudaFree(q);
  CK(cudaMalloc(&k.raw, rb));
  CK(cudaMalloc((void**)&k.h16, (size_t)cap_pad * 256));
  CK(cudaMalloc((void**)&k.nbh, (size_t)cap_pad * 4));
  CK(cudaMalloc((void**)&k.nrm, (size_t)cap_pad * 4));
  CK(cudaMalloc((void**)&k.aug16, (size_t)cap_pad * 32));
  CK(cudaMalloc((void**)&k.augq16, (size_t)cap_pad * 32));
  CK(cudaMalloc((void**)&k.err, (size_t)cap_pad * 4));
  CK(cudaMalloc((void**)&k.cands, sizeof(Cand) * (size_t)cap_pad));
  CK(cudaMalloc((void**)&k.idx, sizeof(int32_t) * 16 * (size_t)cap));       // NN <= 16 on the generic path
  CK(cudaMalloc((void**)&k.dist, sizeof(uint32_t) * 16 * (size_t)cap));
  CK(cudaMalloc((void**)&k.items, sizeof(WorkItem) * (size_t)(cap_pad / 256 + 1)));
  if (!k.small) CK(cudaMalloc((void**)&k.small, 4096));                        // stats (16 B) | flag (4 B) | PairDev | 2 x ViewDev (aligned 128)
  k.cap = cap; k.raw_bytes = rb;
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
  uint32_t* d_stats = reinterpret_cast<uint32_t*>(k.small);
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
    knn_finalize_kernel<<<(nq + 7) / 8, 256, 0, st>>>(d_views, d_pair, k.cands, k.idx, (float*)k.dist, c->d_err);
    CK(cudaGetLastError());
    uint32_t qflags = 0;
    CK(cudaMemcpyAsync(idx, k.idx, sizeof(int32_t) * (size_t)nq * 2, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(dist, k.dist, sizeof(float) * (size_t)nq * 2, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&qflags, d_flag, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&c->err_total, c->d_err, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));               // items / hv / hp are stack objects; results are in the caller's buffers
    done = (qflags & VF_EXACT_MASK) == 0;        // a query batch outside the exact domain (non-integer, huge values): redo on the exact kernels
    c->last_tc_pairs = done ? 1 : 0;
  }
  if (done) return B200M_OK;
  c->last_tc_pairs = 0;

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
    else if (v.dtype == DT_F32) exact_top2_kernel<float, true><<<dim3((nq + EX_TQ - 1) / EX_TQ, 1), 256, EX_SMEM, st>>>(d_views, d_pair, mode, nullptr, nullptr, 0.f, k.idx, (float*)k.dist);
    else exact_top2_kernel<uint8_t, true><<<dim3((nq + EX_TQ - 1) / EX_TQ, 1), 256, EX_SMEM, st>>>(d_views, d_pair, mode, nullptr, nullptr, 0.f, k.idx, (float*)k.dist);
    CK(cudaGetLastError());
  } else {
    const int grid = (nq + 3) / 4;
    if (v.dtype == DT_F32) generic_knn_kernel<float><<<grid, 128, 0, st>>>((const float*)v.raw, v.m, (const float*)k.raw, nq, v.dim, nn, db->metric, k.idx, k.dist);
    else generic_knn_kernel<uint8_t><<<grid, 128, 0, st>>>((const uint8_t*)v.raw, v.m, (const uint8_t*)k.raw, nq, v.dim, nn, db->metric, k.idx, k.dist);
    CK(cudaGetLastError());
  }
  CK(cudaMemcpyAsync(idx, k.idx, sizeof(int32_t) * (size_t)nq * nn, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(dist, k.dist, sizeof(uint32_t) * (size_t)nq * nn, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return B200M_OK;
}

}  // extern "C"

// Pair-list producer ahead of the matching path (include/b200voc.h): vocabulary-tree quantisation and all-against-all
// document scoring on the GPU, top-N selection and pair-list assembly on the host with the reference's own std containers.
//
// Reference semantics reproduced (file:line relative to src/aliceVision/):
//   voctree/VocabularyTree.hpp:169-196   quantize: per level, children first_child..first_child+k-1 until the first invalid one,
//                                         distance voctree/distance.hpp:24-37 (double; diff = (double)a[i] - (double)b[i];
//                                         result += diff*diff, i ascending), strict '<' keeps the first minimum
//   voctree/VocabularyTree.cpp:22-258     sparseDistance "classic" / "commonPoints" / "strongCommonPoints"
//   voctree/Database.cpp:44-63,118-137,145-157   insert / find (partial_sort on score only) / computeTfIdfWeights
//   imageMatching/ImageMatching.cpp:107-143,191-238   convertAllMatchesToPairList, generateFromVoctree (a/a)
#include "../../include/b200voc.h"
#include "cuda_owner.cuh"

#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

using namespace b200m;

// ------------------------------------------------------------------------------------------------ data model
struct b200v_tree {
  uint32_t k = 0, levels = 0, num_words = 0, word_start = 0; int dim = 0;
  std::vector<float> centers; std::vector<uint8_t> valid;
  // device copies per GPU ordinal (created on first use)
  struct Dev { DeviceBuffer<float> centers; DeviceBuffer<uint8_t> valid; };
  mutable std::map<int, Dev> dev;
};

struct b200v_db {
  const b200v_tree* tree = nullptr; int device = 0;
  Stream stream; Event e0, e1;
  std::map<uint32_t, std::vector<int32_t>> docs;     // doc id -> words in feature order (std::map: ascending id, like database_)
  std::vector<float> word_weights;
  std::vector<int32_t> last_scores; int64_t last_n = 0; double last_gpu_ms = 0;
};

namespace {

bool node_count_ok(uint32_t k, uint32_t levels, uint32_t n_nodes, uint32_t& num_words, uint32_t& word_start) {
  if (k < 1 || levels < 1) return false;
  uint64_t nw = k, ws = 0;                        // VocabularyTree::setNodeCounts (VocabularyTree.hpp:285-296)
  for (uint32_t i = 0; i + 1 < levels; ++i) { ws += nw; nw *= k; if (nw > (1ull << 31)) return false; }
  num_words = (uint32_t)nw; word_start = (uint32_t)ws;
  return (uint64_t)n_nodes == nw + ws;
}

int tree_to_device(const b200v_tree* t, int device, const float** centers, const uint8_t** valid) {
  auto it = t->dev.find(device);
  if (it == t->dev.end()) {
    b200v_tree::Dev d;
    int rc;
    CK(cudaSetDevice(device));
    if ((rc = d.centers.reserve(t->centers.size() * sizeof(float))) || (rc = d.valid.reserve(t->valid.size()))) return rc;
    CK(cudaMemcpy(d.centers, t->centers.data(), t->centers.size() * sizeof(float), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d.valid, t->valid.data(), t->valid.size(), cudaMemcpyHostToDevice));
    it = t->dev.emplace(device, std::move(d)).first;
  }
  *centers = it->second.centers; *valid = it->second.valid;
  return B200M_OK;
}

// ---- K5: tree descent. One warp per descriptor; lane l evaluates children l, l+32, ...; every distance is the
// reference's sequential double-precision sum (separate multiply and add, no contraction), so words are bit-identical.
constexpr int QZ_WARPS = 4;

template <typename T>
__global__ void __launch_bounds__(QZ_WARPS * 32)
quantize_kernel(const T* __restrict__ descs, long long n, int dim, const float* __restrict__ centers, const uint8_t* __restrict__ valid,
                unsigned k, unsigned levels, unsigned word_start, int* __restrict__ words) {
  extern __shared__ double feat_s[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long q = (long long)blockIdx.x * QZ_WARPS + warp;
  if (q >= n) return;
  double* feat = feat_s + (size_t)warp * dim;
  for (int i = lane; i < dim; i += 32) feat[i] = (double)descs[(size_t)q * dim + i];
  __syncwarp();
  int index = -1;
  for (unsigned level = 0; level < levels; ++level) {
    const int first = (index + 1) * (int)k;
    // children after the first invalid one are never looked at (VocabularyTree.hpp:182-183)
    unsigned limit = k;
    for (unsigned base = 0; base < k; base += 32) {
      const unsigned c = base + lane;
      const unsigned inval = __ballot_sync(0xffffffffu, c < k && !valid[first + c]);
      if (inval) { limit = base + (unsigned)__ffs(inval) - 1; break; }
    }
    double best = DBL_MAX; int bestc = first;
    for (unsigned c = lane; c < limit; c += 32) {
      const float* ctr = centers + (size_t)(first + c) * dim;
      double r = 0.0;
      for (int i = 0; i < dim; ++i) {
        const double diff = __dsub_rn(feat[i], (double)ctr[i]);
        r = __dadd_rn(r, __dmul_rn(diff, diff));
      }
      if (r < best) { best = r; bestc = first + (int)c; }            // per lane c ascends: strict '<' keeps the first minimum
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oc = __shfl_xor_sync(0xffffffffu, bestc, o);
      if (ob < best || (ob == best && oc < bestc)) { best = ob; bestc = oc; }
    }
    index = (best < DBL_MAX) ? bestc : first;                         // nothing below numeric_limits::max(): best_child stays first_child
  }
  if (lane == 0) words[q] = index - (int)word_start;
}

// ---- K6: scoring over the inverted file.  Entries are the unique (word, document) pairs sorted by word then document, with
// their multiplicity; one warp per word adds f(count_a, count_b) to S[a][b] and S[b][a] for every pair of its posting list.
__global__ void make_keys_kernel(const int* __restrict__ words, const unsigned* __restrict__ docpos, long long n, unsigned long long* __restrict__ keys) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keys[i] = ((unsigned long long)(unsigned)words[i] << 32) | docpos[i];
}
__global__ void key_words_kernel(const unsigned long long* __restrict__ ukeys, int n, unsigned* __restrict__ w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) w[i] = (unsigned)(ukeys[i] >> 32);
}
// method: 0 = commonPoints (sum of min), 1 = strongCommonPoints (both counts == 1)
__global__ void __launch_bounds__(256)
score_postings_kernel(const unsigned long long* __restrict__ ukeys, const int* __restrict__ counts, const int* __restrict__ list_start,
                      const int* __restrict__ list_len, int n_lists, int method, int n_docs, int* __restrict__ S) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n_lists) return;
  const int s = list_start[w], L = list_len[w];
  for (int i = 0; i < L; ++i) {
    const int ci = counts[s + i];
    if (method == 1 && ci != 1) continue;
    const unsigned di = (unsigned)(ukeys[s + i] & 0xffffffffull);
    for (int j = i + lane; j < L; j += 32) {
      const int cj = counts[s + j];
      const int f = method == 1 ? (cj == 1 ? 1 : 0) : min(ci, cj);
      if (!f) continue;
      const unsigned dj = (unsigned)(ukeys[s + j] & 0xffffffffull);
      atomicAdd(&S[(size_t)di * n_docs + dj], f);
      if (j != i) atomicAdd(&S[(size_t)dj * n_docs + di], f);
    }
  }
}

// ---- K6b: "inversedWeightedCommonPoints" (VocabularyTree.cpp:192-247): score(a, b) = sum over the common words, in ASCENDING word id, of
// (1.f / min(count_a, count_b)) * weight[word] - a float accumulation whose order matters, so every (a, b) is summed by ONE thread that merges the two
// documents' sorted (word, count) lists exactly like the reference's std::map walk (division, multiplication and addition rounded separately).
// Entries: the unique (document, word) pairs sorted by document then word; doc_start[d] .. doc_start[d + 1] is document d's list.
__global__ void doc_keys_kernel(const unsigned long long* __restrict__ ukeys, int n, unsigned long long* __restrict__ dkeys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dkeys[i] = (ukeys[i] << 32) | (ukeys[i] >> 32);            // (word, doc) -> (doc, word)
}
__global__ void doc_starts_kernel(const unsigned long long* __restrict__ dkeys, int n, int n_docs, int* __restrict__ doc_start) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  const int prev = i == 0 ? -1 : (int)(dkeys[i - 1] >> 32);
  const int cur = i == n ? n_docs : (int)(dkeys[i] >> 32);
  for (int d = prev + 1; d <= cur; ++d) doc_start[d] = i;                // documents without words get an empty range
}
__global__ void __launch_bounds__(128)
weighted_pairs_kernel(const unsigned long long* __restrict__ dkeys, const int* __restrict__ dcounts, const int* __restrict__ doc_start,
                      const float* __restrict__ weights, int n_docs, float* __restrict__ S) {
  const int a = blockIdx.y;
  const int b = a + blockIdx.x * blockDim.x + threadIdx.x;               // upper triangle incl. the diagonal
  if (b >= n_docs) return;
  int i = doc_start[a]; const int ie = doc_start[a + 1];
  int j = doc_start[b]; const int je = doc_start[b + 1];
  float score = 0.f;
  while (i < ie && j < je) {
    const unsigned wi = (unsigned)(dkeys[i] & 0xffffffffull), wj = (unsigned)(dkeys[j] & 0xffffffffull);
    if (wj < wi) ++j;
    else if (wi < wj) ++i;
    else {
      const int m = min(dcounts[i], dcounts[j]);
      score = __fadd_rn(score, __fmul_rn(__fdiv_rn(1.f, (float)m), weights[wi]));
      ++i; ++j;
    }
  }
  S[(size_t)a * n_docs + b] = score;
  S[(size_t)b * n_docs + a] = score;
}

int quantize_on(int device, cudaStream_t stream, const b200v_tree* tree, const void* descs, int64_t n, int dtype, int32_t* words) {
  if (n == 0) return B200M_OK;
  const float* dc; const uint8_t* dv;
  int rc = tree_to_device(tree, device, &dc, &dv);
  if (rc) return rc;
  CK(cudaSetDevice(device));
  const size_t esz = dtype == B200M_F32 ? 4 : 1;
  DeviceBuffer<> dd, dw;
  if ((rc = dd.reserve((size_t)n * tree->dim * esz)) || (rc = dw.reserve((size_t)n * 4))) return rc;
  CK(cudaMemcpyAsync(dd, descs, (size_t)n * tree->dim * esz, cudaMemcpyHostToDevice, stream));
  const int grid = (int)((n + QZ_WARPS - 1) / QZ_WARPS);
  const size_t smem = (size_t)QZ_WARPS * tree->dim * sizeof(double);
  if (dtype == B200M_F32)
    quantize_kernel<float><<<grid, QZ_WARPS * 32, smem, stream>>>(dd.as<float>(), n, tree->dim, dc, dv, tree->k, tree->levels, tree->word_start, dw.as<int>());
  else
    quantize_kernel<uint8_t><<<grid, QZ_WARPS * 32, smem, stream>>>(dd.as<uint8_t>(), n, tree->dim, dc, dv, tree->k, tree->levels, tree->word_start, dw.as<int>());
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(words, dw, (size_t)n * 4, cudaMemcpyDeviceToHost, stream));
  CK(cudaStreamSynchronize(stream));
  return B200M_OK;
}

}  // namespace

extern "C" {

// ------------------------------------------------------------------------------------------------ tree
int b200v_tree_create(uint32_t k, uint32_t levels, int dim, const float* centers, const uint8_t* valid, uint32_t n_nodes, b200v_tree** out) {
  if (!out || !centers || !valid || dim < 1 || dim > 1024) return set_error(B200M_ERR_ARG, "bad tree arguments");
  *out = nullptr;
  std::unique_ptr<b200v_tree> t(new b200v_tree());
  if (!node_count_ok(k, levels, n_nodes, t->num_words, t->word_start))
    return set_error(B200M_ERR_ARG, "n_nodes must be k + k^2 + ... + k^levels (VocabularyTree.hpp:283-296)");
  t->k = k; t->levels = levels; t->dim = dim;
  t->centers.assign(centers, centers + (size_t)n_nodes * dim);
  t->valid.assign(valid, valid + n_nodes);
  *out = t.release();
  return B200M_OK;
}

int b200v_tree_load(const char* path, int dim, b200v_tree** out) {
  if (!path || !out || dim < 1 || dim > 1024) return set_error(B200M_ERR_ARG, "bad arguments");
  *out = nullptr;
  std::ifstream in(path, std::ios_base::binary);
  uint32_t k = 0, levels = 0, size = 0;
  if (!in.is_open() || !in.read((char*)&k, 4) || !in.read((char*)&levels, 4) || !in.read((char*)&size, 4))
    return set_error(B200M_ERR_ARG, std::string("Failed to load vocabulary tree file") + path);
  std::vector<float> centers((size_t)size * dim); std::vector<uint8_t> valid(size);
  if (!in.read((char*)centers.data(), centers.size() * sizeof(float)) || !in.read((char*)valid.data(), valid.size()))
    return set_error(B200M_ERR_ARG, std::string("Failed to load vocabulary tree file") + path);
  return b200v_tree_create(k, levels, dim, centers.data(), valid.data(), size, out);
}

int b200v_tree_save(const b200v_tree* t, const char* path) {
  if (!t || !path) return set_error(B200M_ERR_ARG, "bad arguments");
  std::ofstream o(path, std::ios_base::binary);
  if (!o.is_open()) return set_error(B200M_ERR_ARG, std::string("cannot write ") + path);
  const uint32_t size = (uint32_t)t->valid.size();
  o.write((const char*)&t->k, 4); o.write((const char*)&t->levels, 4); o.write((const char*)&size, 4);
  o.write((const char*)t->centers.data(), t->centers.size() * sizeof(float));
  o.write((const char*)t->valid.data(), t->valid.size());
  return o.good() ? B200M_OK : set_error(B200M_ERR_INTERNAL, std::string("write failed: ") + path);
}

void b200v_tree_destroy(b200v_tree* t) {
  if (!t) return;
  for (auto& kv : t->dev) { cudaSetDevice(kv.first); kv.second = b200v_tree::Dev(); }   // each copy is freed on its own device
  delete t;
}
uint32_t b200v_tree_levels(const b200v_tree* t) { return t ? t->levels : 0; }
uint32_t b200v_tree_splits(const b200v_tree* t) { return t ? t->k : 0; }
uint32_t b200v_tree_words(const b200v_tree* t) { return t ? t->num_words : 0; }

int b200v_quantize(int device, const b200v_tree* tree, const void* descs, int64_t n, int dtype, int32_t* words) {
  if (!tree || n < 0 || (n > 0 && (!descs || !words)) || (dtype != B200M_F32 && dtype != B200M_U8)) return set_error(B200M_ERR_ARG, "bad arguments");
  int nd = 0;
  if (cudaGetDeviceCount(&nd) != cudaSuccess || nd == 0) { cudaGetLastError(); return set_error(B200M_ERR_CUDA, "no CUDA device: the quantiser has no CPU path"); }
  if (device < 0 || device >= nd) return set_error(B200M_ERR_ARG, "bad device ordinal");
  return quantize_on(device, nullptr, tree, descs, n, dtype, words);
}

// ------------------------------------------------------------------------------------------------ database
int b200v_db_create(const b200v_tree* tree, int device, b200v_db** out) {
  if (!tree || !out) return set_error(B200M_ERR_ARG, "bad arguments");
  *out = nullptr;
  int nd = 0;
  if (cudaGetDeviceCount(&nd) != cudaSuccess || nd == 0) { cudaGetLastError(); return set_error(B200M_ERR_CUDA, "no CUDA device: the database has no CPU path"); }
  if (device < 0 || device >= nd) return set_error(B200M_ERR_ARG, "bad device ordinal");
  std::unique_ptr<b200v_db> db(new b200v_db());
  db->tree = tree; db->device = device;
  CK(cudaSetDevice(device));
  int rc;
  if ((rc = db->stream.create()) || (rc = db->e0.create()) || (rc = db->e1.create())) return rc;
  db->word_weights.assign(tree->num_words, 1.0f);                 // Database::Database (Database.cpp:39-42)
  *out = db.release();
  return B200M_OK;
}

void b200v_db_destroy(b200v_db* db) {
  if (!db) return;
  cudaSetDevice(db->device);
  delete db;
}

int b200v_db_insert_words(b200v_db* db, uint32_t doc_id, const int32_t* words, int64_t n) {
  if (!db || n < 0 || (n > 0 && !words)) return set_error(B200M_ERR_ARG, "bad arguments");
  if (db->docs.count(doc_id)) return set_error(B200M_ERR_ARG, "document already in the database (Database.cpp:47 asserts)");
  for (int64_t i = 0; i < n; ++i)
    if (words[i] < 0 || (uint32_t)words[i] >= db->tree->num_words) return set_error(B200M_ERR_ARG, "word outside the vocabulary");
  db->docs[doc_id].assign(words, words + n);
  return B200M_OK;
}

int b200v_db_insert_descriptors(b200v_db* db, uint32_t doc_id, const void* descs, int64_t n, int dtype, int64_t nmax) {
  if (!db || n < 0 || (n > 0 && !descs) || (dtype != B200M_F32 && dtype != B200M_U8)) return set_error(B200M_ERR_ARG, "bad arguments");
  if (db->docs.count(doc_id)) return set_error(B200M_ERR_ARG, "document already in the database (Database.cpp:47 asserts)");
  if (nmax > 0) n = std::min(n, nmax);                                 // loadDescsFromBinFile(..., Nmax), Descriptor.hpp:263-266
  std::vector<int32_t> words((size_t)n);
  int rc = quantize_on(db->device, db->stream, db->tree, descs, n, dtype, words.data());
  if (rc) return rc;
  db->docs[doc_id] = std::move(words);
  return B200M_OK;
}

int64_t b200v_db_size(const b200v_db* db) { return db ? (int64_t)db->docs.size() : 0; }

int b200v_db_document(const b200v_db* db, uint32_t doc_id, const int32_t** words, int64_t* n) {
  if (!db) return set_error(B200M_ERR_ARG, "db is null");
  auto it = db->docs.find(doc_id);
  if (it == db->docs.end()) return set_error(B200M_ERR_ARG, "unknown document");
  if (words) *words = it->second.data();
  if (n) *n = (int64_t)it->second.size();
  return B200M_OK;
}

int b200v_db_compute_tfidf(b200v_db* db, float default_weight, float* weights) {
  if (!db) return set_error(B200M_ERR_ARG, "db is null");
  // Ni = number of documents whose inverted file holds word i (Database.cpp:145-157)
  std::vector<uint32_t> ni(db->tree->num_words, 0), stamp(db->tree->num_words, 0xFFFFFFFFu);
  uint32_t d = 0;
  for (auto& kv : db->docs) {                       // one pass: a word counts once per document
    for (int32_t w : kv.second) if (stamp[w] != d) { stamp[w] = d; ++ni[w]; }
    ++d;
  }
  const float N = (float)db->docs.size();
  for (size_t i = 0; i < ni.size(); ++i) {
    const std::size_t Ni = ni[i];
    db->word_weights[i] = Ni != 0 ? std::log(N / Ni) : default_weight;
  }
  if (weights) std::memcpy(weights, db->word_weights.data(), db->word_weights.size() * sizeof(float));
  return B200M_OK;
}

int b200v_db_query_all(b200v_db* db, size_t numImageQuery, const char* distanceMethod, uint32_t* query_ids, uint32_t* match_ids, float* scores,
                       size_t* n_keep_out) {
  if (!db || !distanceMethod) return set_error(B200M_ERR_ARG, "bad arguments");
  const std::string method(distanceMethod);
  int mode;                                        // which statistic the GPU accumulates: 0 / 1 integer counts over the inverted file, 2 the weighted float sum per document pair
  if (method == "strongCommonPoints") mode = 1;
  else if (method == "commonPoints" || method == "classic") mode = 0;
  else if (method == "inversedWeightedCommonPoints") mode = 2;
  else if (method == "weightedStrongCommonPoints")
    return set_error(B200M_ERR_UNSUPPORTED, "distance method " + method + " is not implemented (the reference's own loop for it reads past the end of the histograms, VocabularyTree.cpp:153-171)");
  else return set_error(B200M_ERR_ARG, "distance method " + method + " unknown!");     // std::invalid_argument in the reference (:251-253)
  const size_t n_docs = db->docs.size();
  const size_t n_keep = std::min(numImageQuery == 0 ? n_docs : numImageQuery, n_docs);   // ImageMatching.cpp:198-201, Database.cpp:134
  if (n_keep_out) *n_keep_out = n_keep;
  if (n_docs == 0) return B200M_OK;
  if (!query_ids || !match_ids || !scores) return set_error(B200M_ERR_ARG, "null output");
  CK(cudaSetDevice(db->device));

  // flatten: words of all documents + their position in ascending-id order
  std::vector<uint32_t> ids; ids.reserve(n_docs);
  std::vector<int64_t> nfeat; nfeat.reserve(n_docs);
  size_t total = 0;
  for (auto& kv : db->docs) { ids.push_back(kv.first); nfeat.push_back((int64_t)kv.second.size()); total += kv.second.size(); }
  std::vector<int32_t> flat(total); std::vector<uint32_t> pos(total);
  {
    size_t o = 0; uint32_t d = 0;
    for (auto& kv : db->docs) { std::copy(kv.second.begin(), kv.second.end(), flat.begin() + o); std::fill(pos.begin() + o, pos.begin() + o + kv.second.size(), d); o += kv.second.size(); ++d; }
  }
  db->last_scores.assign(n_docs * n_docs, 0);
  db->last_n = (int64_t)n_docs;
  std::vector<float> wscores;                      // mode 2: the weighted scores (the integer matrix stays zero)
  if (mode == 2) wscores.assign(n_docs * n_docs, 0.f);
  if (total > 0) {
    if (total > 0x7fffffffull) return set_error(B200M_ERR_UNSUPPORTED, "more than 2^31 features in the database");
    const int n = (int)total;
    DeviceBuffer<> d_words, d_pos, d_keys, d_keys2, d_ukeys, d_cnt, d_nu, d_w, d_uw, d_len, d_nw, d_start, d_S, d_tmp;
    int rc;
    if ((rc = d_words.reserve(total * 4)) || (rc = d_pos.reserve(total * 4)) || (rc = d_keys.reserve(total * 8)) || (rc = d_keys2.reserve(total * 8)) ||
        (rc = d_ukeys.reserve(total * 8)) || (rc = d_cnt.reserve(total * 4)) || (rc = d_nu.reserve(4)) || (rc = d_w.reserve(total * 4)) || (rc = d_uw.reserve(total * 4)) ||
        (rc = d_len.reserve(total * 4)) || (rc = d_nw.reserve(4)) || (rc = d_start.reserve(total * 4)) || (rc = d_S.reserve(n_docs * n_docs * 4)))
      return rc;
    cudaStream_t st = db->stream;
    CK(cudaMemcpyAsync(d_words, flat.data(), total * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_pos, pos.data(), total * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(d_S, 0, n_docs * n_docs * 4, st));
    CK(cudaEventRecord(db->e0, st));
    make_keys_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_words.as<int>(), d_pos.as<unsigned>(), n, d_keys.as<unsigned long long>());
    size_t tb = 0, tb2 = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, tb, d_keys.as<unsigned long long>(), d_keys2.as<unsigned long long>(), n, 0, 64, st);
    cub::DeviceRunLengthEncode::Encode(nullptr, tb2, d_keys2.as<unsigned long long>(), d_ukeys.as<unsigned long long>(), d_cnt.as<int>(), d_nu.as<int>(), n, st);
    tb = std::max(tb, tb2);
    cub::DeviceRunLengthEncode::Encode(nullptr, tb2, d_w.as<unsigned>(), d_uw.as<unsigned>(), d_len.as<int>(), d_nw.as<int>(), n, st);
    tb = std::max(tb, tb2);
    cub::DeviceScan::ExclusiveSum(nullptr, tb2, d_len.as<int>(), d_start.as<int>(), n, st);
    tb = std::max(tb, tb2);
    if ((rc = d_tmp.reserve(tb))) return rc;
    CK(cub::DeviceRadixSort::SortKeys(d_tmp, tb, d_keys.as<unsigned long long>(), d_keys2.as<unsigned long long>(), n, 0, 64, st));
    CK(cub::DeviceRunLengthEncode::Encode(d_tmp, tb, d_keys2.as<unsigned long long>(), d_ukeys.as<unsigned long long>(), d_cnt.as<int>(), d_nu.as<int>(), n, st));
    int nu = 0;
    CK(cudaMemcpyAsync(&nu, d_nu, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    key_words_kernel<<<(nu + 255) / 256, 256, 0, st>>>(d_ukeys.as<unsigned long long>(), nu, d_w.as<unsigned>());
    CK(cub::DeviceRunLengthEncode::Encode(d_tmp, tb, d_w.as<unsigned>(), d_uw.as<unsigned>(), d_len.as<int>(), d_nw.as<int>(), nu, st));
    int nw = 0;
    CK(cudaMemcpyAsync(&nw, d_nw, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    CK(cub::DeviceScan::ExclusiveSum(d_tmp, tb, d_len.as<int>(), d_start.as<int>(), nw, st));
    if (mode == 2) {
      // per-document sorted (word, count) lists: re-key the unique pairs by (document, word), sort them with their counts
      DeviceBuffer<> d_dk, d_dk2, d_dc2, d_ds, d_wt, d_tmp2;
      if ((rc = d_dk.reserve((size_t)nu * 8)) || (rc = d_dk2.reserve((size_t)nu * 8)) || (rc = d_dc2.reserve((size_t)nu * 4)) || (rc = d_ds.reserve((n_docs + 2) * 4)) ||
          (rc = d_wt.reserve(db->word_weights.size() * 4)))
        return rc;
      CK(cudaMemcpyAsync(d_wt, db->word_weights.data(), db->word_weights.size() * 4, cudaMemcpyHostToDevice, st));
      doc_keys_kernel<<<(nu + 255) / 256, 256, 0, st>>>(d_ukeys.as<unsigned long long>(), nu, d_dk.as<unsigned long long>());
      size_t tb3 = 0;
      cub::DeviceRadixSort::SortPairs(nullptr, tb3, d_dk.as<unsigned long long>(), d_dk2.as<unsigned long long>(), d_cnt.as<int>(), d_dc2.as<int>(), nu, 0, 64, st);
      if ((rc = d_tmp2.reserve(tb3))) return rc;
      CK(cub::DeviceRadixSort::SortPairs(d_tmp2, tb3, d_dk.as<unsigned long long>(), d_dk2.as<unsigned long long>(), d_cnt.as<int>(), d_dc2.as<int>(), nu, 0, 64, st));
      doc_starts_kernel<<<(nu + 1 + 255) / 256, 256, 0, st>>>(d_dk2.as<unsigned long long>(), nu, (int)n_docs, d_ds.as<int>());
      weighted_pairs_kernel<<<dim3((unsigned)((n_docs + 127) / 128), (unsigned)n_docs), 128, 0, st>>>(d_dk2.as<unsigned long long>(), d_dc2.as<int>(), d_ds.as<int>(), d_wt.as<float>(),
                                                                                                  (int)n_docs, d_S.as<float>());
      CK(cudaGetLastError());
      CK(cudaEventRecord(db->e1, st));
      CK(cudaMemcpyAsync(wscores.data(), d_S, n_docs * n_docs * 4, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
    } else {
    score_postings_kernel<<<(int)(((size_t)nw * 32 + 255) / 256), 256, 0, st>>>(d_ukeys.as<unsigned long long>(), d_cnt.as<int>(), d_start.as<int>(), d_len.as<int>(), nw, mode, (int)n_docs, d_S.as<int>());
    CK(cudaGetLastError());
    CK(cudaEventRecord(db->e1, st));
    CK(cudaMemcpyAsync(db->last_scores.data(), d_S, n_docs * n_docs * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    }
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, db->e0, db->e1));
    db->last_gpu_ms = ms;
  }

  // Database::find per query (Database.cpp:118-137): distances in ascending-id order, partial_sort on the score only
  struct DocMatch { uint32_t id; float score; bool operator<(const DocMatch& o) const { return score < o.score; } };
  std::vector<DocMatch> m(n_docs);
  for (size_t q = 0; q < n_docs; ++q) {
    const int32_t* row = db->last_scores.data() + q * n_docs;
    for (size_t d = 0; d < n_docs; ++d) {
      float dist;
      if (mode == 2) dist = -wscores[q * n_docs + d];                                           // distance = -score, VocabularyTree.cpp:246
      else if (method == "classic") dist = (float)(nfeat[q] + nfeat[d] - 2 * (int64_t)row[d]);     // sum |c1 - c2| = n1 + n2 - 2 sum min(c1, c2); integers < 2^24
      else dist = -(float)row[d];
      m[d] = DocMatch{ids[d], dist};
    }
    std::partial_sort(m.begin(), m.begin() + n_keep, m.end());
    query_ids[q] = ids[q];
    for (size_t r = 0; r < n_keep; ++r) { match_ids[q * n_keep + r] = m[r].id; scores[q * n_keep + r] = m[r].score; }
  }
  return B200M_OK;
}

int b200v_db_last_scores(const b200v_db* db, const int32_t** scores, int64_t* n_docs) {
  if (!db) return set_error(B200M_ERR_ARG, "db is null");
  if (scores) *scores = db->last_scores.data();
  if (n_docs) *n_docs = db->last_n;
  return B200M_OK;
}
double b200v_db_last_gpu_ms(const b200v_db* db) { return db ? db->last_gpu_ms : 0; }

int b200v_convert_matches_to_pairs(const uint32_t* query_ids, const uint32_t* match_ids, size_t n_docs, size_t n_keep, size_t numMatches,
                                   uint32_t* pairs, int64_t cap_pairs, int64_t* n_pairs) {
  if (!n_pairs || (n_docs > 0 && (!query_ids || (n_keep > 0 && !match_ids)))) return set_error(B200M_ERR_ARG, "bad arguments");
  typedef std::size_t ImageID;
  std::map<ImageID, std::vector<ImageID>> allMatches;                         // PairList (ImageMatching.hpp:34)
  for (size_t q = 0; q < n_docs; ++q) {
    std::vector<ImageID>& v = allMatches[query_ids[q]];
    for (size_t r = 0; r < n_keep; ++r) v.push_back(match_ids[q * n_keep + r]);
  }
  std::map<ImageID, std::set<ImageID>> outPairList;                           // OrderedPairList (:37)
  if (numMatches == 0) numMatches = allMatches.size();                        // ImageMatching.cpp:111-112
  for (const auto& match : allMatches) {                                      // :114-142
    const ImageID currImageId = match.first;
    std::set<ImageID> bestMatches;
    for (const ImageID currMatchId : match.second) {
      if (currMatchId == currImageId) continue;
      if (currMatchId < currImageId) {
        auto currMatches = outPairList.find(currMatchId);
        if (currMatches != outPairList.end() && currMatches->second.find(currImageId) == currMatches->second.end()) bestMatches.insert(currMatchId);
      } else {
        bestMatches.insert(currMatchId);
      }
      if (bestMatches.size() == numMatches) break;
    }
    if (!bestMatches.empty()) outPairList[currImageId] = bestMatches;
  }
  int64_t n = 0;
  for (const auto& kv : outPairList)
    for (const ImageID j : kv.second) {
      if (pairs && n < cap_pairs) { pairs[2 * n] = (uint32_t)kv.first; pairs[2 * n + 1] = (uint32_t)j; }
      ++n;
    }
  *n_pairs = n;
  if (pairs && n > cap_pairs) return set_error(B200M_ERR_ARG, "pair buffer too small");
  return B200M_OK;
}

}  // extern "C"

// Graph handle: receiver-sorted CSR (stable counting sort), sender CSR, tensor-core tile table.
// Replaces the edge_index bookkeeping of InteractionNet.__init__ (reference
// neural_lam/gnn_layers.py:73-86) and PyG's per-call index handling.
#include <stdarg.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <numeric>

#include "common.cuh"

namespace nlam {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }
static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int64_t launch_count() { return g_launches.load(std::memory_order_relaxed); }

struct ProfRec {
  const char* name;
  double bytes;
  cudaEvent_t e0, e1;
};
static std::mutex g_prof_mu;
static std::vector<ProfRec> g_prof;
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_pool;
static bool g_prof_on = false;

void prof_begin(const char* name, cudaStream_t st, double bytes) {
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  ProfRec r{name, bytes, nullptr, nullptr};
  if (!g_prof_pool.empty()) {
    r.e0 = g_prof_pool.back().first;
    r.e1 = g_prof_pool.back().second;
    g_prof_pool.pop_back();
  } else if (cudaEventCreate(&r.e0) != cudaSuccess || cudaEventCreate(&r.e1) != cudaSuccess) {
    return;
  }
  cudaEventRecord(r.e0, st);
  g_prof.push_back(r);
}
void prof_end(cudaStream_t st) {
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (!g_prof.empty()) cudaEventRecord(g_prof.back().e1, st);
}

double rowmlp_algorithmic_bytes(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res,
                                const NlamRowSrc* res2, int64_t n_rows, int B, bool out2, const StepEpilogue* ep) {
  double b = 0;
  const void* seen[8];
  int n_seen = 0;
  auto add = [&](const NlamRowSrc* r) {
    if (!r || !r->ptr) return;
    for (int i = 0; i < n_seen; ++i)
      if (seen[i] == r->ptr) return;
    if (n_seen < 8) seen[n_seen++] = r->ptr;
    // gathered sources are counted per output row (upper bound of the distinct rows read)
    b += 4.0 * (double)n_rows * r->dim * ((r->bstride != 0 && B > 1) ? B : 1);
    if (r->idx) b += 4.0 * (double)n_rows;
  };
  for (int s = 0; s < n_src; ++s) add(&srcs[s]);
  add(res);
  add(res2);
  const int nout = mlp->out_dim[mlp->n_linear - 1];
  b += 4.0 * (double)n_rows * nout * B * (out2 ? 2 : 1);
  if (ep) {
    b += 4.0 * (double)n_rows * nout * B;                     // previous state
    if (ep->boundary) b += 4.0 * (double)n_rows * nout * B + 4.0 * (double)n_rows;  // boundary state + mask
  }
  double w = mlp->in_dim;
  for (int l = 0; l < mlp->n_linear; ++l) {
    b += 4.0 * (w * mlp->out_dim[l] + mlp->out_dim[l]);
    w = mlp->out_dim[l];
  }
  return b;
}
}  // namespace nlam

extern "C" void nlam_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(nlam::g_prof_mu);
  for (auto& r : nlam::g_prof) nlam::g_prof_pool.push_back({r.e0, r.e1});
  nlam::g_prof.clear();
  nlam::g_prof_on = on != 0;
}
extern "C" int nlam_profile_count(void) {
  std::lock_guard<std::mutex> lk(nlam::g_prof_mu);
  return (int)nlam::g_prof.size();
}
extern "C" int nlam_profile_get(int i, char* name, int name_cap, float* ms, double* bytes) {
  std::lock_guard<std::mutex> lk(nlam::g_prof_mu);
  NLAM_REQUIRE(i >= 0 && i < (int)nlam::g_prof.size() && name && ms && bytes && name_cap > 0, NLAM_E_INVALID,
               "nlam_profile_get: bad index / null argument");
  const nlam::ProfRec& r = nlam::g_prof[i];
  NLAM_CUDA_OK(cudaEventSynchronize(r.e1));
  NLAM_CUDA_OK(cudaEventElapsedTime(ms, r.e0, r.e1));
  snprintf(name, name_cap, "%s", r.name);
  *bytes = r.bytes;
  return NLAM_OK;
}

using namespace nlam;

extern "C" int nlam_abi_version(void) { return NLAM_ABI_VERSION; }
extern "C" const char* nlam_last_error(void) { return nlam::get_error(); }
extern "C" int64_t nlam_launch_count(void) { return nlam::launch_count(); }
extern "C" const char* nlam_build_info(void) {
  return "libnlam_b200 abi=2 arch=sm_90a cuda=" __DATE__;
}

template <class T>
static int upload(T** dptr, const std::vector<T>& h) {
  size_t bytes = std::max<size_t>(h.size(), 1) * sizeof(T);
  NLAM_CUDA_OK(cudaMalloc((void**)dptr, bytes));
  if (!h.empty()) NLAM_CUDA_OK(cudaMemcpy(*dptr, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  return NLAM_OK;
}

extern "C" int nlam_graph_create(NlamGraph** out, const int64_t* edge_index, int64_t E,
                                 int64_t n_rec_hint, int device) {
  NLAM_REQUIRE(out && edge_index, NLAM_E_INVALID, "nlam_graph_create: null argument");
  NLAM_REQUIRE(E >= 1 && E < (int64_t(1) << 31), NLAM_E_INVALID, "nlam_graph_create: bad edge count %lld", (long long)E);
  const int64_t* snd = edge_index;
  const int64_t* rcv = edge_index + E;
  int64_t max_r = -1, max_s = -1;
  for (int64_t i = 0; i < E; ++i) {
    NLAM_REQUIRE(snd[i] >= 0 && rcv[i] >= 0, NLAM_E_INVALID, "nlam_graph_create: negative index at edge %lld", (long long)i);
    max_r = std::max(max_r, rcv[i]);
    max_s = std::max(max_s, snd[i]);
  }
  NLAM_REQUIRE(max_r < (int64_t(1) << 31) - 1 && max_s < (int64_t(1) << 31) - 1, NLAM_E_INVALID, "index too large");
  int64_t n_rec = std::max(max_r + 1, n_rec_hint);
  int64_t n_send = max_s + 1;

  NlamGraph* g = new NlamGraph();
  g->device = device;
  g->n_edges = E;
  g->n_rec = n_rec;
  g->n_send = n_send;

  // stable counting sort by receiver
  std::vector<int32_t> rowptr(n_rec + 1, 0);
  for (int64_t i = 0; i < E; ++i) rowptr[rcv[i] + 1]++;
  int32_t maxdeg = 0;
  for (int64_t r = 0; r < n_rec; ++r) {
    maxdeg = std::max(maxdeg, rowptr[r + 1]);
    rowptr[r + 1] += rowptr[r];
  }
  std::vector<int32_t> cursor(rowptr.begin(), rowptr.end() - 1);
  std::vector<int32_t> perm(E), inv_perm(E), src(E), dst(E);
  bool sorted = true;
  for (int64_t i = 0; i < E; ++i) {
    int32_t k = cursor[rcv[i]]++;
    perm[k] = (int32_t)i;
    inv_perm[i] = k;
    src[k] = (int32_t)snd[i];
    dst[k] = (int32_t)rcv[i];
    if (k != i) sorted = false;
  }
  g->max_in_degree = maxdeg;
  g->is_sorted = sorted ? 1 : 0;
  {
    bool uniform = maxdeg >= 1 && (int64_t)maxdeg * n_rec == E;
    for (int64_t r = 0; uniform && r < n_rec; ++r) uniform = (rowptr[r + 1] - rowptr[r]) == maxdeg;
    g->uniform_degree = uniform ? maxdeg : 0;
  }

  // sender CSR over CSR-ordered edges (stable): backward of the sender gather
  std::vector<int32_t> sptr(n_send + 1, 0), sperm(E);
  for (int64_t k = 0; k < E; ++k) sptr[src[k] + 1]++;
  for (int64_t s = 0; s < n_send; ++s) sptr[s + 1] += sptr[s];
  {
    std::vector<int32_t> cur(sptr.begin(), sptr.end() - 1);
    for (int64_t k = 0; k < E; ++k) sperm[cur[src[k]]++] = (int32_t)k;
  }

  // tensor-core tile table: whole receivers, <=kTileEdges edges and <=kTileEdges receivers
  std::vector<int32_t> tile_rec, tile_edge;
  if (maxdeg <= kTileEdges) {
    tile_rec.push_back(0);
    int64_t r = 0;
    while (r < n_rec) {
      int64_t r0 = r;
      int32_t e0 = rowptr[r0];
      while (r < n_rec && (r - r0) < kTileEdges && rowptr[r + 1] - e0 <= kTileEdges) ++r;
      tile_rec.push_back((int32_t)r);
    }
    g->n_tiles = (int32_t)tile_rec.size() - 1;
    for (int32_t r : tile_rec) tile_edge.push_back(rowptr[r]);
  }

  int prev_dev = 0;
  cudaError_t e = cudaGetDevice(&prev_dev);
  if (e != cudaSuccess) {
    set_error("nlam_graph_create: cudaGetDevice failed: %s (no CPU fallback)", cudaGetErrorString(e));
    delete g;
    return NLAM_E_CUDA;
  }
  e = cudaSetDevice(device);
  if (e != cudaSuccess) {
    set_error("nlam_graph_create: cudaSetDevice(%d) failed: %s", device, cudaGetErrorString(e));
    delete g;
    return NLAM_E_CUDA;
  }
  int rc = NLAM_OK;
  if ((rc = upload(&g->rowptr, rowptr)) || (rc = upload(&g->src, src)) || (rc = upload(&g->dst, dst)) ||
      (rc = upload(&g->perm, perm)) || (rc = upload(&g->inv_perm, inv_perm)) ||
      (rc = upload(&g->sptr, sptr)) || (rc = upload(&g->sperm, sperm)) ||
      (rc = upload(&g->tile_rec, tile_rec)) || (rc = upload(&g->tile_edge, tile_edge))) {
    cudaSetDevice(prev_dev);
    nlam_graph_destroy(g);
    return rc;
  }
  cudaSetDevice(prev_dev);
  *out = g;
  return NLAM_OK;
}

extern "C" void nlam_graph_destroy(NlamGraph* g) {
  if (!g) return;
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(g->device);
  cudaFree(g->rowptr);
  cudaFree(g->src);
  cudaFree(g->dst);
  cudaFree(g->perm);
  cudaFree(g->inv_perm);
  cudaFree(g->sptr);
  cudaFree(g->sperm);
  cudaFree(g->tile_rec);
  cudaFree(g->tile_edge);
  cudaSetDevice(prev);
  delete g;
}

extern "C" int64_t nlam_graph_num_edges(const NlamGraph* g) { return g->n_edges; }
extern "C" int64_t nlam_graph_num_rec(const NlamGraph* g) { return g->n_rec; }
extern "C" int64_t nlam_graph_num_send(const NlamGraph* g) { return g->n_send; }
extern "C" int32_t nlam_graph_max_in_degree(const NlamGraph* g) { return g->max_in_degree; }
extern "C" int32_t nlam_graph_is_sorted(const NlamGraph* g) { return g->is_sorted; }
extern "C" int32_t nlam_graph_uniform_degree(const NlamGraph* g) { return g->uniform_degree; }
extern "C" const int32_t* nlam_graph_rowptr(const NlamGraph* g) { return g->rowptr; }
extern "C" const int32_t* nlam_graph_src(const NlamGraph* g) { return g->src; }
extern "C" const int32_t* nlam_graph_dst(const NlamGraph* g) { return g->dst; }
extern "C" const int32_t* nlam_graph_perm(const NlamGraph* g) { return g->perm; }
extern "C" const int32_t* nlam_graph_inv_perm(const NlamGraph* g) { return g->inv_perm; }
extern "C" const int32_t* nlam_graph_sptr(const NlamGraph* g) { return g->sptr; }
extern "C" const int32_t* nlam_graph_sperm(const NlamGraph* g) { return g->sperm; }

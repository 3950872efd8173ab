// Shared declarations for libnlam_b200.so (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "nlam_b200.h"

namespace nlam {

// thread-local last-error text (nlam_last_error)
void set_error(const char* fmt, ...);
const char* get_error();

#define NLAM_CUDA_OK(expr)                                                              \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      nlam::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return NLAM_E_CUDA;                                                               \
    }                                                                                   \
  } while (0)

#define NLAM_REQUIRE(cond, code, ...) \
  do {                                \
    if (!(cond)) {                    \
      nlam::set_error(__VA_ARGS__);   \
      return (code);                  \
    }                                 \
  } while (0)

void count_launch(int n = 1);
int64_t launch_count();

// Per-launch profile (nlam_profile_*): when enabled, every kernel launch of the library is bracketed by CUDA events
// on its stream and recorded with its name and its ALGORITHMIC bytes (distinct input bytes + output bytes of that
// launch) — the per-kernel roofline table of bench.py.  Off by default; never enable it inside a stream capture.
void prof_begin(const char* name, cudaStream_t st, double bytes);
void prof_end(cudaStream_t st);
struct ProfScope {
  cudaStream_t st;
  ProfScope(const char* name, cudaStream_t s, double bytes) : st(s) { prof_begin(name, s, bytes); }
  ~ProfScope() { prof_end(st); }
};

constexpr int kTileEdges = 128;  // rows of one tensor-core edge tile

// LayerNorm statistics of one row held by the 4 threads of a quad (lanes 4q .. 4q + 3, as in a wgmma accumulator
// fragment), each with n of the row's 4n values in v.  The mean comes first, summed over the values shifted by the row's
// first value k (quad lane 0's v[0]); then the mean square deviation from it over the same registers.  The one-pass
// E[x²] − μ² cancels catastrophically once |μ| is large against the row's spread (|μ| / σ = 1 000 put x̂ off by about 1);
// this form keeps x̂ at the resolution of the fp32 inputs, and the shift makes μ of a constant row exactly its value, so
// its v − μ is exactly 0.  Every lane of the quad returns the same μ and rstd = 1 / sqrt(var + eps).
template <int n>
__device__ __forceinline__ void quad_row_stats(const float* v, float eps, float& mu, float& rstd) {
  const float k = __shfl_sync(0xffffffffu, v[0], 0, 4);
  float s = 0.f;
#pragma unroll
  for (int t = 0; t < n; ++t) s += v[t] - k;
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  mu = k + s * (1.0f / (4 * n));
  float q = 0.f;
#pragma unroll
  for (int t = 0; t < n; ++t) {
    const float d = v[t] - mu;
    q = fmaf(d, d, q);
  }
  q += __shfl_xor_sync(0xffffffffu, q, 1);
  q += __shfl_xor_sync(0xffffffffu, q, 2);
  rstd = rsqrtf(q * (1.0f / (4 * n)) + eps);
}

struct StepEpilogue {  // fused forecast-step epilogue of a narrow-output row MLP (see TcParams::ep_*)
  const float* prev;
  const float* boundary;
  const float* mask;
  const float* std;
  const float* mean;
  float* std_out = nullptr;  // predicted-std form: the MLP has 2·d outputs, std_out (B, rows, d) = softplus(outputs d..2d-1)
};
// tc7.cu: generic wgmma Linear (any K multiple of 32, N <= 256) and the layer paths built from it
struct LinearCall {
  const float* x0;      // (B|1, n_rows, k0) rows; row pitch x0_pitch (0: dense = k0)
  int64_t x0_bs;
  int k0;
  int64_t x0_pitch;
  const float* x1;      // optional second K block (B|1, n_rows, k1)
  int64_t x1_bs;
  int k1;
  const float* w;       // (n_out, k0 + k1) slice of a row-major matrix with row pitch ldw
  int ldw;
  int w_cols;           // real columns of W (0: k0 + k1); columns past it read as zero (zero-padded inputs)
  int64_t w_bs;         // batch stride of W in elements (0: one W for every batch; != 0: split-K partial products)
  const float* bias;    // optional (n_out)
  int n_out;
  int act;              // 0 none, 1 SiLU
  const float* gamma;   // optional LayerNorm over the n_out columns
  const float* beta;
  float eps;
  const float* add[2];  // optional gathered pre-activation addends: add[i][b, idx[i][r], :]
  const int32_t* add_idx[2];
  int64_t add_bs[2];
  const float* post;    // optional gathered post-epilogue addend
  const int32_t* post_idx;
  int64_t post_bs;
  const float* res;     // optional residual (row r)
  int64_t res_bs;
  int64_t n_rows;
  int B;
  float* out;           // (B, n_rows, n_out)
  float* out2;          // optional: the value before the residual
};
int tc_linear(const LinearCall& c, cudaStream_t st);
bool tc_mlp2_supported(const NlamMlp* m, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res, const NlamRowSrc* res2);
int tc_mlp2(const NlamMlp* m, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res, float* out, int64_t n_rows, int B,
            cudaStream_t st, float* ws);
bool tc_mlp2_packed_supported(const NlamMlp* m, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res, const NlamRowSrc* res2);
size_t tc_mlp2_packed_workspace_floats(const NlamMlp* m, int64_t n_rows, int B);
int tc_mlp2_packed(const NlamMlp* m, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res, float* out, int64_t n_rows, int B,
                   cudaStream_t st, float* ws);
bool tc_inet_gen_supported(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp, int flags, const float* send,
                           int64_t send_bs, const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs);
size_t tc_inet_gen_workspace_floats(const NlamGraph* g, int B, int H);
int tc_inet_gen(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp, const float* send, int64_t send_bs,
                const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs, float* rec_out, float* edge_out,
                float* aggr, int B, int flags, float* ws, cudaStream_t st);
// fused.cu: the grid side of the encoder in one kernel: grid embedder on the concatenated sources, the g2m edge MLP's node
// projections P_s (per batch element) and P_r = mesh·W1rᵀ + b1 (once), and grid_rep = grid_emb + grid_mlp(grid_emb);
// grid_emb itself is stored where grid_emb is not NULL
bool tc_encode_supported(const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src, const NlamMlp* grid_mlp,
                         const NlamMlp* g2m_edge_mlp, const float* mesh, int64_t n_mesh, int64_t n_rows, int B, int flags);
int tc_encode(const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src, const NlamMlp* grid_mlp, const NlamMlp* g2m_edge_mlp,
              const float* mesh, int64_t n_mesh, int64_t n_rows, int B, int flags, float* grid_rep, float* ps, float* pr,
              float* grid_emb, cudaStream_t st, const NlamMlp* g2m_edge_mlp_b = nullptr, float* ps_b = nullptr,
              float* pr_b = nullptr);
// fused.cu: Graph-EFM's latent step in one kernel: prior latent_param_map, reparameterised sample, decoder latent_embedder
bool tc_latent_supported(const NlamMlp* param_mlp, const NlamMlp* embed_mlp, const float* x, int64_t x_bs, const float* eps,
                         int64_t eps_bs, const float* out, int64_t n_rows, int B, int flags);
int tc_latent(const NlamMlp* param_mlp, const NlamMlp* embed_mlp, const float* x, int64_t x_bs, const float* eps, int64_t eps_bs,
              float* out, int64_t n_rows, int B, int flags, cudaStream_t st);
// fused.cu: node update of the mesh->grid layer + output_map + step epilogue in one kernel
bool tc_node_out_supported(const NlamMlp* node_mlp, const NlamMlp* out_mlp, const float* rec, int64_t rec_bs, const float* aggr,
                           int64_t n_rows, int B, const float* out, const StepEpilogue* ep);
int tc_node_out(const NlamMlp* node_mlp, const NlamMlp* out_mlp, const float* rec, int64_t rec_bs, const float* aggr,
                int64_t n_rows, int B, float* out, const StepEpilogue* ep, cudaStream_t st);
// fused.cu: the whole mesh->grid decoder (edge projections + one kernel for edges, aggregation, node update, output_map and
// step epilogue) on a uniform in-degree graph; ws holds tc_decode_workspace_floats floats
bool tc_decode_supported(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* node_mlp, const NlamMlp* out_mlp, int flags,
                         const float* send, int64_t send_bs, const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs,
                         int B, const float* out, const StepEpilogue* ep);
size_t tc_decode_workspace_floats(const NlamGraph* g, int B);
int tc_decode(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* node_mlp, const NlamMlp* out_mlp, int flags,
              const float* send, int64_t send_bs, const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs, int B,
              float* out, const StepEpilogue* ep, float* ws, cudaStream_t st);
// fused.cu: node update + the next layer's node projections in one kernel (stacks of layers over one node set)
bool tc_node_proj_supported(const NlamMlp* node_mlp, const NlamMlp* next_edge_mlp, const float* rec, int64_t rec_bs,
                            const float* aggr, int64_t n_rows, const float* out, const float* proj_out);
int tc_node_proj(const NlamMlp* node_mlp, const NlamMlp* next_edge_mlp, const float* rec, int64_t rec_bs, const float* aggr,
                 int64_t n_rows, int B, float* out, float* proj_out, cudaStream_t st);
// algorithmic bytes of the edge work of one InteractionNet call (SURVEY.md 8d without the node update)
inline double edge_algorithmic_bytes(const NlamGraph* g, int B, int64_t send_bs, int64_t rec_bs, int64_t edge_bs, bool has_out,
                                     int H);
// algorithmic bytes of a row-MLP launch: every distinct source / residual / epilogue input once, the output once
double rowmlp_algorithmic_bytes(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res,
                                const NlamRowSrc* res2, int64_t n_rows, int B, bool out2, const StepEpilogue* ep);
}  // namespace nlam

// Receiver-sorted CSR of one edge set + sender CSR + tensor-core tile table.
struct NlamGraph {
  int device = 0;
  int64_t n_edges = 0, n_rec = 0, n_send = 0;
  int32_t max_in_degree = 0;
  int32_t is_sorted = 0;
  int32_t uniform_degree = 0;   // d if every receiver has exactly d incoming edges (E = d * n_rec), else 0
  // device arrays (int32)
  int32_t* rowptr = nullptr;    // n_rec+1
  int32_t* src = nullptr;       // E, sender of CSR edge k
  int32_t* dst = nullptr;       // E, receiver of CSR edge k
  int32_t* perm = nullptr;      // E, original edge id of CSR edge k
  int32_t* inv_perm = nullptr;  // E
  int32_t* sptr = nullptr;      // n_send+1
  int32_t* sperm = nullptr;     // E
  // tensor-core tiles: whole receivers packed into <=128-edge tiles.
  // tile t covers receivers [tile_rec[t], tile_rec[t+1]) and edges
  // [rowptr[tile_rec[t]], rowptr[tile_rec[t+1]]).  n_tiles == 0 if some in-degree > 128.
  int32_t n_tiles = 0;
  int32_t* tile_rec = nullptr;  // n_tiles+1
  int32_t* tile_edge = nullptr; // n_tiles+1: rowptr[tile_rec[t]], the first CSR edge of tile t
};

namespace nlam {
inline double edge_algorithmic_bytes(const NlamGraph* g, int B, int64_t send_bs, int64_t rec_bs, int64_t edge_bs, bool has_out,
                                     int H) {
  const double row = 4.0 * H;
  const int Bs = (send_bs != 0 && B > 1) ? B : 1, Br = (rec_bs != 0 && B > 1) ? B : 1, Be = (edge_bs != 0 && B > 1) ? B : 1;
  return row * ((double)g->n_edges * Be + (double)g->n_send * Bs + (double)g->n_rec * Br + (double)g->n_rec * B +
                (has_out ? (double)g->n_edges * B : 0.0)) +
         4.0 * g->n_edges + 4.0 * (g->n_rec + 1) + 4.0 * (4.0 * H * H + 5.0 * H);
}

// ensemble.cu: ensemble mean / spread per point and interior-mean scores of K members (nlam_ensemble_stats)
size_t ens_stats_workspace_bytes(int B, int64_t G, int d);
int ens_stats(const float* x, int64_t x_bs, int64_t x_ks, int B, int K, int64_t G, int d, const float* y, int64_t y_bs,
              const float* interior, float* mean, float* std, float* scores, void* ws, size_t ws_bytes, cudaStream_t st);
int ens_stats_bwd(const float* x, int64_t x_bs, int64_t x_ks, int B, int K, int64_t G, int d, const float* y, int64_t y_bs,
                  const float* interior, const float* gup, float* grad, cudaStream_t st);

// simt.cu
int rowmlp_simt(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res,
                const NlamRowSrc* res2, float* out, float* out2, int64_t n_rows, int B,
                cudaStream_t stream);
// fused.cu
bool tc_rowmlp_supported(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res,
                         const NlamRowSrc* res2, int64_t n_rows);
int tc_rowmlp(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res,
              float* out, int64_t n_rows, int B, cudaStream_t stream, const StepEpilogue* ep = nullptr);
// H = 64 edge stage of an InteractionNet call.  tc_edge_path decides which form and launch label the call takes (the rules
// are listed at its definition); label NULL: the H = 64 edge kernels do not cover the call.
struct TcEdgePath {
  const char* label = nullptr;
  bool split = false;       // split first Linear: node projections + K = 64 edge GEMM (tc_edge_split); else K = 192 (tc_edge)
  bool reads_proj = false;  // the split form can take projections an earlier kernel computed (proj_in) instead of its own pass
};
TcEdgePath tc_edge_path(const NlamGraph* g, const NlamMlp* edge_mlp, int flags, const float* send, int64_t send_bs,
                        const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs, const float* edge_out, int B);
// ws: [P_s | P_r], tc_edge_split_workspace_floats floats; have_proj: filled by an earlier kernel (tc_node_proj, tc_encode)
size_t tc_edge_split_workspace_floats(const NlamGraph* g, int B);
int tc_edge_split(const NlamGraph* g, const NlamMlp* edge_mlp, const float* send, int64_t send_bs, const float* rec,
                  int64_t rec_bs, const float* edge, int64_t edge_bs, float* edge_out, float* aggr_out, int B, int flags,
                  cudaStream_t stream, float* ws, bool have_proj, const char* label);
int tc_edge(const NlamGraph* g, const NlamMlp* edge_mlp, const float* send, int64_t send_bs,
            const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs, float* edge_out,
            float* aggr_out, int B, int flags, cudaStream_t stream);
}  // namespace nlam

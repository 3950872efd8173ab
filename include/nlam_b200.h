/*
 * nlam_b200.h — C ABI of libnlam_b200.so: H100 (sm_90a) kernels for the Neural-LAM
 * InteractionNet message-passing hot path.
 *
 * This is the drop-in boundary.  The reference has no native code at all: the path is
 * Python calling torch_geometric.  Each entry point below names the reference interface
 * it replaces (paths relative to the reference repo, mllam/neural-lam @ 434d5fab):
 *
 *   nlam_graph_create        <- InteractionNet.__init__ edge_index handling
 *                               (neural_lam/gnn_layers.py:73-86)
 *   nlam_inet_fwd            <- InteractionNet.forward / PropagationNet
 *                               (neural_lam/gnn_layers.py:110-157, :231-249) incl. PyG
 *                               MessagePassing.propagate/aggregate (gnn_layers.py:145,:188)
 *   nlam_rowmlp_fwd          <- utils.make_mlp networks (neural_lam/utils/networks.py:27-40)
 *                               as used by embedders / grid MLPs
 *                               (models/step_predictors/graph/base.py:286-310, :322)
 *   nlam_segment_sum         <- PyG SumAggregation/MeanAggregation (scatter_add_) reached
 *                               from gnn_layers.py:188; also the backward of the gathers
 *   nlam_gather_rows         <- x.index_select(-2, edge_index[k]) in PyG propagate
 *   nlam_step_epilogue       <- rescale + residual + boundary mix
 *   nlam_rowmlp_step_fwd     <- output_map MLP + that epilogue in one launch
 *                               (graph/base.py:339-342, forecasters/autoregressive.py:128-131)
 *
 * Conventions
 *   - All tensors are device pointers owned by the caller (PyTorch), fp32, row-major with
 *     the feature dimension contiguous; a "batch stride" is in ELEMENTS and may be 0 for
 *     batch-broadcast (torch.expand) inputs (reference expand_to_batch,
 *     models/step_predictors/base.py:122-139).
 *   - Every call is asynchronous on `stream` (a cudaStream_t / CUstream passed as void*);
 *     no entry point synchronises the device.
 *   - Return value: 0 on success, non-zero error code otherwise (NLAM_E_*), with a message
 *     retrievable through nlam_last_error().  Nothing throws or exits across the ABI.
 *   - There is no CPU fallback: calls fail with NLAM_E_CUDA if no device is usable.
 */
#ifndef NLAM_B200_H
#define NLAM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NLAM_ABI_VERSION 1

/* error codes */
#define NLAM_OK 0
#define NLAM_E_INVALID 1     /* bad argument / shape */
#define NLAM_E_UNSUPPORTED 2 /* shape not supported by the requested kernel family */
#define NLAM_E_CUDA 3        /* CUDA runtime/driver error */
#define NLAM_E_WORKSPACE 4   /* workspace too small */

/* flags for nlam_inet_fwd / nlam_rowmlp_fwd */
#define NLAM_AGGR_MEAN 0x1        /* mean instead of sum aggregation */
#define NLAM_PROPAGATION 0x2      /* PropagationNet: msg = x_j + mlp(..), node residual = aggr */
#define NLAM_MATH_TF32 0x10       /* wgmma TF32 tensor-core kernels (fp32 accumulate) */
#define NLAM_MATH_FP32 0x20       /* exact fp32 FFMA kernels */
#define NLAM_HINT_ONE_HIDDEN 0x100 /* promise to nlam_inet_workspace_bytes: both MLPs are Linear-SiLU-Linear-LayerNorm */
#define NLAM_EDGE_ONLY 0x200      /* nlam_inet_fwd: stop after the aggregation (aggr_out required; rec_out unused): the node
                                     update runs in a later call, e.g. nlam_node_update_step_fwd */
/* neither math flag: TF32 when the shape is supported by the tensor-core kernels, else FP32 */

#define NLAM_MAX_LINEAR 4
#define NLAM_MAX_SRC 4

/* One make_mlp network: Linear -> SiLU -> ... -> Linear [-> LayerNorm].
 * w[l] is the nn.Linear weight (out_dim[l], in_dim[l]) row-major, b[l] its bias. */
typedef struct NlamMlp {
  int32_t n_linear;                 /* hidden_layers + 1 */
  int32_t in_dim;                   /* input width of w[0] */
  int32_t out_dim[NLAM_MAX_LINEAR]; /* output width of each Linear */
  const float* w[NLAM_MAX_LINEAR];
  const float* b[NLAM_MAX_LINEAR];
  const float* ln_gamma; /* NULL: no LayerNorm */
  const float* ln_beta;
  float ln_eps;
  int32_t _pad;
} NlamMlp;

/* One input block of a row-MLP: rows of width `dim`, optionally gathered through idx. */
typedef struct NlamRowSrc {
  const float* ptr;
  const int32_t* idx; /* NULL: row r reads row r; else row r reads row idx[r] */
  int64_t bstride;    /* elements between batches (0 = broadcast) */
  int32_t dim;        /* width; rows are contiguous with pitch `dim` */
  int32_t _pad;
} NlamRowSrc;

typedef struct NlamGraph NlamGraph; /* opaque: receiver-sorted CSR (+ sender CSR) of one edge set */

/* library info */
int nlam_abi_version(void);
const char* nlam_last_error(void);
const char* nlam_build_info(void);
/* number of kernel launches this library has issued in this process (host-side counter; a
 * launch recorded into a CUDA graph during stream capture counts once) */
int64_t nlam_launch_count(void);

/* Per-launch profile (measurement aid for bench.py's per-kernel roofline table): while enabled, every kernel
 * launch of the library is bracketed by CUDA events on its stream.  nlam_profile_enable(1) clears the record and
 * starts collecting, (0) stops; nlam_profile_get returns launch i's kernel name, device time (ms; waits for the
 * launch to finish) and its algorithmic bytes (distinct input bytes + output bytes).  Not for use inside a CUDA
 * stream capture. */
void nlam_profile_enable(int on);
int nlam_profile_count(void);
int nlam_profile_get(int i, char* name, int name_cap, float* ms, double* bytes);

/* Build the device CSR of one edge set.  edge_index is a HOST pointer to the (2,E) int64
 * array the reference passes to InteractionNet (row 0 senders, row 1 receivers, both
 * zero-based in their own node set).  num_rec = max(receiver)+1 as the reference infers it
 * (gnn_layers.py:73) unless n_rec_hint > that. */
int nlam_graph_create(NlamGraph** out, const int64_t* edge_index, int64_t n_edges,
                      int64_t n_rec_hint, int device);
void nlam_graph_destroy(NlamGraph* g);
int64_t nlam_graph_num_edges(const NlamGraph* g);
int64_t nlam_graph_num_rec(const NlamGraph* g);
int64_t nlam_graph_num_send(const NlamGraph* g);   /* max(sender)+1 */
int32_t nlam_graph_max_in_degree(const NlamGraph* g);
int32_t nlam_graph_is_sorted(const NlamGraph* g);   /* 1 if the given order already is CSR order */
/* d if every receiver has exactly d incoming edges (mesh->grid: 4 nearest mesh nodes, reference
 * create_graph.py:779-792; mesh-down: one parent), else 0; such edge sets with update_edges=False take the
 * receiver-tiled kernels.  ell_window: 1 if additionally d <= 8 (the uniform-degree edge path applies). */
int32_t nlam_graph_uniform_degree(const NlamGraph* g);
int32_t nlam_graph_ell_window(const NlamGraph* g);
/* device pointers (int32): receiver CSR, sender CSR (for gather backward), permutations */
const int32_t* nlam_graph_rowptr(const NlamGraph* g);   /* (num_rec+1) */
const int32_t* nlam_graph_src(const NlamGraph* g);      /* (E) sender of CSR-ordered edge k */
const int32_t* nlam_graph_dst(const NlamGraph* g);      /* (E) receiver of CSR-ordered edge k */
const int32_t* nlam_graph_perm(const NlamGraph* g);     /* (E) original edge id of CSR edge k */
const int32_t* nlam_graph_inv_perm(const NlamGraph* g); /* (E) CSR position of original edge i */
const int32_t* nlam_graph_sptr(const NlamGraph* g);     /* (num_send+1) sender CSR offsets */
const int32_t* nlam_graph_sperm(const NlamGraph* g);    /* (E) CSR-order edge ids grouped by sender */

/* Workspace (bytes) nlam_inet_fwd needs for batch B and width H. */
size_t nlam_inet_workspace_bytes(const NlamGraph* g, int B, int H, int flags);

/* One InteractionNet / PropagationNet forward.  `edge` and `edge_out` are in CSR edge order
 * (nlam_graph_perm); send (B,Ns,H), rec (B,Nr,H), edge (B,E,H), rec_out (B,Nr,H),
 * edge_out (B,E,H) or NULL (update_edges=False).  aggr_out (B,Nr,H) may be NULL (then it
 * lives in the workspace); out strides are dense.
 * edge_out may ALIAS edge (e' written over e: the middle layers of a processor stack whose intermediate edge tensors
 * nobody else reads) only for the call shapes nlam_inet_inplace_supported reports; aliasing is an error otherwise. */
int nlam_inet_fwd(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp,
                  const float* send, int64_t send_bstride, const float* rec, int64_t rec_bstride,
                  const float* edge, int64_t edge_bstride, float* rec_out, float* edge_out,
                  float* aggr_out, int B, int flags, void* workspace, size_t ws_bytes,
                  void* stream);

/* Stack of InteractionNet layers over ONE node set (send == rec: the mesh processor, reference graph_lam.py:117-126).  With
 * next_edge_mlp + proj_out the node update of this call also computes the node projections of the NEXT layer's edge MLP,
 * P_s = W1s'·x', P_r = W1r'·x' + b1' (proj_out: (2, B, n_rec, 64)), in the same kernel (csrc/fused.cu); with proj_in the edge stage
 * of this call takes its projections from the previous call instead of launching its own projection pass.  Both NULL: exactly
 * nlam_inet_fwd.  nlam_inet_chain_supported says whether a call shape can be a consumer (next_edge_mlp NULL) and a producer. */
int nlam_inet_chain_supported(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp, const NlamMlp* next_edge_mlp,
                              const float* send, int64_t send_bstride, const float* rec, int64_t rec_bstride, int B, int flags);
int nlam_inet_fwd_chain(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp, const NlamMlp* next_edge_mlp,
                        const float* send, int64_t send_bstride, const float* rec, int64_t rec_bstride, const float* edge,
                        int64_t edge_bstride, float* rec_out, float* edge_out, float* aggr_out, const float* proj_in,
                        float* proj_out, int B, int flags, void* workspace, size_t ws_bytes, void* stream);

/* 1 if nlam_inet_fwd with these arguments may be called with edge_out == edge (tensor-core path with node projections on a
 * general CSR edge set, dense batches: each tile reads its edge rows and writes e + m back, csrc/fused.cu), else 0. */
int nlam_inet_inplace_supported(const NlamGraph* g, const NlamMlp* edge_mlp, const float* send, int64_t send_bstride,
                                const float* rec, int64_t rec_bstride, const float* edge, int64_t edge_bstride, int B,
                                int flags);

/* out[b,r,:] = (res ? res[b, ridx ? ridx[r] : r, :] : 0) + MLP(concat_s src_s[b, idx_s[r], :])
 * for r in [0,n_rows); out2 (nullable) = res2[b,r,:] + out[b,r,:]. */
int nlam_rowmlp_fwd(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res,
                    const NlamRowSrc* res2, float* out, float* out2, int64_t n_rows, int B,
                    int flags, void* stream);

/* Tail of the grid side of a forecast step in one launch (csrc/fused.cu): the node update of the mesh->grid InteractionNet
 *   grid' = rec + node_mlp([rec | aggr])              (reference gnn_layers.py:148-151)
 * chained with output_map and the step epilogue of nlam_rowmlp_step_fwd; grid' never leaves the SM.  rec (B, n_rows, 64)
 * with batch stride rec_bstride, aggr (B, n_rows, 64) dense (nlam_inet_fwd with NLAM_EDGE_ONLY).  NLAM_E_UNSUPPORTED for
 * shapes / math modes the fused kernel does not cover (callers then run nlam_inet_fwd + nlam_rowmlp_step_fwd). */
int nlam_node_update_step_fwd(const NlamMlp* node_mlp, const NlamMlp* out_mlp, const float* rec, int64_t rec_bstride,
                              const float* aggr, const float* prev, const float* boundary, const float* bmask,
                              const float* diff_std, const float* diff_mean, float* new_state, int64_t n_rows, int B,
                              int flags, void* stream);

/* The whole mesh->grid decoder of a forecast step (reference gnn_layers.py:110-157 for the m2g InteractionNet, then
 * graph/base.py:322-342 and forecasters/autoregressive.py:128-131) in two launches (csrc/fused.cu): the edge projections
 * P_s = send·W1sᵀ (per batch element) and P_e = edge·W1eᵀ + b1 (once), then one kernel for the edge MLP, the per-receiver
 * aggregation, the node update rec' = rec + node_mlp([rec | aggr]), output_map and the step epilogue of
 * nlam_rowmlp_step_fwd.  Neither the aggregate nor rec' goes to HBM.  send (B, n_send, 64), rec (B, n_rec, 64) with batch
 * strides, edge (E, 64) in CSR edge order shared by the batch (edge_bstride 0, or B = 1).  Covered: TF32 math, H = 64,
 * hidden_layers = 1, edge MLP 192 -> 64 -> 64 with LayerNorm (sum or mean aggregation, no edge update), node MLP
 * 128 -> 64 -> 64 with LayerNorm, output_map 64 -> 64 -> D (D < 64, no LayerNorm), uniform in-degree d in {1, 2, 4, 8}.
 * NLAM_E_UNSUPPORTED otherwise (callers then run nlam_inet_fwd with NLAM_EDGE_ONLY + nlam_node_update_step_fwd).
 * workspace: at least nlam_decode_workspace_bytes(g, B) bytes. */
size_t nlam_decode_workspace_bytes(const NlamGraph* g, int B);
int nlam_decode_step_fwd(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* node_mlp, const NlamMlp* out_mlp,
                         const float* send, int64_t send_bstride, const float* rec, int64_t rec_bstride, const float* edge,
                         int64_t edge_bstride, const float* prev, const float* boundary, const float* bmask,
                         const float* diff_std, const float* diff_mean, float* new_state, int B, int flags, void* workspace,
                         size_t ws_bytes, void* stream);
/* The grid side of a forecast step's encoder (reference graph/base.py:275-310) in one launch (csrc/fused.cu).  For the
 * concatenated inputs x = [src_0 | src_1 | ...] (at most 64 columns, dense rows without index) of each grid row:
 *   grid_emb = embed_mlp(x)                          never leaves the SM
 *   P_s      = grid_emb·W1sᵀ                         W1s = columns 64..127 of the g2m edge MLP's first Linear
 *   grid_rep = grid_emb + grid_mlp(grid_emb)
 * and once for the batch P_r = mesh·W1rᵀ + b1 (W1r = columns 128..191; mesh (g2m receivers, 64) shared by the batch).
 * grid_rep (B, n_rows, 64) dense; proj = [P_s (B, n_rows, 64) | P_r (n_rec, 64)], 16-byte aligned: the proj_in of the g2m call
 * nlam_inet_fwd_chain(g2m, ..., send = P_s, rec = mesh, edge = g2m_edge, next_edge_mlp = NULL, proj_in = proj), whose edge
 * stage then skips its own projection pass.  Covered: TF32 math, H = 64, every MLP in -> 64 -> 64 with biases and an affine
 * LayerNorm, g2m senders = the n_rows grid rows, and a g2m call that takes the batch-broadcast split edge path (edge features
 * and mesh rows shared by the batch); nlam_encode_supported says whether a call is.  NLAM_E_UNSUPPORTED otherwise (callers
 * then run nlam_rowmlp_fwd for the embedder, nlam_inet_fwd for g2m and nlam_rowmlp_fwd for grid_mlp). */
int nlam_encode_supported(const NlamGraph* g2m, const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src, const NlamMlp* grid_mlp,
                          const NlamMlp* g2m_edge_mlp, const float* mesh, int64_t mesh_bstride, const float* g2m_edge,
                          int64_t edge_bstride, const float* grid_rep, const float* proj, int64_t n_rows, int B, int flags);
int nlam_encode_fwd(const NlamGraph* g2m, const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src, const NlamMlp* grid_mlp,
                    const NlamMlp* g2m_edge_mlp, const float* mesh, int64_t mesh_bstride, const float* g2m_edge, int64_t edge_bstride,
                    float* grid_rep, float* proj, int64_t n_rows, int B, int flags, void* stream);
/* nlam_encode_fwd that also stores grid_emb (B, n_rows, 64) dense, 16-byte aligned: Graph-EFM's decoder reads it as the
 * senders of its grid -> mesh layer (reference latent/base_decoder.py:145-155).  Same coverage as nlam_encode_fwd. */
int nlam_encode_emb_fwd(const NlamGraph* g2m, const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src, const NlamMlp* grid_mlp,
                        const NlamMlp* g2m_edge_mlp, const float* mesh, int64_t mesh_bstride, const float* g2m_edge,
                        int64_t edge_bstride, float* grid_rep, float* proj, float* grid_emb, int64_t n_rows, int B, int flags,
                        void* stream);
/* nlam_encode_fwd for two grid -> mesh layers on the same grid embedding, receivers and edge features (the hierarchical
 * Graph-EFM's prior and decoder g2m layers, reference latent/hi_graph_encoder.py:148-150, hi_graph_decoder.py:216-218): the
 * launch also computes proj_b = [P_s_b (B, n_rows, 64) | P_r_b (n_rec, 64)] of g2m_edge_mlp_b, the proj_in of the second
 * layer's nlam_inet_fwd_chain call (send = P_s_b).  grid_emb is not stored.  Covered where nlam_encode_fwd covers the first
 * layer and the second layer's call takes the same batch-broadcast split edge path; nlam_encode2_supported says whether a
 * call is.  NLAM_E_UNSUPPORTED otherwise. */
int nlam_encode2_supported(const NlamGraph* g2m, const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src,
                           const NlamMlp* grid_mlp, const NlamMlp* g2m_edge_mlp, const NlamMlp* g2m_edge_mlp_b, const float* mesh,
                           int64_t mesh_bstride, const float* g2m_edge, int64_t edge_bstride, const float* grid_rep,
                           const float* proj, const float* proj_b, int64_t n_rows, int B, int flags);
int nlam_encode2_fwd(const NlamGraph* g2m, const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src, const NlamMlp* grid_mlp,
                     const NlamMlp* g2m_edge_mlp, const NlamMlp* g2m_edge_mlp_b, const float* mesh, int64_t mesh_bstride,
                     const float* g2m_edge, int64_t edge_bstride, float* grid_rep, float* proj, float* proj_b, int64_t n_rows,
                     int B, int flags, void* stream);
/* The stochastic step of Graph-EFM (reference latent/graph_encoder.py:102-105, base_encoder.py:85-94,
 * base_decoder.py:145) in one launch (csrc/fused.cu).  Per row r of batch element b, x (B, n_rows, 64) the prior's mesh
 * representation and eps (B, n_rows, 64) standard normal noise, both with dense rows and batch strides x_bstride /
 * eps_bstride (floats):
 *   p          = param_mlp(x)                         latent_param_map: Linear-SiLU-Linear, no LayerNorm, 64 or 128 outputs
 *   mean, std  = p[:, :64], 1 (64 outputs) or 1e-4 + softplus(p[:, 64:]) (128 outputs)
 *   z          = mean + eps*std                       torch's rounding: the product, then the sum
 *   latent_emb = embed_mlp(z)                         latent_embedder: 64 -> 64 -> 64 with LayerNorm
 * Only latent_emb (B, n_rows, 64) dense is written.  Covered: TF32 math, H = latent_dim = 64, hidden_layers = 1, 16-byte
 * aligned tensors; nlam_latent_sample_supported says whether a call is.  NLAM_E_UNSUPPORTED otherwise (callers then run
 * param_mlp, the sample and embed_mlp as separate calls). */
int nlam_latent_sample_supported(const NlamMlp* param_mlp, const NlamMlp* embed_mlp, const float* x, int64_t x_bstride,
                                 const float* eps, int64_t eps_bstride, const float* latent_emb, int64_t n_rows, int B, int flags);
int nlam_latent_sample_fwd(const NlamMlp* param_mlp, const NlamMlp* embed_mlp, const float* x, int64_t x_bstride, const float* eps,
                           int64_t eps_bstride, float* latent_emb, int64_t n_rows, int B, int flags, void* stream);
/* Statistics of an ensemble of K forecast members (csrc/ensemble.cu, DESIGN §4.5).  members (B, K, G, d): member k of
 * initial condition b starts at members + b*member_bstride + k*member_kstride (elements) and holds a dense (G, d) block, so
 * rows b*K + k of a forecast batch and a time slice of a (B, K, T, G, d) tensor both qualify.  Per point, x_1..x_K its
 * members and y = target[b*target_bstride + g*d + v]:
 *   mean = (1/K) Σ x_k,   std = sqrt((1/(K-1)) Σ (x_k - mean)²)                     (B, G, d) dense
 *   SE = (mean - y)²,  s² = std²,  A = (1/K) Σ |x_k - y|,  D = (1/(K(K-1))) Σ_{k≠l} |x_k - x_l|
 * scores (B, d, 4) (NULL: not computed; then target, interior and the workspace may be NULL) holds the means of
 * [SE, s², A, D] over the interior grid nodes (interior[g] != 0; the reference's interior_mask_bool).  Exact fp32; the grid
 * reduction is two-stage in a fixed order (no atomics): bit-reproducible, and row b's results do not depend on the other
 * rows.  2 <= K <= 64, else NLAM_E_UNSUPPORTED.  workspace: nlam_ensemble_stats_workspace_bytes(B, G, d) bytes when
 * scores is given. */
size_t nlam_ensemble_stats_workspace_bytes(int B, int64_t G, int d);
int nlam_ensemble_stats(const float* members, int64_t member_bstride, int64_t member_kstride, int B, int K, int64_t G, int d,
                        const float* target, int64_t target_bstride, const float* interior, float* mean, float* std,
                        float* scores, void* workspace, size_t ws_bytes, void* stream);
/* out[b,n,:] = scale_n * sum_{k in [ptr[n],ptr[n+1])} x[b, order ? order[k] : k, :]
 * scale_n = 1 (sum) or 1/max(deg,1) (mean).  Deterministic, CSR order. */
int nlam_segment_sum(const int32_t* ptr, const int32_t* order, int64_t n_seg, const float* x,
                     int64_t x_bstride, float* out, int64_t out_bstride, int B, int H, int mean,
                     void* stream);

/* out[b,r,:] = scale * x[b, idx[r], :]   (scale_by_deg_ptr: optional CSR offsets; when given,
 * row r is additionally scaled by 1/max(deg(idx[r]),1) — backward of the mean aggregation). */
int nlam_gather_rows(const float* x, int64_t x_bstride, const int32_t* idx, int64_t n_rows,
                     float* out, int64_t out_bstride, int B, int H, const int32_t* deg_ptr,
                     void* stream);

/* Node-partitioned rollout (one process per GPU): copy this rank's own sender rows (B, n_own, H) into the front of its
 * extended buffer ext_local (B, ext rows, H; batch stride ext_bs, the same on every rank) and store the rows listed in
 * send_rows[send_ptr[p] .. send_ptr[p+1]) into peer p's extended buffer peer_ext[p] (a DEVICE array of `world`
 * pointers to the peers' buffers mapped into this process: CUDA IPC / symmetric memory) at rows peer_dst_off[p] .. —
 * direct stores over NVLink from this kernel.  The caller issues a cross-rank barrier before the buffers are read.
 * Replaces the pack + NCCL send/recv + concatenation of a halo exchange (SURVEY.md 8e). */
int nlam_halo_push(const float* own, int64_t own_bs, int64_t n_own, float* ext_local, int64_t ext_bs,
                   float* const* peer_ext, const int32_t* send_rows, const int32_t* send_ptr,
                   const int32_t* peer_dst_off, int64_t n_send_total, int world, int B, int H, void* stream);

/* ---- Backward building blocks (bwd.cu) and the generic wgmma Linear (tc7.cu) -------------------------------
 * The backward of the path (reference: autograd through gnn_layers.py:110-157 / utils/networks.py:27-40) is composed
 * from these launches by the host side (neural_lam_b200/backward.py): dX = dY · W and dW = dYᵀ · X run on nlam_linear
 * (dW as split-K partial products over zero-padded transposes, reduced in a fixed order by nlam_reduce_partials). */
/* out = epi([x0 | x1] · wᵀ + bias + add0[add0_idx] + add1[add1_idx]); epi = SiLU (act) / LayerNorm (gamma, beta), then
 * + post[post_idx], optional second output out2 (before the residual), + res.  x0: (B|1, n_rows, k0) with row pitch
 * x0_pitch (0 = k0); w: (n_out, w_cols) with row pitch ldw, batch stride w_bs (0 = shared).  K multiple of 32, n_out <= 256. */
int nlam_linear(const float* x0, int64_t x0_bs, int k0, int64_t x0_pitch, const float* x1, int64_t x1_bs, int k1,
                const float* w, int ldw, int w_cols, int64_t w_bs, const float* bias, int n_out, int act, const float* gamma,
                const float* beta, float eps, const float* add0, const int32_t* add0_idx, int64_t add0_bs, const float* add1,
                const int32_t* add1_idx, int64_t add1_bs, const float* post, const int32_t* post_idx, int64_t post_bs,
                const float* res, int64_t res_bs, int64_t n_rows, int B, float* out, float* out2, void* stream);
/* out[b, r, :kp] = [s0 | s1 | s2 | s3 | zeros]: the concatenation the reference materialises with torch.cat
 * (graph/base.py:275-283), zero-padded to kp columns (the generic Linear wants K a multiple of 32) */
int nlam_pack_rows(const float* s0, const float* s1, const float* s2, const float* s3, int d0, int d1, int d2, int d3,
                   int64_t bs0, int64_t bs1, int64_t bs2, int64_t bs3, float* out, int kp, int64_t n_rows, int B, void* stream);
/* Parameter-gradient destinations of one make_mlp network (same layout as NlamMlp; every buffer is OVERWRITTEN). */
typedef struct NlamMlpGrads {
  float* w[NLAM_MAX_LINEAR];
  float* b[NLAM_MAX_LINEAR];
  float* ln_gamma;
  float* ln_beta;
} NlamMlpGrads;

/* Backward of out = mlp(concat_s src_s[b, r, :]) (two Linear layers; residuals pass their gradient through on the host
 * side): g_out (B, n_rows, n_out) dense -> g_srcs[s] (B, n_rows, dim_s) dense (NULL: not needed) and the parameter
 * gradients.  Sources may be batch-broadcast (bstride 0).  Replaces autograd through utils/networks.py:27-40. */
size_t nlam_mlp_bwd_workspace_bytes(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, int64_t n_rows, int B);
int nlam_mlp_bwd(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const float* g_out, float* const* g_srcs,
                 const NlamMlpGrads* grads, int64_t n_rows, int B, void* workspace, size_t ws_bytes, void* stream);

/* Backward of nlam_inet_fwd (reference: autograd through gnn_layers.py:110-157 / :231-249; tests/test_gnn_layers.py
 * section F): recompute-in-backward from the layer inputs (edge tensors in CSR order), g_rec_out (B, n_rec, H) and
 * g_edge_out (B, E, H; NULL if the edge output is unused) -> g_send (B, n_send, H), g_rec, g_edge (dense, per batch
 * element even for batch-broadcast inputs) and all parameter gradients.  hidden_layers = 1, H in {64, 128, 256};
 * flags: NLAM_AGGR_MEAN, NLAM_PROPAGATION.  TF32 tensor-core products, ordered reductions (bit-reproducible). */
size_t nlam_inet_bwd_workspace_bytes(const NlamGraph* g, int B, int H, int flags);
int nlam_inet_bwd(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp, const float* send, int64_t send_bs,
                  const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs, const float* g_rec_out,
                  const float* g_edge_out, float* g_send, float* g_rec, float* g_edge, const NlamMlpGrads* edge_grads,
                  const NlamMlpGrads* aggr_grads, int B, int flags, void* workspace, size_t ws_bytes, void* stream);

/* gh == NULL: out = SiLU(z); else out = gh * SiLU'(z)  (n elements, n % 4 == 0) */
int nlam_silu(const float* z, const float* gh, float* out, int64_t n, void* stream);
int nlam_layernorm_fwd(const float* y, const float* gamma, const float* beta, float eps, float* out, int64_t rows, int H,
                       void* stream);
/* gy = dL/dy for out = LayerNorm(y); dgamma / dbeta (H) overwritten; scratch: nlam_bwd_scratch_floats(H) floats */
int nlam_layernorm_bwd(const float* g, const float* y, const float* gamma, float eps, float* gy, float* dgamma, float* dbeta,
                       int64_t rows, int H, float* scratch, void* stream);
size_t nlam_bwd_scratch_floats(int C);
/* out[c] = sum_r g[r, c]  (bias gradients); scratch: nlam_bwd_scratch_floats(C) floats */
int nlam_colsum(const float* g, int64_t rows, int C, float* out, float* scratch, void* stream);
/* out[r, c] (+)= sum_p part[p, r, c]  (ordered) */
int nlam_reduce_partials(const float* part, int P, int64_t R, int C, float* out, int64_t out_pitch, int accumulate,
                         void* stream);
/* xt[c, r] = x[r, c] (row pitch x_pitch), zero for rows <= r < rows_pad */
int nlam_transpose_pad(const float* x, int64_t rows, int C, int64_t x_pitch, float* xt, int64_t rows_pad, void* stream);
/* out[b, e, :] = (a ? a[b, e, :] : 0) + v[b, idx[e], :] * (deg_ptr ? 1 / max(deg(idx[e]), 1) : 1) */
int nlam_add_gather(const float* a, const float* v, const int32_t* idx, const int32_t* deg_ptr, int64_t n_e, int64_t n_v, int H,
                    int B, float* out, void* stream);

/* Strided host <-> device copy of `height` rows of `width_bytes` (cudaMemcpy2DAsync on `stream`): the per-step slice of a
 * (B, T, G, F) pinned host tensor in ONE call (ARForecaster.rollout_from_host). */
int nlam_memcpy2d_async(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width_bytes, size_t height,
                        int host_to_device, void* stream);

/* The same with a depth: `depth` slices of `height` rows; slice stride = pitch * rows-per-slice on either side
 * (cudaMemcpy3DAsync).  Used to move only the boundary frame of a forecast step's boundary tensor. */
int nlam_memcpy3d_async(void* dst, size_t dpitch, size_t drows, const void* src, size_t spitch, size_t srows, size_t width_bytes,
                        size_t height, size_t depth, int host_to_device, void* stream);

/* new_state = bmask * boundary + (1-bmask) * (prev + net_out*diff_std + diff_mean)
 * over (B,G,D); bmask (G), diff_std/mean (D); boundary may be NULL (then bmask ignored). */
int nlam_step_epilogue(const float* net_out, const float* prev, const float* boundary,
                       const float* bmask, const float* diff_std, const float* diff_mean,
                       float* new_state, int64_t B, int64_t G, int64_t D, void* stream);

/* The same with the reference's CLAMPED update for state variables with configured limits (models/step_predictors/
 * base.py:296-396): clamp_kind[d] = 0 plain residual, 1 sigmoid between (clamp_lo[d], clamp_up[d]), 2 softplus above
 * clamp_lo[d], 3 mirrored softplus below clamp_up[d]; new = f(f^-1(prev) + net_out*diff_std + diff_mean), then the
 * boundary mix.  Limits in standardised units. */
int nlam_step_epilogue_clamped(const float* net_out, const float* prev, const float* boundary, const float* bmask,
                               const float* diff_std, const float* diff_mean, const int32_t* clamp_kind, const float* clamp_lo,
                               const float* clamp_up, float* new_state, int64_t B, int64_t G, int64_t D, void* stream);

/* output_map + step epilogue in one launch (reference graph/base.py:322-342 followed by
 * forecasters/autoregressive.py:128-131):
 *   y = MLP(concat_s src_s[b, r, :])                      (narrow output D < 64, no LayerNorm)
 *   new_state = bmask * boundary + (1-bmask) * (prev + (y*diff_std + diff_mean))
 * Tensor-core (TF32) path only: returns NLAM_E_UNSUPPORTED for other shapes / NLAM_MATH_FP32, in which case the
 * caller issues nlam_rowmlp_fwd + nlam_step_epilogue. */
int nlam_rowmlp_step_fwd(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const float* prev,
                         const float* boundary, const float* bmask, const float* diff_std,
                         const float* diff_mean, float* new_state, int64_t n_rows, int B, int flags,
                         void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NLAM_B200_H */

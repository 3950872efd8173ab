// C-ABI entry points that dispatch between the wgmma (TF32) kernels and the exact fp32
// kernels.  See include/nlam_b200.h for the contract and the reference interfaces replaced.
#include "common.cuh"

#include <algorithm>

using namespace nlam;

static bool want_tf32(int flags) { return !(flags & NLAM_MATH_FP32); }

extern "C" int nlam_rowmlp_fwd(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res,
                               const NlamRowSrc* res2, float* out, float* out2, int64_t n_rows, int B, int flags,
                               void* stream) {
  NLAM_REQUIRE(mlp && srcs && out, NLAM_E_INVALID, "nlam_rowmlp_fwd: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (want_tf32(flags) && tc_rowmlp_supported(mlp, srcs, n_src, res, res2, n_rows))
    return tc_rowmlp(mlp, srcs, n_src, res, out, n_rows, B, st);
  if (want_tf32(flags) && !out2 && tc_mlp2_supported(mlp, srcs, n_src, res, res2)) {
    // H = 128 / 256: two launches of the generic wgmma Linear kernel; the hidden activations live in a
    // stream-ordered scratch allocation (legal inside a stream capture)
    float* ws = nullptr;
    NLAM_CUDA_OK(cudaMallocAsync((void**)&ws, (size_t)n_rows * B * mlp->out_dim[0] * sizeof(float), st));
    const int rc = tc_mlp2(mlp, srcs, n_src, res, out, n_rows, B, st, ws);
    NLAM_CUDA_OK(cudaFreeAsync(ws, st));
    return rc;
  }
  if (want_tf32(flags) && !out2 && tc_mlp2_packed_supported(mlp, srcs, n_src, res, res2)) {
    // narrow / concatenated / gathered inputs (any H of the generic kernel): pack, then the two generic Linear launches
    float* ws = nullptr;
    NLAM_CUDA_OK(cudaMallocAsync((void**)&ws, tc_mlp2_packed_workspace_floats(mlp, n_rows, B) * sizeof(float), st));
    const int rc = tc_mlp2_packed(mlp, srcs, n_src, res, out, n_rows, B, st, ws);
    NLAM_CUDA_OK(cudaFreeAsync(ws, st));
    return rc;
  }
  NLAM_REQUIRE(!(flags & NLAM_MATH_TF32), NLAM_E_UNSUPPORTED,
               "nlam_rowmlp_fwd: shape not supported by the tensor-core kernels (in=%d)", mlp->in_dim);
  return rowmlp_simt(mlp, srcs, n_src, res, res2, out, out2, n_rows, B, st);
}

extern "C" int nlam_rowmlp_step_fwd(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const float* prev,
                                    const float* boundary, const float* bmask, const float* diff_std,
                                    const float* diff_mean, float* new_state, int64_t n_rows, int B, int flags,
                                    void* stream) {
  NLAM_REQUIRE(mlp && srcs && prev && diff_std && diff_mean && new_state, NLAM_E_INVALID, "nlam_rowmlp_step_fwd: null argument");
  NLAM_REQUIRE((boundary == nullptr) || bmask, NLAM_E_INVALID, "nlam_rowmlp_step_fwd: boundary without mask");
  const int nout = mlp->out_dim[mlp->n_linear - 1];
  // only the tensor-core path fuses the epilogue; callers fall back to nlam_rowmlp_fwd + nlam_step_epilogue
  NLAM_REQUIRE(want_tf32(flags) && nout < 64 && !mlp->ln_gamma && tc_rowmlp_supported(mlp, srcs, n_src, nullptr, nullptr, n_rows),
               NLAM_E_UNSUPPORTED, "nlam_rowmlp_step_fwd: shape / math mode not covered by the fused kernel");
  StepEpilogue ep = {prev, boundary, bmask, diff_std, diff_mean};
  return tc_rowmlp(mlp, srcs, n_src, nullptr, new_state, n_rows, B, (cudaStream_t)stream, &ep);
}

extern "C" int nlam_node_update_step_fwd(const NlamMlp* node_mlp, const NlamMlp* out_mlp, const float* rec, int64_t rec_bs,
                                         const float* aggr, const float* prev, const float* boundary, const float* bmask,
                                         const float* diff_std, const float* diff_mean, float* new_state, int64_t n_rows, int B,
                                         int flags, void* stream) {
  NLAM_REQUIRE(node_mlp && out_mlp && rec && aggr && prev && diff_std && diff_mean && new_state, NLAM_E_INVALID,
               "nlam_node_update_step_fwd: null argument");
  NLAM_REQUIRE((boundary == nullptr) || bmask, NLAM_E_INVALID, "nlam_node_update_step_fwd: boundary without mask");
  StepEpilogue ep = {prev, boundary, bmask, diff_std, diff_mean};
  NLAM_REQUIRE(want_tf32(flags) && tc_node_out_supported(node_mlp, out_mlp, rec, rec_bs, aggr, n_rows, B, new_state, &ep),
               NLAM_E_UNSUPPORTED, "nlam_node_update_step_fwd: shape / math mode not covered by the fused kernel");
  return tc_node_out(node_mlp, out_mlp, rec, rec_bs, aggr, n_rows, B, new_state, &ep, (cudaStream_t)stream);
}

static size_t rup256(size_t n) { return (n + 255) / 256 * 256; }

extern "C" size_t nlam_decode_workspace_bytes(const NlamGraph* g, int B) {
  if (!g || B < 1) return 0;
  return rup256(tc_decode_workspace_floats(g, B) * sizeof(float));
}

extern "C" int nlam_decode_step_fwd(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* node_mlp, const NlamMlp* out_mlp,
                                    const float* send, int64_t send_bs, const float* rec, int64_t rec_bs, const float* edge,
                                    int64_t edge_bs, const float* prev, const float* boundary, const float* bmask,
                                    const float* diff_std, const float* diff_mean, float* new_state, int B, int flags,
                                    void* workspace, size_t ws_bytes, void* stream) {
  NLAM_REQUIRE(g && edge_mlp && node_mlp && out_mlp && send && rec && edge && prev && diff_std && diff_mean && new_state,
               NLAM_E_INVALID, "nlam_decode_step_fwd: null argument");
  NLAM_REQUIRE((boundary == nullptr) || bmask, NLAM_E_INVALID, "nlam_decode_step_fwd: boundary without mask");
  StepEpilogue ep = {prev, boundary, bmask, diff_std, diff_mean};
  NLAM_REQUIRE(want_tf32(flags) && tc_decode_supported(g, edge_mlp, node_mlp, out_mlp, flags, send, send_bs, rec, rec_bs, edge,
                                                       edge_bs, B, new_state, &ep),
               NLAM_E_UNSUPPORTED, "nlam_decode_step_fwd: graph / shape / math mode not covered by the fused decoder");
  NLAM_REQUIRE(workspace && ws_bytes >= nlam_decode_workspace_bytes(g, B), NLAM_E_WORKSPACE,
               "nlam_decode_step_fwd: workspace too small (%zu < %zu bytes; see nlam_decode_workspace_bytes)", ws_bytes,
               nlam_decode_workspace_bytes(g, B));
  return tc_decode(g, edge_mlp, node_mlp, out_mlp, flags, send, send_bs, rec, rec_bs, edge, edge_bs, B, new_state, &ep,
                   (float*)workspace, (cudaStream_t)stream);
}

// Workspace layout: [aggregate | path-specific scratch].  Sized per path: the fused H = 64 kernels need only the node
// projections, the generic tensor-core path its projections / hidden activations / messages, the exact fp32 path the
// message buffer.
enum InetPath { PATH_EXACT = 0, PATH_TC64 = 1, PATH_GEN = 2 };
static size_t inet_scratch_bytes(const NlamGraph* g, int B, int H, InetPath path) {
  if (path == PATH_TC64) return rup256(tc_edge2_workspace_floats(g, B, 0) * sizeof(float));  // node projections
  if (path == PATH_GEN) return rup256(tc_inet_gen_workspace_floats(g, B, H) * sizeof(float));
  return rup256((size_t)B * g->n_edges * H * sizeof(float));  // exact path: messages
}

extern "C" size_t nlam_inet_workspace_bytes(const NlamGraph* g, int B, int H, int flags) {
  if (!g) return 0;
  // the path is chosen from the MLP shapes at call time; without the NLAM_HINT_ONE_HIDDEN promise (both MLPs are
  // Linear-SiLU-Linear-LayerNorm, the reference's hidden_layers = 1) the bound covers every path
  const bool tf32 = !(flags & NLAM_MATH_FP32), prop = flags & NLAM_PROPAGATION, one = flags & NLAM_HINT_ONE_HIDDEN;
  size_t need;
  if (tf32 && one && H == 64 && !prop && g->n_tiles > 0) need = inet_scratch_bytes(g, B, H, PATH_TC64);
  else if (tf32 && one && (H == 128 || H == 256 || (H == 64 && prop))) need = inet_scratch_bytes(g, B, H, PATH_GEN);
  else if (!tf32) need = inet_scratch_bytes(g, B, H, PATH_EXACT);
  else need = std::max(inet_scratch_bytes(g, B, H, PATH_EXACT),
                       std::max(inet_scratch_bytes(g, B, H, PATH_TC64), inet_scratch_bytes(g, B, H, PATH_GEN)));
  return rup256((size_t)B * g->n_rec * H * sizeof(float)) + need;
}

// the call shapes that take tc_edge_rmw (fused.cu) when edge_out aliases edge
static bool inplace_path(const NlamGraph* g, const NlamMlp* edge_mlp, const float* send, int64_t send_bs, const float* rec,
                         int64_t rec_bs, const float* edge, int64_t edge_bs, int B, int flags) {
  const int H = edge_mlp->out_dim[edge_mlp->n_linear - 1];
  if (!(want_tf32(flags) && tc_edge_supported(g, edge_mlp, flags))) return false;
  const int64_t send_rows = (B > 1 && send_bs > 0) ? send_bs / H : g->n_send;
  if (tc_ell_supported(g, edge_mlp, flags, send, send_bs, rec, rec_bs, true)) return false;
  if (!tc_edge2_supported(g, edge_mlp, flags, send, send_bs, rec, rec_bs, B, send_rows)) return false;
  return tc_edge_rmw_supported(g, edge, edge_bs, edge, B);
}

extern "C" int nlam_inet_inplace_supported(const NlamGraph* g, const NlamMlp* edge_mlp, const float* send, int64_t send_bs,
                                           const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs, int B,
                                           int flags) {
  if (!g || !edge_mlp || !send || !rec || !edge || B < 1 || edge_mlp->n_linear < 1) return 0;
  return inplace_path(g, edge_mlp, send, send_bs, rec, rec_bs, edge, edge_bs, B, flags) ? 1 : 0;
}

// chain of layers over ONE node set (the mesh processor): can this call consume node projections computed by the previous
// layer's node kernel and, with next_mlp, produce those of the next layer (fused.cu)?
static bool chain_path(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp, const NlamMlp* next_mlp,
                       const float* send, int64_t send_bs, const float* rec, int64_t rec_bs, int B, int flags) {
  if (!(want_tf32(flags) && tc_edge_supported(g, edge_mlp, flags)) || (flags & (NLAM_PROPAGATION | NLAM_EDGE_ONLY))) return false;
  if (send != rec || send_bs != rec_bs || g->n_send != g->n_rec || (B > 1 && rec_bs != g->n_rec * 64)) return false;
  if (tc_ell_supported(g, edge_mlp, flags, send, send_bs, rec, rec_bs, true)) return false;
  if (!tc_edge2_supported(g, edge_mlp, flags, send, send_bs, rec, rec_bs, B, g->n_send)) return false;
  if (next_mlp && !tc_node_proj_supported(aggr_mlp, next_mlp, rec, rec_bs, rec, g->n_rec, rec, rec)) return false;
  return true;
}

// grid -> mesh call (batch-broadcast edge features and receivers, no edge update): does nlam_inet_fwd take the split
// tc_edge_bcast path, which can consume node projections computed by nlam_encode_fwd?
static bool bcast_path(const NlamGraph* g, const NlamMlp* edge_mlp, const float* send, int64_t send_bs, const float* rec,
                       int64_t rec_bs, const float* edge, int64_t edge_bs, int B, int flags) {
  if (!(want_tf32(flags) && tc_edge_supported(g, edge_mlp, flags))) return false;
  const int64_t send_rows = (B > 1 && send_bs > 0) ? send_bs / 64 : g->n_send;
  if (tc_ell_supported(g, edge_mlp, flags, send, send_bs, rec, rec_bs, false)) return false;
  if (tc_edge2_supported(g, edge_mlp, flags, send, send_bs, rec, rec_bs, B, send_rows)) return false;
  return tc_edge_bcast_supported(g, edge_mlp, flags, send, send_bs, rec, rec_bs, edge, edge_bs, B, false);
}

extern "C" int nlam_encode_supported(const NlamGraph* g2m, const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src,
                                     const NlamMlp* grid_mlp, const NlamMlp* g2m_edge_mlp, const float* mesh, int64_t mesh_bs,
                                     const float* g2m_edge, int64_t edge_bs, const float* grid_rep, const float* proj,
                                     int64_t n_rows, int B, int flags) {
  if (!g2m || !embed_mlp || !srcs || !grid_mlp || !g2m_edge_mlp || !mesh || !g2m_edge || !grid_rep || !proj) return 0;
  if (B < 1 || g2m->n_send != n_rows || (B > 1 && mesh_bs != 0) || (((uintptr_t)grid_rep | (uintptr_t)proj) & 15)) return 0;
  if (!tc_encode_supported(embed_mlp, srcs, n_src, grid_mlp, g2m_edge_mlp, mesh, g2m->n_rec, n_rows, B, flags)) return 0;
  // the g2m call that consumes the projections: send = P_s, dense (B, n_rows, 64) at the start of proj
  return bcast_path(g2m, g2m_edge_mlp, proj, B > 1 ? n_rows * 64 : 0, mesh, mesh_bs, g2m_edge, edge_bs, B, flags) ? 1 : 0;
}

extern "C" int nlam_encode_fwd(const NlamGraph* g2m, const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src,
                               const NlamMlp* grid_mlp, const NlamMlp* g2m_edge_mlp, const float* mesh, int64_t mesh_bs,
                               const float* g2m_edge, int64_t edge_bs, float* grid_rep, float* proj, int64_t n_rows, int B,
                               int flags, void* stream) {
  NLAM_REQUIRE(g2m && embed_mlp && srcs && grid_mlp && g2m_edge_mlp && mesh && g2m_edge && grid_rep && proj, NLAM_E_INVALID,
               "nlam_encode_fwd: null argument");
  NLAM_REQUIRE(nlam_encode_supported(g2m, embed_mlp, srcs, n_src, grid_mlp, g2m_edge_mlp, mesh, mesh_bs, g2m_edge, edge_bs,
                                     grid_rep, proj, n_rows, B, flags),
               NLAM_E_UNSUPPORTED, "nlam_encode_fwd: graph / shape / math mode not covered by the fused encoder");
  return tc_encode(embed_mlp, srcs, n_src, grid_mlp, g2m_edge_mlp, mesh, g2m->n_rec, n_rows, B, flags, grid_rep, proj,
                   proj + (size_t)B * n_rows * 64, nullptr, (cudaStream_t)stream);
}

extern "C" int nlam_encode_emb_fwd(const NlamGraph* g2m, const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src,
                                   const NlamMlp* grid_mlp, const NlamMlp* g2m_edge_mlp, const float* mesh, int64_t mesh_bs,
                                   const float* g2m_edge, int64_t edge_bs, float* grid_rep, float* proj, float* grid_emb,
                                   int64_t n_rows, int B, int flags, void* stream) {
  NLAM_REQUIRE(g2m && embed_mlp && srcs && grid_mlp && g2m_edge_mlp && mesh && g2m_edge && grid_rep && proj && grid_emb,
               NLAM_E_INVALID, "nlam_encode_emb_fwd: null argument");
  NLAM_REQUIRE(((uintptr_t)grid_emb & 15) == 0, NLAM_E_INVALID, "nlam_encode_emb_fwd: unaligned grid_emb");
  NLAM_REQUIRE(nlam_encode_supported(g2m, embed_mlp, srcs, n_src, grid_mlp, g2m_edge_mlp, mesh, mesh_bs, g2m_edge, edge_bs,
                                     grid_rep, proj, n_rows, B, flags),
               NLAM_E_UNSUPPORTED, "nlam_encode_emb_fwd: graph / shape / math mode not covered by the fused encoder");
  return tc_encode(embed_mlp, srcs, n_src, grid_mlp, g2m_edge_mlp, mesh, g2m->n_rec, n_rows, B, flags, grid_rep, proj,
                   proj + (size_t)B * n_rows * 64, grid_emb, (cudaStream_t)stream);
}

extern "C" int nlam_encode2_supported(const NlamGraph* g2m, const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src,
                                      const NlamMlp* grid_mlp, const NlamMlp* g2m_edge_mlp, const NlamMlp* g2m_edge_mlp_b,
                                      const float* mesh, int64_t mesh_bs, const float* g2m_edge, int64_t edge_bs,
                                      const float* grid_rep, const float* proj, const float* proj_b, int64_t n_rows, int B,
                                      int flags) {
  if (!g2m_edge_mlp_b || !proj_b || ((uintptr_t)proj_b & 15)) return 0;
  if (!nlam_encode_supported(g2m, embed_mlp, srcs, n_src, grid_mlp, g2m_edge_mlp, mesh, mesh_bs, g2m_edge, edge_bs, grid_rep,
                             proj, n_rows, B, flags))
    return 0;
  if (!tc_encode_supported(embed_mlp, srcs, n_src, grid_mlp, g2m_edge_mlp_b, mesh, g2m->n_rec, n_rows, B, flags)) return 0;
  // the second g2m call consumes its projections on the same path as the first
  return bcast_path(g2m, g2m_edge_mlp_b, proj_b, B > 1 ? n_rows * 64 : 0, mesh, mesh_bs, g2m_edge, edge_bs, B, flags) ? 1 : 0;
}

extern "C" int nlam_encode2_fwd(const NlamGraph* g2m, const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src,
                                const NlamMlp* grid_mlp, const NlamMlp* g2m_edge_mlp, const NlamMlp* g2m_edge_mlp_b,
                                const float* mesh, int64_t mesh_bs, const float* g2m_edge, int64_t edge_bs, float* grid_rep,
                                float* proj, float* proj_b, int64_t n_rows, int B, int flags, void* stream) {
  NLAM_REQUIRE(g2m && embed_mlp && srcs && grid_mlp && g2m_edge_mlp && g2m_edge_mlp_b && mesh && g2m_edge && grid_rep && proj &&
                   proj_b,
               NLAM_E_INVALID, "nlam_encode2_fwd: null argument");
  NLAM_REQUIRE(nlam_encode2_supported(g2m, embed_mlp, srcs, n_src, grid_mlp, g2m_edge_mlp, g2m_edge_mlp_b, mesh, mesh_bs,
                                      g2m_edge, edge_bs, grid_rep, proj, proj_b, n_rows, B, flags),
               NLAM_E_UNSUPPORTED, "nlam_encode2_fwd: graph / shape / math mode not covered by the fused encoder");
  const size_t grid_floats = (size_t)B * n_rows * 64;
  return tc_encode(embed_mlp, srcs, n_src, grid_mlp, g2m_edge_mlp, mesh, g2m->n_rec, n_rows, B, flags, grid_rep, proj,
                   proj + grid_floats, nullptr, (cudaStream_t)stream, g2m_edge_mlp_b, proj_b, proj_b + grid_floats);
}

extern "C" int nlam_latent_sample_supported(const NlamMlp* param_mlp, const NlamMlp* embed_mlp, const float* x, int64_t x_bs,
                                            const float* eps, int64_t eps_bs, const float* latent_emb, int64_t n_rows, int B,
                                            int flags) {
  if (!param_mlp || !embed_mlp) return 0;
  return tc_latent_supported(param_mlp, embed_mlp, x, x_bs, eps, eps_bs, latent_emb, n_rows, B, flags) ? 1 : 0;
}

extern "C" int nlam_latent_sample_fwd(const NlamMlp* param_mlp, const NlamMlp* embed_mlp, const float* x, int64_t x_bs,
                                      const float* eps, int64_t eps_bs, float* latent_emb, int64_t n_rows, int B, int flags,
                                      void* stream) {
  NLAM_REQUIRE(param_mlp && embed_mlp && x && eps && latent_emb, NLAM_E_INVALID, "nlam_latent_sample_fwd: null argument");
  NLAM_REQUIRE(nlam_latent_sample_supported(param_mlp, embed_mlp, x, x_bs, eps, eps_bs, latent_emb, n_rows, B, flags),
               NLAM_E_UNSUPPORTED, "nlam_latent_sample_fwd: shape / math mode not covered by the fused latent kernel");
  return tc_latent(param_mlp, embed_mlp, x, x_bs, eps, eps_bs, latent_emb, n_rows, B, flags, (cudaStream_t)stream);
}

extern "C" int nlam_inet_chain_supported(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp,
                                         const NlamMlp* next_edge_mlp, const float* send, int64_t send_bs, const float* rec,
                                         int64_t rec_bs, int B, int flags) {
  if (!g || !edge_mlp || !aggr_mlp || !send || !rec || B < 1 || edge_mlp->n_linear < 1) return 0;
  return chain_path(g, edge_mlp, aggr_mlp, next_edge_mlp, send, send_bs, rec, rec_bs, B, flags) ? 1 : 0;
}

static int inet_fwd_impl(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp, const NlamMlp* next_mlp,
                         const float* send, int64_t send_bs, const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs,
                         float* rec_out, float* edge_out, float* aggr_out, const float* proj_in, float* proj_out, int B, int flags,
                         void* workspace, size_t ws_bytes, void* stream);

extern "C" int nlam_inet_fwd(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp,
                             const float* send, int64_t send_bs, const float* rec, int64_t rec_bs,
                             const float* edge, int64_t edge_bs, float* rec_out, float* edge_out,
                             float* aggr_out, int B, int flags, void* workspace, size_t ws_bytes,
                             void* stream) {
  return inet_fwd_impl(g, edge_mlp, aggr_mlp, nullptr, send, send_bs, rec, rec_bs, edge, edge_bs, rec_out, edge_out, aggr_out,
                       nullptr, nullptr, B, flags, workspace, ws_bytes, stream);
}

extern "C" int nlam_inet_fwd_chain(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp,
                                   const NlamMlp* next_edge_mlp, const float* send, int64_t send_bs, const float* rec,
                                   int64_t rec_bs, const float* edge, int64_t edge_bs, float* rec_out, float* edge_out,
                                   float* aggr_out, const float* proj_in, float* proj_out, int B, int flags, void* workspace,
                                   size_t ws_bytes, void* stream) {
  NLAM_REQUIRE((next_edge_mlp != nullptr) == (proj_out != nullptr), NLAM_E_INVALID,
               "nlam_inet_fwd_chain: next_edge_mlp and proj_out go together");
  return inet_fwd_impl(g, edge_mlp, aggr_mlp, next_edge_mlp, send, send_bs, rec, rec_bs, edge, edge_bs, rec_out, edge_out, aggr_out,
                       proj_in, proj_out, B, flags, workspace, ws_bytes, stream);
}

static int inet_fwd_impl(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp, const NlamMlp* next_mlp,
                         const float* send, int64_t send_bs, const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs,
                         float* rec_out, float* edge_out, float* aggr_out, const float* proj_in, float* proj_out, int B, int flags,
                         void* workspace, size_t ws_bytes, void* stream) {
  const bool edge_only = flags & NLAM_EDGE_ONLY;
  NLAM_REQUIRE(g && edge_mlp && aggr_mlp && send && rec && edge && (rec_out || edge_only), NLAM_E_INVALID,
               "nlam_inet_fwd: null argument");
  NLAM_REQUIRE(!edge_only || aggr_out, NLAM_E_INVALID, "nlam_inet_fwd: NLAM_EDGE_ONLY needs aggr_out");
  NLAM_REQUIRE(B >= 1, NLAM_E_INVALID, "nlam_inet_fwd: bad batch");
  const int H = edge_mlp->out_dim[edge_mlp->n_linear - 1];
  NLAM_REQUIRE(edge_mlp->in_dim == 3 * H && aggr_mlp->in_dim == 2 * H &&
                   aggr_mlp->out_dim[aggr_mlp->n_linear - 1] == H,
               NLAM_E_INVALID, "nlam_inet_fwd: MLP widths inconsistent with H=%d", H);
  const bool chained = proj_in || next_mlp;
  // projections from nlam_encode_fwd: the grid -> mesh call on the tc_edge_bcast path
  const bool bcast_proj = proj_in && !next_mlp && !edge_out &&
                          bcast_path(g, edge_mlp, send, send_bs, rec, rec_bs, edge, edge_bs, B, flags);
  NLAM_REQUIRE(!chained || bcast_proj || chain_path(g, edge_mlp, aggr_mlp, next_mlp, send, send_bs, rec, rec_bs, B, flags),
               NLAM_E_UNSUPPORTED, "nlam_inet_fwd_chain: call shape without a chained path (see nlam_inet_chain_supported)");
  NLAM_REQUIRE(!next_mlp || ((((uintptr_t)rec_out | (uintptr_t)proj_out) & 15) == 0), NLAM_E_INVALID,
               "nlam_inet_fwd_chain: unaligned outputs");
  NLAM_REQUIRE(edge_out != edge || inplace_path(g, edge_mlp, send, send_bs, rec, rec_bs, edge, edge_bs, B, flags),
               NLAM_E_INVALID, "nlam_inet_fwd: edge_out aliases edge for a call shape without in-place support "
               "(see nlam_inet_inplace_supported)");
  cudaStream_t st = (cudaStream_t)stream;
  const int mean = (flags & (NLAM_AGGR_MEAN | NLAM_PROPAGATION)) ? 1 : 0;  // PropagationNet forces mean
  const bool prop = flags & NLAM_PROPAGATION;
  const size_t agg_bytes = rup256((size_t)B * g->n_rec * H * sizeof(float));
  const bool use_tc = want_tf32(flags) && tc_edge_supported(g, edge_mlp, flags);
  const bool use_gen = !use_tc && want_tf32(flags) &&
                       tc_inet_gen_supported(g, edge_mlp, aggr_mlp, flags, send, send_bs, rec, rec_bs, edge, edge_bs);
  const size_t scratch_bytes = inet_scratch_bytes(g, B, H, use_tc ? PATH_TC64 : use_gen ? PATH_GEN : PATH_EXACT);
  NLAM_REQUIRE(workspace && ws_bytes >= agg_bytes + scratch_bytes, NLAM_E_WORKSPACE,
               "nlam_inet_fwd: workspace too small (%zu < %zu bytes; see nlam_inet_workspace_bytes)", ws_bytes,
               agg_bytes + scratch_bytes);
  float* aggr = aggr_out ? aggr_out : (float*)workspace;
  float* scratch = (float*)((char*)workspace + agg_bytes);
  const int64_t aggr_bs = (int64_t)g->n_rec * H;

  NLAM_REQUIRE(use_tc || use_gen || !(flags & NLAM_MATH_TF32), NLAM_E_UNSUPPORTED,
               "nlam_inet_fwd: shape (H=%d, max in-degree %d, hidden_layers=%d) not supported by the tensor-core kernels",
               H, g->max_in_degree, edge_mlp->n_linear - 1);
  NLAM_REQUIRE(!(use_gen && edge_only), NLAM_E_UNSUPPORTED, "nlam_inet_fwd: NLAM_EDGE_ONLY is not available on the generic path");
  if (use_gen)
    return tc_inet_gen(g, edge_mlp, aggr_mlp, send, send_bs, rec, rec_bs, edge, edge_bs, rec_out, edge_out, aggr, B, flags,
                       scratch, st);

  if (use_tc) {
    // rows of the sender tensor: known exactly when the batches are dense, else at least n_send
    const int64_t send_rows = (B > 1 && send_bs > 0) ? send_bs / H : g->n_send;
    int rc;
    if (tc_ell_supported(g, edge_mlp, flags, send, send_bs, rec, rec_bs, edge_out != nullptr)) {
      // uniform in-degree edge sets (fused.cu)
      rc = tc_ell_edge(g, edge_mlp, send, send_bs, rec, rec_bs, edge, edge_bs, aggr, B, flags, st, scratch);
    } else if (tc_edge2_supported(g, edge_mlp, flags, send, send_bs, rec, rec_bs, B, send_rows)) {
      // split first Linear: node projections + K=64 edge kernel (fused.cu)
      // (tc_edge_rmw when the edge tensor is updated in place or not written at all)
      // (projections computed by the previous layer's node kernel: proj_in holds [P_s | P_r] in the scratch layout)
      float* pws = proj_in ? const_cast<float*>(proj_in) : scratch;
      if (tc_edge_rmw_supported(g, edge, edge_bs, edge_out, B))
        rc = tc_edge_rmw(g, edge_mlp, send, send_bs, rec, rec_bs, edge, edge_bs, edge_out, aggr, B, flags, st, pws, proj_in != nullptr);
      else
        rc = tc_edge3(g, edge_mlp, send, send_bs, rec, rec_bs, edge, edge_bs, edge_out, aggr, B, flags, st, pws, proj_in != nullptr);
    } else if (tc_edge_bcast_supported(g, edge_mlp, flags, send, send_bs, rec, rec_bs, edge, edge_bs, B, edge_out != nullptr)) {
      // batch-broadcast edge features and receivers, large sender set, no edge update (grid -> mesh): tile-major
      // K = 192 kernel on raw gathered sender rows (fused.cu)
      rc = tc_edge_bcast(g, edge_mlp, send, send_bs, rec, rec_bs, edge, aggr, B, flags, st,
                         proj_in ? const_cast<float*>(proj_in) : scratch, proj_in != nullptr);
    } else {
      rc = tc_edge(g, edge_mlp, send, send_bs, rec, rec_bs, edge, edge_bs, edge_out, aggr, B, flags, st, send_rows);
    }
    if (rc) return rc;
  } else {
    float* msg = scratch;
    NlamRowSrc srcs[3] = {{edge, nullptr, edge_bs, H, 0}, {send, g->src, send_bs, H, 0}, {rec, g->dst, rec_bs, H, 0}};
    NlamRowSrc res = {send, g->src, send_bs, H, 0};
    NlamRowSrc res2 = {edge, nullptr, edge_bs, H, 0};
    int rc = rowmlp_simt(edge_mlp, srcs, 3, prop ? &res : nullptr, edge_out ? &res2 : nullptr, msg, edge_out,
                         g->n_edges, B, st);
    if (rc) return rc;
    rc = nlam_segment_sum(g->rowptr, nullptr, g->n_rec, msg, (int64_t)g->n_edges * H, aggr, aggr_bs, B, H, mean, st);
    if (rc) return rc;
  }
  if (edge_only) return NLAM_OK;
  // node update: rec' = base + aggr_mlp(cat(rec, aggr)); base = rec (InteractionNet) or aggr (PropagationNet)
  NlamRowSrc nsrcs[2] = {{rec, nullptr, rec_bs, H, 0}, {aggr, nullptr, aggr_bs, H, 0}};
  NlamRowSrc nres = prop ? nsrcs[1] : nsrcs[0];
  if (next_mlp)  // node update + the next layer's node projections (fused.cu)
    return tc_node_proj(aggr_mlp, next_mlp, rec, rec_bs, aggr, g->n_rec, B, rec_out, proj_out, st);
  if (use_tc && tc_rowmlp_supported(aggr_mlp, nsrcs, 2, &nres, nullptr, g->n_rec))
    return tc_rowmlp(aggr_mlp, nsrcs, 2, &nres, rec_out, g->n_rec, B, st);
  return rowmlp_simt(aggr_mlp, nsrcs, 2, &nres, nullptr, rec_out, nullptr, g->n_rec, B, st);
}

extern "C" size_t nlam_ensemble_stats_workspace_bytes(int B, int64_t G, int d) {
  return (B >= 1 && G >= 1 && d >= 1) ? ens_stats_workspace_bytes(B, G, d) : 0;
}

extern "C" int nlam_ensemble_stats(const float* members, int64_t member_bstride, int64_t member_kstride, int B, int K,
                                   int64_t G, int d, const float* target, int64_t target_bstride, const float* interior,
                                   float* mean, float* std, float* scores, void* workspace, size_t ws_bytes, void* stream) {
  NLAM_REQUIRE(members && mean && std && B >= 1 && G >= 1 && d >= 1, NLAM_E_INVALID, "nlam_ensemble_stats: bad arguments");
  NLAM_REQUIRE(!scores || (target && interior), NLAM_E_INVALID, "nlam_ensemble_stats: scores need a target and an interior mask");
  return ens_stats(members, member_bstride, member_kstride, B, K, G, d, target, target_bstride, interior, mean, std, scores,
                   workspace, ws_bytes, (cudaStream_t)stream);
}

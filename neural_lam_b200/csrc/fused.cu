// Fused H = 64 kernels for sm_90a (wgmma TF32, fp32 accumulate): one CTA works on tiles of 128 rows (node rows, or the CSR
// edges of whole receivers), two warp groups own 64 rows each.  Per tile:
//
//   A  = [src_0 | src_1 | ...] rows (gathered through row indices, zero-padded to a multiple of 32 columns) -> shared memory
//   h  = SiLU(A · W1ᵀ + b1)                                wgmma, accumulators in registers, h back to shared memory
//   y  = LN(h · W2ᵀ + b2) [+ residual]                     wgmma
//
// then one of: the row output (optionally the forecast-step epilogue), or the edge output e' = e + y together with the
// deterministic per-receiver sum of y over the tile's edges (every receiver lies in one tile).  All weights of a launch
// stay in shared memory for the whole persistent CTA; operands are written in the 128-byte swizzle wgmma reads, and every
// generic-proxy write of an operand is followed by fence.proxy.async before the warp group's MMAs read it.
//
// Launch names (nlam_profile_*): tc_rowmlp_kernel (row MLPs, output_map + step epilogue), tc_rowlinear_kernel (node
// projections P_s = x_s·W1sᵀ, P_r = x_r·W1rᵀ + b1 of the split first edge Linear, both node sets in one grid), tc_edge_kernel
// (K = 192 edge MLP on raw gathered rows).  The other kernels of this file each run one job: the node updates
// (tc_node_proj_kernel, tc_node_out_kernel and the node-update form of tc_rowmlp_kernel) run on tc_node_kernel, the whole
// mesh -> grid decoder of a forecast step on tc_decode_kernel.  The split-form edge stage
// (first edge Linear split into e·W1eᵀ and node projections gathered in its epilogue) runs in tc_edge_split_kernel below
// (tc_edge_split).  tc_edge_path decides, in one place, whether an edge stage takes the split or the K = 192 form and under
// which label the split kernel is launched: tc_edge3_kernel (out-of-place edge output), tc_edge_rmw_kernel (edge tensor
// updated in place or not written), tc_ell_window_kernel (uniform in-degree edge sets) or tc_edge_bcast_kernel
// (batch-broadcast edge features and receivers).
#include "tc_ptx.cuh"
#include "wgmma_tf32.cuh"

namespace nlam {

namespace fz {
constexpr int THREADS = 256;
constexpr uint32_t CH_A = 128 * 128;  // one 32-column chunk of a 128-row operand
constexpr uint32_t CH_W = 64 * 128;   // one 32-column chunk of a 64-row weight
constexpr uint32_t OFF_A = 0;
enum Mode { ROWS = 0, EDGE = 1, ROWLIN = 2 };
// Shared memory, sized per launch so that the K = 64 launches fit two CTAs per SM:
//   A (max(kc1, 2) chunks) | W1 (kc1 chunks) | W2 (2) | EDGE: the 128 x 64 fp32 message buffer, ROWLIN: W3 (2)
//   | b1 | b2 | gamma | beta | b1 of problem 1 (64 floats each, in a block of 7: the launch sizes, and with them the CTAs
//   per SM, are those the kernel was tuned and measured at)
struct Layout {
  uint32_t w1, w2, w3, prm, bytes;
};
__host__ __device__ inline Layout layout(int kc1, int mode) {
  Layout l;
  l.w1 = (uint32_t)(kc1 > 2 ? kc1 : 2) * CH_A;
  l.w2 = l.w1 + (uint32_t)kc1 * CH_W;
  l.w3 = l.w2 + 2 * CH_W;
  l.prm = l.w3 + (mode == EDGE ? 4 * CH_W : mode == ROWLIN ? 2 * CH_W : 0);
  l.bytes = l.prm + 7 * 64 * 4 + 1024;  // + alignment slack
  return l;
}
}  // namespace fz

struct FzSrc {
  const float* ptr;
  const int32_t* idx;  // row r reads row idx[r] (NULL: row r)
  long long bs;        // batch stride in elements (0: broadcast)
  int dim;
};
struct FzW {           // rows x cols slice of a row-major matrix with row pitch ld
  const float* ptr;
  int ld, rows, cols;
};

struct FzParams {
  int mode, B, kc1, n_src;
  FzSrc src[4];
  FzW w1, w2, w3;
  const float *b1, *b2, *gamma, *beta;
  float eps;
  int act1, has_gemm2;
  const float* res;     // residual rows (64 wide)
  long long res_bs;
  float* out;           // (B, n_rows, out_w)
  int out_w;
  long long n_rows;
  int n_tiles;
  // EDGE
  const int32_t* tile_rec;
  const int32_t* rowptr;
  int mean;
  const float* edge;
  long long edge_bs;
  float* edge_out;      // (B, n_edges, 64) dense
  float* aggr;          // (B, n_rec, 64) dense
  long long n_rec, n_edges;
  // forecast-step epilogue on the final narrow output (width out_w)
  int step;
  const float *prev, *bnd, *mask, *dstd, *dmean;
  // ROWLIN problem 1 (problem 0 = src[0], w1, b1, out, n_rows, n_tiles, B): weights in the W3 slot
  FzSrc src1;
  const float* b1_1;
  float* out_1;
  long long n_rows1;
  int n_tiles1, B1;
  float* std_out;       // predicted-std form of the step epilogue (fused_mlp_kernel<true>): (B, n_rows, out_w / 2)
};

// byte offset of operand element (row R, column c) in a 128B-swizzled operand stored as 32-column chunks
__device__ __forceinline__ uint32_t fz_off(uint32_t chunk_bytes, int R, int c) {
  return (uint32_t)(c >> 5) * chunk_bytes + swz(R, (c & 31) >> 2) + (uint32_t)(c & 3) * 4;
}

__device__ void fz_load_w(uint8_t* s, const FzW& w, int kc, int tid) {
  // rows 0..63 x 32*kc columns, zero past the real rows / columns
  const int groups = 64 * kc * 8;
  for (int g = tid; g < groups; g += fz::THREADS) {
    const int n = g / (kc * 8), c = (g % (kc * 8)) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (w.ptr && n < w.rows) {
      const float* p = w.ptr + (long long)n * w.ld + c;
      if (c + 0 < w.cols) v.x = p[0];
      if (c + 1 < w.cols) v.y = p[1];
      if (c + 2 < w.cols) v.z = p[2];
      if (c + 3 < w.cols) v.w = p[3];
    }
    *reinterpret_cast<float4*>(s + fz_off(fz::CH_W, n, c)) = tf32r4(v);
  }
}

// A tile: rows row0 .. row0 + nrows - 1 of the concatenated sources (batch b), zero-padded to 32 * kc columns
__device__ void fz_load_a(uint8_t* s, const FzSrc* src, int n_src, int kc, int b, long long row0, int nrows, int tid) {
  const int gpr = kc * 8;
  for (int g = tid; g < 128 * gpr; g += fz::THREADS) {
    const int i = g / gpr, c = (g % gpr) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < nrows) {
      const long long r = row0 + i;
      float* pv = &v.x;
      int off = 0;
      for (int q = 0; q < n_src; ++q) {
        const FzSrc& sq = src[q];
        // vector load only for a whole group at a 16-byte aligned position of one source (rows of a width % 4 == 0)
        if (c >= off && c + 4 <= off + sq.dim && ((c - off) & 3) == 0 && (sq.dim & 3) == 0) {
          const long long rr = sq.idx ? (long long)__ldg(sq.idx + r) : r;
          v = __ldg(reinterpret_cast<const float4*>(sq.ptr + b * sq.bs + rr * sq.dim + (c - off)));
          break;
        }
        for (int e = 0; e < 4; ++e) {
          const int cc = c + e - off;
          if (cc >= 0 && cc < sq.dim) {
            const long long rr = sq.idx ? (long long)__ldg(sq.idx + r) : r;
            pv[e] = __ldg(sq.ptr + b * sq.bs + rr * sq.dim + cc);
          }
        }
        off += sq.dim;
      }
    }
    *reinterpret_cast<float4*>(s + fz_off(fz::CH_A, i, c)) = tf32r4(v);
  }
}

// warp group MMA: acc (64 rows of this warp group x 64) = A[rows] · Wᵀ over kc chunks
__device__ __forceinline__ void fz_gemm(float* acc, uint32_t a, uint32_t w, int kc) {
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  wgmma_fence(acc, 32);
  for (int c = 0; c < kc; ++c) {
    const uint64_t da = gmma_desc(a + c * fz::CH_A), db = gmma_desc(w + c * fz::CH_W);
#pragma unroll
    for (int k = 0; k < 4; ++k) Wgmma<64>::mma(acc, da + 2 * k, db + 2 * k, (uint32_t)((c | k) != 0));
  }
  wgmma_commit();
  wgmma_wait0(acc, 32);
}

// fragment of m64n64: acc[4j + 2i + e] is local row rq + 8i, column 8j + cq + e
__device__ __forceinline__ void fz_unpack(const float* acc, float (*v)[16], const float* bias) {
  const int cq = 2 * (threadIdx.x & 3);
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) v[i][2 * j + e] = acc[4 * j + 2 * i + e] + (bias ? bias[8 * j + cq + e] : 0.f);
}

// this warp group's rows of v -> shared-memory operand (chunks 0-1 of A), then make them visible to its MMAs
__device__ __forceinline__ void fz_store_op(uint8_t* sA, float (*v)[16], int rq, int wg) {
  const int cq = 2 * (threadIdx.x & 3);
  named_bar_sync(1 + wg, 128);  // every MMA of this warp group has finished reading the rows being replaced
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<float2*>(sA + fz_off(fz::CH_A, rq + 8 * i, 8 * j + cq)) =
          make_float2(tf32r(v[i][2 * j]), tf32r(v[i][2 * j + 1]));
  fence_proxy_async();
  named_bar_sync(1 + wg, 128);
}

__device__ __forceinline__ void fz_layernorm(float (*v)[16], const float* gamma, const float* beta, float eps) {
  const int cq = 2 * (threadIdx.x & 3);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float mu, rstd;
    quad_row_stats<16>(v[i], eps, mu, rstd);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = 8 * j + cq + e;
        v[i][2 * j + e] = fmaf((v[i][2 * j + e] - mu) * rstd, gamma[c], beta[c]);
      }
  }
}

// add 64-wide rows base[row(i)] (+ column offset of this thread) to v; row(i) < 0: skipped
__device__ __forceinline__ void fz_add_rows(float (*v)[16], const float* p0, const float* p1) {
  const int cq = 2 * (threadIdx.x & 3);
  const float* p[2] = {p0, p1};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (!p[i]) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 x = __ldg(reinterpret_cast<const float2*>(p[i] + 8 * j + cq));
      v[i][2 * j] += x.x;
      v[i][2 * j + 1] += x.y;
    }
  }
}

// this thread's 16 columns of one fragment row -> a 64-wide output row
__device__ __forceinline__ void fz_store_row64(float* row, const float* v) {
  const int cq = 2 * (threadIdx.x & 3);
#pragma unroll
  for (int j = 0; j < 8; ++j) *reinterpret_cast<float2*>(row + 8 * j + cq) = make_float2(v[2 * j], v[2 * j + 1]);
}

// narrow / full-width row store with the optional forecast-step epilogue (P: FzParams, DecParams or NodeParams).
// STD (the predicted-std form of the step epilogue): the W = 2d outputs are d state deltas, then d raw stds.  Column c < d
// takes the step epilogue, column d + c is stored as std_out[b, r, c] = softplus(y) with torch's threshold 20 and without
// the boundary mix; prev, boundary, the new state and std_out have rows of d.
template <bool STD = false, class P>
__device__ __forceinline__ void fz_store_rows(const P& p, float* out, int W, long long n_rows, bool step, float (*v)[16],
                                              int b, long long r0, bool valid0, bool valid1) {
  const int cq = 2 * (threadIdx.x & 3);
  const int Ws = STD ? W >> 1 : W;  // row pitch of the stored rows
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (!(i ? valid1 : valid0)) continue;
    const long long r = r0 + 8 * i;
    const long long o = ((long long)b * n_rows + r) * Ws;
    if (step) {
      const float mk = p.bnd ? __ldg(p.mask + r) : 0.f;
#pragma unroll
      for (int t = 0; t < 16; ++t) {
        const int c = 8 * (t >> 1) + cq + (t & 1);
        if (c < Ws) {
          const float nw = __ldg(p.prev + o + c) + (v[i][t] * __ldg(p.dstd + c) + __ldg(p.dmean + c));
          out[o + c] = p.bnd ? mk * __ldg(p.bnd + o + c) + (1.f - mk) * nw : nw;
        } else if (STD && c < W) {
          const float y = v[i][t];
          p.std_out[o + c - Ws] = y > 20.f ? y : log1pf(expf(y));
        }
      }
    } else if (W == 64) {
      fz_store_row64(out + o, v[i]);
    } else {
#pragma unroll
      for (int t = 0; t < 16; ++t) {
        const int c = 8 * (t >> 1) + cq + (t & 1);
        if (c < W) out[o + c] = v[i][t];
      }
    }
  }
}

template <bool STD>  // STD: the step epilogue's predicted-std form (fz_store_rows)
__global__ void __launch_bounds__(fz::THREADS, 2) fused_mlp_kernel(const __grid_constant__ FzParams p) {
  using namespace fz;
  const Layout L = layout(p.kc1, p.mode);
  const uint32_t OFF_W1 = L.w1, OFF_W2 = L.w2, OFF_W3 = L.w3, OFF_PRM = L.prm;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* s = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t sb = smem_u32(s);
  uint8_t* sA = s + OFF_A;
  float* prm = reinterpret_cast<float*>(s + OFF_PRM);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2;
  const int rq = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // local row of fragment half 0 (half 1: + 8)
  const int cq = 2 * (lane & 3);

  fz_load_w(s + OFF_W1, p.w1, p.kc1, tid);
  if (p.has_gemm2) fz_load_w(s + OFF_W2, p.w2, 2, tid);
  if (p.mode == ROWLIN) fz_load_w(s + OFF_W3, p.w3, 2, tid);
  for (int i = tid; i < 64; i += THREADS) {
    prm[i] = p.b1 ? p.b1[i] : 0.f;
    prm[64 + i] = p.b2 ? p.b2[i] : 0.f;
    prm[128 + i] = p.gamma ? p.gamma[i] : 1.f;
    prm[192 + i] = p.beta ? p.beta[i] : 0.f;
    prm[256 + i] = p.b1_1 ? p.b1_1[i] : 0.f;
  }
  const long long n_work0 = (long long)p.n_tiles * p.B;
  const long long n_work = n_work0 + (p.mode == ROWLIN ? (long long)p.n_tiles1 * p.B1 : 0);
  float acc[32];
  float v[2][16];
  for (long long w = blockIdx.x; w < n_work; w += gridDim.x) {
    // ------------------------------------------------------------------ which rows
    int b, prob = 0;
    long long t;
    if (w < n_work0) {
      b = (int)(w / p.n_tiles);
      t = w - (long long)b * p.n_tiles;
    } else {
      prob = 1;
      b = (int)((w - n_work0) / p.n_tiles1);
      t = (w - n_work0) - (long long)b * p.n_tiles1;
    }
    long long row0;
    int nrows;
    if (p.mode == EDGE) {
      const int ra = __ldg(p.tile_rec + t), rb = __ldg(p.tile_rec + t + 1);
      row0 = __ldg(p.rowptr + ra);
      nrows = __ldg(p.rowptr + rb) - (int)row0;
    } else {
      const long long n = prob ? p.n_rows1 : p.n_rows;
      row0 = t * 128;
      nrows = (int)min(128LL, n - row0);
    }
    __syncthreads();  // the previous tile's readers of the operand / message buffers are done
    if (prob == 0) fz_load_a(sA, p.src, p.n_src, p.kc1, b, row0, nrows, tid);
    else fz_load_a(sA, &p.src1, 1, p.kc1, b, row0, nrows, tid);
    fence_proxy_async();
    __syncthreads();
    // ------------------------------------------------------------------ GEMM 1
    fz_gemm(acc, sb + OFF_A + wg * (CH_A / 2), sb + (prob ? OFF_W3 : OFF_W1), p.kc1);
    const long long r0 = row0 + rq;
    const bool valid0 = rq < nrows, valid1 = rq + 8 < nrows;
    fz_unpack(acc, v, prm + (prob ? 256 : 0));
    if (p.mode == ROWLIN) {
      fz_store_rows(p, prob ? p.out_1 : p.out, 64, prob ? p.n_rows1 : p.n_rows, false, v, b, r0, valid0, valid1);
      continue;
    }
    if (p.act1) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int t2 = 0; t2 < 16; ++t2) v[i][t2] = silu_fast(v[i][t2]);
    }
    // ------------------------------------------------------------------ GEMM 2
    fz_store_op(sA, v, rq, wg);
    fz_gemm(acc, sb + OFF_A + wg * (CH_A / 2), sb + OFF_W2, 2);
    fz_unpack(acc, v, prm + 64);
    if (p.gamma) fz_layernorm(v, prm + 128, prm + 192, p.eps);
    if (p.mode == EDGE) {
      // e' = e + m; m -> message buffer (row = local edge), then the per-receiver sums of the tile
      if (p.edge_out) {
        const float* e = p.edge + (long long)b * p.edge_bs;
        float* eo = p.edge_out + (long long)b * p.n_edges * 64;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          if (!(i ? valid1 : valid0)) continue;
          const long long k = r0 + 8 * i;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float2 x = *reinterpret_cast<const float2*>(e + k * 64 + 8 * j + cq);
            *reinterpret_cast<float2*>(eo + k * 64 + 8 * j + cq) = make_float2(x.x + v[i][2 * j], x.y + v[i][2 * j + 1]);
          }
        }
      }
      float* msg = reinterpret_cast<float*>(s + OFF_W3);
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<float2*>(msg + (rq + 8 * i) * 64 + 8 * j + cq) = make_float2(v[i][2 * j], v[i][2 * j + 1]);
      __syncthreads();
      const int ra = __ldg(p.tile_rec + t), nrec = __ldg(p.tile_rec + t + 1) - ra;
      for (int x = tid; x < nrec * 16; x += THREADS) {
        const int rr = x >> 4, c4 = (x & 15) * 4;
        const int k0 = __ldg(p.rowptr + ra + rr) - (int)row0, k1 = __ldg(p.rowptr + ra + rr + 1) - (int)row0;
        float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int k = k0; k < k1; ++k) {
          const float4 m = *reinterpret_cast<const float4*>(msg + k * 64 + c4);
          sum.x += m.x; sum.y += m.y; sum.z += m.z; sum.w += m.w;
        }
        if (p.mean) {
          const float sc = 1.f / (float)max(k1 - k0, 1);
          sum.x *= sc; sum.y *= sc; sum.z *= sc; sum.w *= sc;
        }
        *reinterpret_cast<float4*>(p.aggr + ((long long)b * p.n_rec + ra + rr) * 64 + c4) = sum;
      }
      continue;
    }
    if (p.res) {
      const float* base = p.res + (long long)b * p.res_bs;
      fz_add_rows(v, valid0 ? base + r0 * 64 : nullptr, valid1 ? base + (r0 + 8) * 64 : nullptr);
    }
    fz_store_rows<STD>(p, p.out, p.out_w, p.n_rows, p.step, v, b, r0, valid0, valid1);
  }
}

// ------------------------------------------------------------------------------------ split-form edge kernel
// The edge stage of an InteractionNet layer whose first edge Linear is split, P_s = x_s·W1sᵀ and P_r = x_r·W1rᵀ + b1 given.
// Per CSR tile (whole receivers, <= 128 edges) of batch element b, the arithmetic of fused_mlp_kernel's EDGE mode:
//   m     = LN(SiLU(e·W1eᵀ + P_s[b, src[k]] + P_r[b, dst[k]])·W2ᵀ + b2)
//   e'    = e + m                         (optional: out of place, in place, or not written)
//   aggr  = sum (or mean) of m over each receiver's edges, k0 to k1 in CSR order
// __launch_bounds__(256, 1): one persistent CTA per SM, each warp group owns 64 rows of the tile.  The whole load chain of
// the next tile runs while this tile computes: its edge rows (one contiguous 16-byte aligned span per batch element) and
// its rowptr entries are copied with cp.async into raw staging buffers before this tile's GEMMs, and its gathered P_s / P_r
// rows right after this tile's GEMM 1 epilogue has read its own.  The tile bounds come two tiles ahead and the src / dst
// indices one tile ahead, so no copy waits on the load of its address.  The raw staged e rows are rounded to TF32 (to
// nearest) as they become the operand, and the residual e + m reads them from staging; the staging buffer then holds the
// tile's messages for the per-receiver sums.
namespace edg {
using fz::CH_A;
using fz::CH_W;
constexpr int PITCH = 72;  // staged rows: 64 floats + 8 (fragment-layout float2 reads of a half warp hit distinct banks)
constexpr uint32_t STG_BYTES = 128 * PITCH * 4;
constexpr uint32_t W1 = 0, W2 = W1 + 2 * CH_W;
constexpr uint32_t A = W2 + 2 * CH_W;          // 128 x 64 operand
constexpr uint32_t STG = A + 2 * CH_A;         // two raw edge-row staging buffers (tiles of even / odd iteration)
constexpr uint32_t PS = STG + 2 * STG_BYTES;   // staged P_s[src] rows of one tile
constexpr uint32_t PR = PS + STG_BYTES;        // staged P_r[dst] rows of one tile
constexpr uint32_t RP = PR + STG_BYTES;        // two copies of a tile's rowptr entries (<= 129)
constexpr uint32_t PRM = RP + 2 * 132 * 4;     // b2 | gamma | beta
constexpr uint32_t BYTES = PRM + 3 * 64 * 4 + 1024;  // + alignment slack
static_assert(BYTES <= 227 * 1024, "edge kernel shared memory exceeds the sm_90 limit");
}  // namespace edg

struct EdgeParams {
  int B, n_tiles, mean;
  const int32_t *tile_rec, *tile_edge, *rowptr, *src, *dst;
  const float* edge;     // (B | 1, n_edges, 64), batch stride edge_bs (0: shared by the batch)
  long long edge_bs;
  float* edge_out;       // NULL, edge (in place) or (B, n_edges, 64) dense
  float* aggr;           // (B, n_rec, 64) dense
  const float *ps, *pr;  // P_s (B | 1, n_send, 64), P_r (B | 1, n_rec, 64)
  long long ps_bs, pr_bs;
  FzW w1, w2;
  const float *b2, *gamma, *beta;
  float eps;
  long long n_rec, n_edges;
};

struct EdgeTile {
  int b, ra, rb, row0, nrows;  // b < 0: no such tile
};

__device__ __forceinline__ EdgeTile edge_tile(const EdgeParams& p, long long w, long long n_work) {
  EdgeTile T{-1, 0, 0, 0, 0};
  if (w < n_work) {
    T.b = (int)(w / p.n_tiles);
    const int t = (int)(w - (long long)T.b * p.n_tiles);
    T.ra = __ldg(p.tile_rec + t);
    T.rb = __ldg(p.tile_rec + t + 1);
    T.row0 = __ldg(p.tile_edge + t);
    T.nrows = __ldg(p.tile_edge + t + 1) - T.row0;
  }
  return T;
}

__global__ void __launch_bounds__(fz::THREADS, 1) tc_edge_split_kernel(const __grid_constant__ EdgeParams p) {
  using namespace fz;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* s = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t sb = smem_u32(s);
  uint8_t* sA = s + edg::A;
  float* prm = reinterpret_cast<float*>(s + edg::PRM);
  const float* sps = reinterpret_cast<const float*>(s + edg::PS);
  const float* spr = reinterpret_cast<const float*>(s + edg::PR);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2, gt = tid & 127, bar = 1 + wg;
  const int rq = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // local row of fragment half 0 (half 1: + 8)
  const int cq = 2 * (lane & 3);
  const uint32_t aA = sb + edg::A + wg * (CH_A / 2);

  fz_load_w(s + edg::W1, p.w1, 2, tid);
  fz_load_w(s + edg::W2, p.w2, 2, tid);
  for (int i = tid; i < 64; i += THREADS) {
    prm[i] = p.b2 ? p.b2[i] : 0.f;
    prm[64 + i] = p.gamma ? p.gamma[i] : 1.f;
    prm[128 + i] = p.beta ? p.beta[i] : 0.f;
  }

  const long long n_work = (long long)p.n_tiles * p.B, stride = gridDim.x;
  const uint64_t pol_stream = policy_evict_first(), pol_shared = policy_evict_normal();
  const uint64_t pol_e = p.edge_bs ? pol_stream : pol_shared;
  // the edge rows and rowptr entries of tile T -> staging buffer `buf`
  auto issue_edges = [&](const EdgeTile& T, int buf) {
    if (T.b < 0) return;
    const float* g = p.edge + (long long)T.b * p.edge_bs + (long long)T.row0 * 64;
    const uint32_t dst = sb + edg::STG + buf * edg::STG_BYTES;
    for (int k = tid; k < T.nrows * 16; k += THREADS)
      cp_async_16(dst + 4u * (uint32_t)((k >> 4) * edg::PITCH + (k & 15) * 4), g + 4 * k, pol_e);
    const uint32_t rp = sb + edg::RP + buf * 132 * 4;
    for (int x = tid; x <= T.rb - T.ra; x += THREADS) cp_async_4(rp + 4u * x, p.rowptr + T.ra + x);
  };
  // this thread's gather rows of tile T: row 64 wg + (gt >> 4) + 8 q, 16-byte piece gt & 15 (-1: past the tile's edges)
  int sidx[8], didx[8];
  auto load_idx = [&](const EdgeTile& T) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int r = 64 * wg + (gt >> 4) + 8 * q;
      const bool ok = T.b >= 0 && r < T.nrows;
      sidx[q] = ok ? __ldg(p.src + T.row0 + r) : -1;
      didx[q] = ok ? __ldg(p.dst + T.row0 + r) : -1;
    }
  };
  auto issue_proj = [&](const EdgeTile& T) {
    if (T.b < 0) return;
    const float* ps = p.ps + (long long)T.b * p.ps_bs + (gt & 15) * 4;
    const float* pr = p.pr + (long long)T.b * p.pr_bs + (gt & 15) * 4;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      if (sidx[q] < 0) continue;
      const uint32_t o = 4u * (uint32_t)((64 * wg + (gt >> 4) + 8 * q) * edg::PITCH + (gt & 15) * 4);
      cp_async_16(sb + edg::PS + o, ps + (long long)sidx[q] * 64, pol_shared);
      cp_async_16(sb + edg::PR + o, pr + (long long)didx[q] * 64, pol_shared);
    }
  };

  // Every thread commits one cp.async group per issue call, empty or not, so that the groups pending at each wait are the
  // same for all threads: the edge group of tile j + 1 is committed before tile j's GEMM 1, its projection group after it.
  EdgeTile cur = edge_tile(p, blockIdx.x, n_work), nxt = edge_tile(p, blockIdx.x + stride, n_work);
  load_idx(cur);
  issue_edges(cur, 0);
  cp_async_commit();
  issue_proj(cur);
  cp_async_commit();
  load_idx(nxt);
  float acc[32];
  float v[2][16];
  int buf = 0;
  for (long long w = blockIdx.x; w < n_work; w += stride, buf ^= 1) {
    float* stg = reinterpret_cast<float*>(s + edg::STG + buf * edg::STG_BYTES);
    const int* rp = reinterpret_cast<const int*>(s + edg::RP + buf * 132 * 4);
    const int nrows = cur.nrows;
    // ---- 1. staged edge rows -> operand (TF32, zero rows past the tile's edges)
    cp_async_wait_group<1>();  // this tile's edge group has landed (its projection group may still be in flight)
    __syncthreads();           // ... for every thread; the previous tile's MMAs and message-buffer readers are done
    for (int g = tid; g < 128 * 16; g += THREADS) {
      const int i = g >> 4, c = (g & 15) * 4;
      const float4 x = i < nrows ? *reinterpret_cast<const float4*>(stg + i * edg::PITCH + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(sA + fz_off(CH_A, i, c)) = tf32r4(x);
    }
    fence_proxy_async();
    __syncthreads();
    // ---- 2. the next tile's edge rows -> the other staging buffer, whose last readers (tile j - 1's per-receiver sums) are
    // done.  In place (edge_out == edge) this never reads a row this CTA or another one writes: tiles are disjoint CSR
    // edge ranges, each (batch element, tile) belongs to one CTA, and this tile's e' rows are written only after its own
    // rows were staged.  Then the bounds of the tile after next.
    issue_edges(nxt, buf ^ 1);
    cp_async_commit();
    const EdgeTile nn = edge_tile(p, w + 2 * stride, n_work);
    // ---- 3. GEMM 1, + P_s[src] + P_r[dst], SiLU
    fz_gemm(acc, aA, sb + edg::W1, 2);
    const bool valid0 = rq < nrows, valid1 = rq + 8 < nrows;
    fz_unpack(acc, v, nullptr);
    cp_async_wait_group<1>();  // this tile's projection group has landed (the next tile's edge group may be in flight)
    named_bar_sync(bar, 128);  // ... for the warp group that gathered (and now reads) its rows
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const float* pa = a ? spr : sps;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (!(i ? valid1 : valid0)) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float2 x = *reinterpret_cast<const float2*>(pa + (rq + 8 * i) * edg::PITCH + 8 * j + cq);
          v[i][2 * j] += x.x;
          v[i][2 * j + 1] += x.y;
        }
      }
    }
    named_bar_sync(bar, 128);  // the warp group's reads of the staged projections are done: gather the next tile's
    issue_proj(nxt);
    cp_async_commit();
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t2 = 0; t2 < 16; ++t2) v[i][t2] = silu_fast(v[i][t2]);
    // ---- 4. GEMM 2, LayerNorm
    fz_store_op(sA, v, rq, wg);
    fz_gemm(acc, aA, sb + edg::W2, 2);
    fz_unpack(acc, v, prm);
    fz_layernorm(v, prm + 64, prm + 128, p.eps);
    load_idx(nn);  // the indices of the tile after next, used after the next tile's GEMM 1
    // ---- 5. e' = e + m from the staged e rows; m over them (each thread reads, then overwrites, its own positions)
    const int b = cur.b;
    float* eo = p.edge_out ? p.edge_out + (long long)b * p.n_edges * 64 : nullptr;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = rq + 8 * i;
      const long long k = (long long)cur.row0 + r;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float2* px = reinterpret_cast<float2*>(stg + r * edg::PITCH + 8 * j + cq);
        if (eo && (i ? valid1 : valid0)) {
          const float2 x = *px;
          *reinterpret_cast<float2*>(eo + k * 64 + 8 * j + cq) = make_float2(x.x + v[i][2 * j], x.y + v[i][2 * j + 1]);
        }
        *px = make_float2(v[i][2 * j], v[i][2 * j + 1]);
      }
    }
    __syncthreads();
    // ---- 6. per-receiver sums over the tile's messages
    const int ra = cur.ra, nrec = cur.rb - ra;
    for (int x = tid; x < nrec * 16; x += THREADS) {
      const int rr = x >> 4, c4 = (x & 15) * 4;
      const int k0 = rp[rr] - cur.row0, k1 = rp[rr + 1] - cur.row0;
      float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int k = k0; k < k1; ++k) {
        const float4 m = *reinterpret_cast<const float4*>(stg + k * edg::PITCH + c4);
        sum.x += m.x; sum.y += m.y; sum.z += m.z; sum.w += m.w;
      }
      if (p.mean) {
        const float sc = 1.f / (float)max(k1 - k0, 1);
        sum.x *= sc; sum.y *= sc; sum.z *= sc; sum.w *= sc;
      }
      *reinterpret_cast<float4*>(p.aggr + ((long long)b * p.n_rec + ra + rr) * 64 + c4) = sum;
    }
    cur = nxt;
    nxt = nn;
  }
  cp_async_wait_group<0>();  // no copy outlives the CTA
}

// ------------------------------------------------------------------------------------ mesh -> grid decoder
// The whole decoder of a forecast step in one kernel, for a uniform in-degree m2g graph (d in {1, 2, 4, 8}, receiver-sorted,
// edge features shared by the batch).  Per receiver r of batch element b, with P_e = e·W1eᵀ + b1 and P_s = send·W1sᵀ from
// one tc_rowlinear_kernel launch before it:
//   P_r   = rec[b, r]·W1rᵀ                                    (fp32, on chip)
//   m_k   = LN(SiLU(P_e[k] + P_s[b, src[k]] + P_r)·W2ᵀ + b2)  for the d edges k of r
//   aggr  = sum (or mean) of the m_k                          (warp shuffles, on chip)
//   grid' = rec + LN(SiLU([rec | aggr]·Wn1ᵀ + bn1)·Wn2ᵀ + bn2)
//   new   = step epilogue of SiLU(grid'·Wo1ᵀ + bo1)·Wo2ᵀ + bo2
// A work item is 64 receivers of one batch element.  The CTA is warp-specialized: warp group 0 loads, warp groups 1 and 2
// compute, one item at a time each; items run batch-fastest, so the B items of one receiver block run at about the same
// time and read its P_e rows from L2.  Half of the load warp group (64 threads) feeds each compute warp group through a
// ring of RING units in shared memory, 64 rows x 64 fp32 each in the operands' 128-byte swizzle, signalled by full / empty
// mbarriers.  Per item the stream is the receiver rows, then for each sub-tile of 64 edges the sums P_e[k] + P_s[b, src[k]]
// (added by the load warps in the order the edge pre-activation adds them).  The load warps hold a whole unit in flight in
// registers and fetch the next sub-tile's sender indices behind it, and they prefetch the item's previous / boundary state
// rows into L2 for the epilogue.  The compute warps read the receiver rows from the ring in fp32 into the accumulator
// layout (the residual, kept in registers) and round them in place to TF32 for P_r and the first half of node GEMM 1
// (K = 64 of 128, its accumulators kept in registers), which frees the unit one item ahead; each sub-tile's SiLU(...) is
// written (TF32) over the sums it was computed from and is the edge GEMM's operand.  Every operand is rounded to nearest
// before an MMA reads it, and every sum, K order and rounding point is that of the node-update and edge paths.
namespace dec {
using fz::CH_A;
using fz::CH_W;
constexpr int THREADS = 384;  // warp group 0 loads, warp groups 1 and 2 compute
constexpr int RING = 2;       // ring units per compute warp group
constexpr uint32_t W1R = 0, W2E = W1R + 2 * CH_W, WN1 = W2E + 2 * CH_W, WN2 = WN1 + 4 * CH_W, WO1 = WN2 + 2 * CH_W,
                   WO2 = WO1 + 2 * CH_W;
constexpr uint32_t NODE = WO2 + 2 * CH_W;  // 128 x 64 operand, 64 rows per compute warp group: P_r (fp32), then aggr, then
                                           // the node / output GEMMs' operands
constexpr uint32_t SLOT = 2 * CH_A;        // one ring slot: 128 x 64, the unit of compute warp group c in rows 64c ..
constexpr uint32_t RINGS = NODE + 2 * CH_A;
constexpr uint32_t PRM = RINGS + RING * SLOT;  // b2, gamma, beta (edge MLP) | bn1, bn2, gamma, beta (node MLP) | bo1, bo2
constexpr uint32_t BAR = PRM + 9 * 64 * 4;     // full[c][slot] (64 arrivals: the load threads), empty[c][slot] (128)
constexpr uint32_t BYTES = BAR + 2 * 2 * RING * 8 + 1024;  // + alignment slack
static_assert(BYTES <= 227 * 1024, "decoder shared memory exceeds the sm_90 limit");
}  // namespace dec

struct DecParams {
  int B, d, mean, D;          // d: uniform in-degree (the kernel's template argument)
  long long n_rec, n_blocks;  // receivers; 64-receiver blocks
  const float* rec;           // (B, n_rec, 64), batch stride rec_bs
  long long rec_bs;
  const float* ps;            // P_s (B | 1, n_send, 64), batch stride ps_bs
  long long ps_bs;
  const float* pe;            // P_e (E, 64), CSR edge order
  const int32_t* src;         // sender of CSR edge k
  FzW w1r, w2e, wn1, wn2, wo1, wo2;
  const float *b2e, *gamma_e, *beta_e, *bn1, *bn2, *gamma_n, *beta_n, *bo1, *bo2;
  float eps_e, eps_n;
  float* out;                 // (B, n_rec, D) new state (D / 2 wide in the STD form)
  const float *prev, *bnd, *mask, *dstd, *dmean;
  float* std_out;             // STD form: (B, n_rec, D / 2) predicted std
};

// warp group MMA that adds to the accumulators: acc += A[rows] · Wᵀ over kc chunks
__device__ __forceinline__ void dec_gemm_add(float* acc, uint32_t a, uint32_t w, int kc) {
  wgmma_fence(acc, 32);
  for (int c = 0; c < kc; ++c) {
    const uint64_t da = gmma_desc(a + c * fz::CH_A), db = gmma_desc(w + c * fz::CH_W);
#pragma unroll
    for (int k = 0; k < 4; ++k) Wgmma<64>::mma(acc, da + 2 * k, db + 2 * k, 1u);
  }
  wgmma_commit();
  wgmma_wait0(acc, 32);
}

// DEG: uniform in-degree 1, 2, 4 or 8; STD: the step epilogue's predicted-std form (fz_store_rows), D = 2d outputs
template <int DEG, bool STD>
__global__ void __launch_bounds__(dec::THREADS, 1) tc_decode_kernel(const __grid_constant__ DecParams p) {
  using namespace fz;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* s = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t sb = smem_u32(s);
  float* prm = reinterpret_cast<float*>(s + dec::PRM);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2;
  auto full = [&](int c, uint32_t slot) { return sb + dec::BAR + 8u * (uint32_t)(c * dec::RING + slot); };
  auto empty = [&](int c, uint32_t slot) { return sb + dec::BAR + 8u * (uint32_t)((2 + c) * dec::RING + slot); };

  if (tid < THREADS) {
    fz_load_w(s + dec::W1R, p.w1r, 2, tid);
    fz_load_w(s + dec::W2E, p.w2e, 2, tid);
    fz_load_w(s + dec::WN1, p.wn1, 4, tid);
    fz_load_w(s + dec::WN2, p.wn2, 2, tid);
    fz_load_w(s + dec::WO1, p.wo1, 2, tid);
    fz_load_w(s + dec::WO2, p.wo2, 2, tid);
  }
  for (int i = tid; i < 64; i += dec::THREADS) {
    prm[i] = p.b2e[i];
    prm[64 + i] = p.gamma_e[i];
    prm[128 + i] = p.beta_e[i];
    prm[192 + i] = p.bn1[i];
    prm[256 + i] = p.bn2[i];
    prm[320 + i] = p.gamma_n[i];
    prm[384 + i] = p.beta_n[i];
    prm[448 + i] = p.bo1[i];
    prm[512 + i] = i < p.D ? p.bo2[i] : 0.f;
  }
  if (tid == 0)
    for (int c = 0; c < 2; ++c)
      for (uint32_t k = 0; k < dec::RING; ++k) {
        mbar_init(full(c, k), 64);
        mbar_init(empty(c, k), 128);
      }
  fence_proxy_async();
  __syncthreads();  // the last CTA-wide barrier: from here on the load halves and compute warp groups run in pairs

  const long long n_items = p.n_blocks * p.B;
  const long long stride = 2LL * gridDim.x;
  if (wg == 0) {
    // ---- load warps: threads 64c .. 64c + 63 feed compute warp group c.  Thread pt moves float4 column q4 of the unit's
    // rows pt / 16 + 4k, k < 16.
    const int c = tid >> 6, pt = tid & 63, q4 = (pt & 15) * 4, row = pt >> 4;
    uint32_t u = 0;  // units sent
    float4 x[16], y[16];
    int sidx[16];    // sender of each edge row of the thread in the coming sub-tile (-1: past the last receiver)
    auto put = [&]() {
      const uint32_t slot = u % dec::RING;
      mbar_wait_nocall(empty(c, slot), ((u / dec::RING) & 1) ^ 1);
      uint8_t* dst = s + dec::RINGS + slot * dec::SLOT;
#pragma unroll
      for (int k = 0; k < 16; ++k) *reinterpret_cast<float4*>(dst + fz_off(CH_A, 64 * c + row + 4 * k, q4)) = x[k];
      mbar_arrive(full(c, slot));
      ++u;
    };
    for (long long item = 2LL * blockIdx.x + c; item < n_items; item += stride) {
      const int b = (int)(item % p.B);
      const long long r0 = (item / p.B) * 64;
      const float* rec = p.rec + (long long)b * p.rec_bs;
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const long long r = r0 + row + 4 * k;
        x[k] = r < p.n_rec ? __ldg(reinterpret_cast<const float4*>(rec + r * 64 + q4)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      auto load_src = [&](int st) {
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          const int e = st * 64 + row + 4 * k;  // edge within the item; its receiver is e / DEG
          sidx[k] = r0 + e / DEG < p.n_rec ? __ldg(p.src + r0 * DEG + e) : -1;
        }
      };
      load_src(0);
      {  // the epilogue's previous / boundary state rows of the item -> L2
        const int Ds = STD ? p.D >> 1 : p.D;  // state columns
        const long long n = min(64LL, p.n_rec - r0) * Ds;
        const float* spans[2] = {p.prev + ((long long)b * p.n_rec + r0) * Ds, p.bnd ? p.bnd + ((long long)b * p.n_rec + r0) * Ds : nullptr};
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          if (!spans[q]) continue;
          const uintptr_t a0 = (uintptr_t)spans[q] & ~(uintptr_t)127, a1 = (uintptr_t)(spans[q] + n);
          for (uintptr_t a = a0 + 128u * (uintptr_t)pt; a < a1; a += 128u * 64u) prefetch_l2(reinterpret_cast<const void*>(a));
        }
      }
      put();
#pragma unroll 1
      for (int st = 0; st < DEG; ++st) {
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          const bool ok = sidx[k] >= 0;
          const float* pk = p.pe + (r0 * DEG + st * 64 + row + 4 * k) * 64 + q4;
          const float* sk = p.ps + (long long)b * p.ps_bs + (long long)(ok ? sidx[k] : 0) * 64 + q4;
          x[k] = ok ? __ldg(reinterpret_cast<const float4*>(pk)) : make_float4(0.f, 0.f, 0.f, 0.f);
          y[k] = ok ? __ldg(reinterpret_cast<const float4*>(sk)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        if (st + 1 < DEG) load_src(st + 1);
#pragma unroll
        for (int k = 0; k < 16; ++k) x[k] = make_float4(x[k].x + y[k].x, x[k].y + y[k].y, x[k].z + y[k].z, x[k].w + y[k].w);
        put();
      }
    }
    return;
  }

  // ---- compute warps
  const int c = wg - 1, bar = 1 + c;
  const int lr = 16 * (warp & 3) + (lane >> 2);  // row of fragment half 0 within the warp group's 64 (half 1: + 8)
  const int rq = 64 * c + lr;                     // the same row in a 128-row operand
  const int cq = 2 * (lane & 3);
  uint8_t* sN = s + dec::NODE;
  const uint32_t aN = sb + dec::NODE + c * (CH_A / 2);
  const float scale = p.mean ? 1.f / (float)DEG : 1.f;
  float acc[32], acc1[32];  // acc1: node GEMM 1, from the receiver rows until the aggregate is added
  float v[2][16], res[2][16];
  uint32_t u = 0;  // units received
  for (long long item = 2LL * blockIdx.x + c; item < n_items; item += stride) {
    const int b = (int)(item % p.B);
    const long long r0 = (item / p.B) * 64;
    // ---- 1. receiver rows: the residual in fp32, the operand rounded in place; P_r and node GEMM 1 on chunks 0-1
    uint32_t slot = u % dec::RING;
    uint8_t* sU = s + dec::RINGS + slot * dec::SLOT;
    uint32_t aU = sb + dec::RINGS + slot * dec::SLOT + c * (CH_A / 2);
    mbar_wait_nocall(full(c, slot), (u / dec::RING) & 1);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float2* px = reinterpret_cast<float2*>(sU + fz_off(CH_A, rq + 8 * i, 8 * j + cq));
        const float2 x = *px;
        res[i][2 * j] = x.x;
        res[i][2 * j + 1] = x.y;
        *px = make_float2(tf32r(x.x), tf32r(x.y));
      }
    fence_proxy_async();
    named_bar_sync(bar, 128);
    fz_gemm(acc, aU, sb + dec::W1R, 2);
    fz_gemm(acc1, aU, sb + dec::WN1, 2);
    mbar_arrive(empty(c, slot));
    ++u;
    // P_r, kept in fp32 (an addend of the edge pre-activation, not an MMA operand).  The previous item's last MMA read of
    // the node operand ended before the barrier above.
    fz_unpack(acc, v, nullptr);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<float2*>(sN + fz_off(CH_A, rq + 8 * i, 8 * j + cq)) = make_float2(v[i][2 * j], v[i][2 * j + 1]);
    named_bar_sync(bar, 128);  // every P_r row of the item is visible to the whole warp group
    // ---- 2. edges: DEG sub-tiles of 64 edges = 64 / DEG receivers each
#pragma unroll 1
    for (int st = 0; st < DEG; ++st) {
      const int rl0 = (st * 64 + lr) / DEG, rl1 = (st * 64 + lr + 8) / DEG;  // receivers of the two fragment rows
      slot = u % dec::RING;
      sU = s + dec::RINGS + slot * dec::SLOT;
      aU = sb + dec::RINGS + slot * dec::SLOT + c * (CH_A / 2);
      mbar_wait_nocall(full(c, slot), (u / dec::RING) & 1);
      // SiLU(P_e + P_s + P_r) over the sums it is computed from: each thread rewrites exactly the elements it reads
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float2* pq = reinterpret_cast<float2*>(sU + fz_off(CH_A, rq + 8 * i, 8 * j + cq));
          const float2 q = *pq;
          const float2 pr = *reinterpret_cast<const float2*>(sN + fz_off(CH_A, 64 * c + (i ? rl1 : rl0), 8 * j + cq));
          *pq = make_float2(tf32r(silu_fast(q.x + pr.x)), tf32r(silu_fast(q.y + pr.y)));
        }
      fence_proxy_async();
      named_bar_sync(bar, 128);  // the edge operand is complete, and every P_r read of this sub-tile is done
      fz_gemm(acc, aU, sb + dec::W2E, 2);
      mbar_arrive(empty(c, slot));
      ++u;
      fz_unpack(acc, v, prm);
      fz_layernorm(v, prm + 64, prm + 128, p.eps_e);
      // per-receiver sum: the DEG edges of a receiver are consecutive fragment rows, held by lanes 4, 8 and 16 apart
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int t = 0; t < 16; ++t) {
          float y = v[i][t];
          if constexpr (DEG >= 2) y += __shfl_xor_sync(0xffffffffu, y, 4);
          if constexpr (DEG >= 4) y += __shfl_xor_sync(0xffffffffu, y, 8);
          if constexpr (DEG >= 8) y += __shfl_xor_sync(0xffffffffu, y, 16);
          v[i][t] = y * scale;
        }
      // aggr (TF32, an operand of the node MLP) over the P_r rows of this sub-tile's receivers, which are read only here
      if (((lane >> 2) & (DEG - 1)) == 0) {
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<float2*>(sN + fz_off(CH_A, 64 * c + (i ? rl1 : rl0), 8 * j + cq)) =
                make_float2(tf32r(v[i][2 * j]), tf32r(v[i][2 * j + 1]));
      }
    }
    fence_proxy_async();
    named_bar_sync(bar, 128);
    // ---- 3. node MLP on [rec | aggr] (chunks 2-3 of Wn1 on aggr) + residual, output_map, step epilogue (as in
    // tc_node_out_kernel)
    dec_gemm_add(acc1, aN, sb + dec::WN1 + 2 * CH_W, 2);
    fz_unpack(acc1, v, prm + 192);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t = 0; t < 16; ++t) v[i][t] = silu_fast(v[i][t]);
    fz_store_op(sN, v, rq, c);
    fz_gemm(acc, aN, sb + dec::WN2, 2);
    fz_unpack(acc, v, prm + 256);
    fz_layernorm(v, prm + 320, prm + 384, p.eps_n);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t = 0; t < 16; ++t) v[i][t] += res[i][t];
    fz_store_op(sN, v, rq, c);
    fz_gemm(acc, aN, sb + dec::WO1, 2);
    fz_unpack(acc, v, prm + 448);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t = 0; t < 16; ++t) v[i][t] = silu_fast(v[i][t]);
    fz_store_op(sN, v, rq, c);
    fz_gemm(acc, aN, sb + dec::WO2, 2);
    fz_unpack(acc, v, prm + 512);
    const long long ra = r0 + lr;
    fz_store_rows<STD>(p, p.out, p.D, p.n_rec, true, v, b, ra, ra < p.n_rec, ra + 8 < p.n_rec);
  }
}

// ------------------------------------------------------------------------------------ grid encoder
// The grid side of a forecast step's encoder in one kernel.  Per grid row of batch element b, x = [src_0 | src_1 | ...]
// zero-padded to 64 columns:
//   grid_emb = LN(SiLU(x·We1ᵀ + be1)·We2ᵀ + be2)               (fp32, on chip)
//   P_s      = grid_emb·W1sᵀ                                    the g2m edge MLP's sender projection
//   grid_rep = grid_emb + LN(SiLU(grid_emb·Wa1ᵀ + ba1)·Wa2ᵀ + ba2)
// and, by extra work items after the grid ones, P_r = mesh·W1rᵀ + b1 once for the batch.  A work item is 64 rows of one
// batch element and belongs to one warp group, which synchronises on its own named barriers.  The item's input rows are
// copied with cp.async into a raw fp32 staging buffer while the previous item's GEMMs run; a dense source's rows of one
// item are one contiguous span, copied in 16-byte pieces where it starts 16-byte aligned and element by element otherwise.
// EMIT_EMB: grid_emb is also stored (B, n_rows, 64): Graph-EFM's decoder reads it as the senders of its g2m layer.
// TWO_G2M (tc_encode2_kernel): the projections of a second g2m edge MLP on the same grid_emb are computed as well,
// P_s_b = grid_emb·W1s_bᵀ after P_s, and P_r_b = mesh·W1r_bᵀ + b1_b by a second set of mesh items: the hierarchical Graph-EFM's
// prior and decoder g2m layers share their senders (grid_emb), receivers and edge features, so grid_emb never goes to HBM.
// The weights go through fz_load_w and grid_emb through fz_store_op as for the first layer: both round to nearest.
namespace enc {
using fz::CH_A;
using fz::CH_W;
constexpr uint32_t WE1 = 0, WE2 = WE1 + 2 * CH_W, W1S = WE2 + 2 * CH_W, WA1 = W1S + 2 * CH_W, WA2 = WA1 + 2 * CH_W,
                   W1R = WA2 + 2 * CH_W, W1S_B = W1R + 2 * CH_W, W1R_B = W1S_B + 2 * CH_W;  // W1S_B / W1R_B: TWO_G2M only
template <bool TWO_G2M>
struct Layout {
  static constexpr uint32_t A = (TWO_G2M ? W1R_B : W1R) + 2 * CH_W;  // 128 x 64 operand, 64 rows per warp group
  static constexpr uint32_t STG = A + 2 * CH_A;  // per warp group: 64 rows x at most 64 columns of raw inputs, source by source
  static constexpr uint32_t COLS = STG + 2 * 64 * 64 * 4;  // operand column c <- staging float cols[c].x + row * cols[c].y (y = 0: zero)
  // be1, be2, gamma, beta (embedder) | ba1, ba2, gamma, beta (grid MLP) | b1 (g2m) | b1_b (second g2m, TWO_G2M only)
  static constexpr uint32_t PRM = COLS + 64 * 8;
  static constexpr uint32_t BYTES = PRM + (TWO_G2M ? 10 : 9) * 64 * 4 + 1024;  // + alignment slack
  static_assert(BYTES <= 227 * 1024, "encoder shared memory exceeds the sm_90 limit");
};
}  // namespace enc

struct EncParams {
  int B, n_src;
  FzSrc src[4];                 // dense rows (idx NULL, row pitch = dim), batch stride bs (0: shared by the batch)
  long long n_rows, n_tiles;    // grid rows; 64-row tiles per batch element
  FzW we1, we2, w1s, wa1, wa2, w1r;
  const float *be1, *be2, *gamma_e, *beta_e, *ba1, *ba2, *gamma_a, *beta_a, *b1;
  float eps_e, eps_a;
  float* grid_rep;              // (B, n_rows, 64)
  float* ps;                    // (B, n_rows, 64)
  float* grid_emb;              // (B, n_rows, 64), EMIT_EMB only
  const float* mesh;            // (n_mesh, 64), shared by the batch
  float* pr;                    // (n_mesh, 64)
  long long n_mesh, n_mesh_tiles;
  FzW w1s_b, w1r_b;             // TWO_G2M only: the second g2m edge MLP
  const float* b1_b;
  float *ps_b, *pr_b;           // (B, n_rows, 64), (n_mesh, 64)
};

template <bool EMIT_EMB, bool TWO_G2M>
__global__ void __launch_bounds__(fz::THREADS, 1) tc_encode_kernel(const __grid_constant__ EncParams p) {
  using namespace fz;
  using Lay = enc::Layout<TWO_G2M>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* s = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t sb = smem_u32(s);
  uint8_t* sA = s + Lay::A;
  float* prm = reinterpret_cast<float*>(s + Lay::PRM);
  int2* cols = reinterpret_cast<int2*>(s + Lay::COLS);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2, gt = tid & 127, bar = 1 + wg;
  const int rq = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // operand row of fragment half 0 (half 1: + 8)
  const int lr = rq - 64 * wg;                              // the same row within the warp group's 64
  const uint32_t aA = sb + Lay::A + wg * (CH_A / 2);
  float* stg = reinterpret_cast<float*>(s + Lay::STG) + wg * 64 * 64;
  const uint32_t stg_u = smem_u32(stg);

  fz_load_w(s + enc::WE1, p.we1, 2, tid);
  fz_load_w(s + enc::WE2, p.we2, 2, tid);
  fz_load_w(s + enc::W1S, p.w1s, 2, tid);
  fz_load_w(s + enc::WA1, p.wa1, 2, tid);
  fz_load_w(s + enc::WA2, p.wa2, 2, tid);
  fz_load_w(s + enc::W1R, p.w1r, 2, tid);
  if (TWO_G2M) {
    fz_load_w(s + enc::W1S_B, p.w1s_b, 2, tid);
    fz_load_w(s + enc::W1R_B, p.w1r_b, 2, tid);
  }
  for (int i = tid; i < 64; i += THREADS) {
    prm[i] = p.be1[i];
    prm[64 + i] = p.be2[i];
    prm[128 + i] = p.gamma_e[i];
    prm[192 + i] = p.beta_e[i];
    prm[256 + i] = p.ba1[i];
    prm[320 + i] = p.ba2[i];
    prm[384 + i] = p.gamma_a[i];
    prm[448 + i] = p.beta_a[i];
    prm[512 + i] = p.b1[i];
    if (TWO_G2M) prm[576 + i] = p.b1_b[i];
    int2 m = make_int2(0, 0);
    for (int q = 0, off = 0; q < p.n_src; off += p.src[q].dim, ++q)
      if (i >= off && i < off + p.src[q].dim) m = make_int2(64 * off + i - off, p.src[q].dim);
    cols[i] = m;
  }
  fence_proxy_async();
  __syncthreads();  // the last CTA-wide barrier: from here on each warp group runs on its own

  const long long n_grid = p.n_tiles * p.B, n_items = n_grid + (TWO_G2M ? 2 : 1) * p.n_mesh_tiles;
  const long long stride = 2LL * gridDim.x;
  const uint64_t pol_stream = policy_evict_first(), pol_shared = policy_evict_normal();
  // the raw input rows of grid item it -> staging (source q at float 64 * (dim_0 + ... + dim_{q-1}), rows dense)
  auto issue = [&](long long it) {
    const int bi = (int)(it / p.n_tiles);
    const long long row0 = (it - (long long)bi * p.n_tiles) * 64;
    const int n = (int)min(64LL, p.n_rows - row0);
    int off = 0;
    for (int q = 0; q < p.n_src; ++q) {
      const FzSrc& sq = p.src[q];
      const float* g = sq.ptr + bi * sq.bs + row0 * sq.dim;
      const uint32_t dst = stg_u + 4u * 64u * (uint32_t)off;
      const int ne = n * sq.dim, n16 = ((uintptr_t)g & 15) == 0 ? ne >> 2 : 0;
      const uint64_t pol = sq.bs ? pol_stream : pol_shared;
      for (int k = gt; k < n16; k += 128) cp_async_16(dst + 16u * k, g + 4 * k, pol);
      for (int k = 4 * n16 + gt; k < ne; k += 128) cp_async_4(dst + 4u * k, g + k);
      off += sq.dim;
    }
  };
  float acc[32];
  float v[2][16], e[2][16];
  long long item = 2LL * blockIdx.x + wg;
  if (item < n_grid) issue(item);
  for (; item < n_items; item += stride) {
    if (item >= n_grid) {
      // ---- P_r = mesh·W1rᵀ + b1 for 64 mesh rows (few items: loaded without staging); TWO_G2M: the items after the first
      // n_mesh_tiles compute P_r_b
      const bool second = TWO_G2M && item - n_grid >= p.n_mesh_tiles;
      const long long row0 = (item - n_grid - (second ? p.n_mesh_tiles : 0)) * 64;
      float4 x[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const long long r = row0 + 8 * q + (gt >> 4);
        x[q] = r < p.n_mesh ? __ldg(reinterpret_cast<const float4*>(p.mesh + r * 64 + (gt & 15) * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      named_bar_sync(bar, 128);  // the previous item's MMAs have finished reading the operand
#pragma unroll
      for (int q = 0; q < 8; ++q)
        *reinterpret_cast<float4*>(sA + fz_off(CH_A, 64 * wg + 8 * q + (gt >> 4), (gt & 15) * 4)) = tf32r4(x[q]);
      fence_proxy_async();
      named_bar_sync(bar, 128);
      fz_gemm(acc, aA, sb + (second ? enc::W1R_B : enc::W1R), 2);
      fz_unpack(acc, v, prm + (second ? 576 : 512));
      const long long r0 = row0 + lr;
      float* pr = second ? p.pr_b : p.pr;
#pragma unroll
      for (int i = 0; i < 2; ++i)
        if (r0 + 8 * i < p.n_mesh) fz_store_row64(pr + (r0 + 8 * i) * 64, v[i]);
      continue;
    }
    const int b = (int)(item / p.n_tiles);
    const long long row0 = (item - (long long)b * p.n_tiles) * 64;
    const int nrows = (int)min(64LL, p.n_rows - row0);
    // ---- 1. staged inputs -> operand (TF32, zero-padded columns and rows)
    cp_async_wait_all();
    named_bar_sync(bar, 128);  // every thread's copies have landed; the previous item's MMAs are done with the operand
    for (int g = gt; g < 64 * 16; g += 128) {
      const int i = g >> 4, c = (g & 15) * 4;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      float* px = &x.x;
      if (i < nrows) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int2 m = cols[c + k];
          if (m.y) px[k] = stg[m.x + i * m.y];
        }
      }
      *reinterpret_cast<float4*>(sA + fz_off(CH_A, 64 * wg + i, c)) = tf32r4(x);
    }
    fence_proxy_async();
    named_bar_sync(bar, 128);  // the operand is complete and the staging buffer free
    if (item + stride < n_grid) issue(item + stride);
    // ---- 2. grid embedder
    fz_gemm(acc, aA, sb + enc::WE1, 2);
    fz_unpack(acc, v, prm);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t = 0; t < 16; ++t) v[i][t] = silu_fast(v[i][t]);
    fz_store_op(sA, v, rq, wg);
    fz_gemm(acc, aA, sb + enc::WE2, 2);
    fz_unpack(acc, v, prm + 64);
    fz_layernorm(v, prm + 128, prm + 192, p.eps_e);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t = 0; t < 16; ++t) e[i][t] = v[i][t];
    fz_store_op(sA, v, rq, wg);  // grid_emb: the operand of the next three GEMMs
    const long long r0 = row0 + lr;
    const bool valid0 = lr < nrows, valid1 = lr + 8 < nrows;
    const long long o = ((long long)b * p.n_rows + r0) * 64;
    if (EMIT_EMB) {
      if (valid0) fz_store_row64(p.grid_emb + o, e[0]);
      if (valid1) fz_store_row64(p.grid_emb + o + 8 * 64, e[1]);
    }
    // ---- 3. P_s = grid_emb·W1sᵀ
    fz_gemm(acc, aA, sb + enc::W1S, 2);
    fz_unpack(acc, v, nullptr);
    if (valid0) fz_store_row64(p.ps + o, v[0]);
    if (valid1) fz_store_row64(p.ps + o + 8 * 64, v[1]);
    if (TWO_G2M) {  // ---- 3b. P_s_b = grid_emb·W1s_bᵀ, on the same operand
      fz_gemm(acc, aA, sb + enc::W1S_B, 2);
      fz_unpack(acc, v, nullptr);
      if (valid0) fz_store_row64(p.ps_b + o, v[0]);
      if (valid1) fz_store_row64(p.ps_b + o + 8 * 64, v[1]);
    }
    // ---- 4. grid_rep = grid_emb + encoding grid MLP(grid_emb)
    fz_gemm(acc, aA, sb + enc::WA1, 2);
    fz_unpack(acc, v, prm + 256);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t = 0; t < 16; ++t) v[i][t] = silu_fast(v[i][t]);
    fz_store_op(sA, v, rq, wg);
    fz_gemm(acc, aA, sb + enc::WA2, 2);
    fz_unpack(acc, v, prm + 320);
    fz_layernorm(v, prm + 384, prm + 448, p.eps_a);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t = 0; t < 16; ++t) v[i][t] += e[i][t];
    if (valid0) fz_store_row64(p.grid_rep + o, v[0]);
    if (valid1) fz_store_row64(p.grid_rep + o + 8 * 64, v[1]);
  }
}

// ------------------------------------------------------------------------------------ Graph-EFM latent sample
// The stochastic part of a Graph-EFM step in one kernel.  Per mesh row of batch element b, with x the prior's mesh
// representation and eps standard normal noise:
//   p          = SiLU(x·W1ᵀ + b1)·W2ᵀ + b2                the prior's latent_param_map (no LayerNorm)
//   mean, std  = p[:, :64], 1 (isotropic) | 1e-4 + softplus(p[:, 64:]) (diagonal; torch's threshold 20)
//   z          = mean + eps·std                           rounded as torch's two ops: the product, then the sum
//   latent_emb = LN(SiLU(z·W3ᵀ + b3)·W4ᵀ + b4)            the decoder's latent_embedder
// p and z never leave the SM; z is rounded to TF32 (to nearest) as the operand of W3.  Work items, warp-group ownership and
// the staging of the next item's rows while this item's GEMMs run are those of tc_encode_kernel; x and eps rows are copied
// in 16-byte pieces into staging rows padded to 68 floats.
namespace lat {
using fz::CH_A;
using fz::CH_W;
constexpr int PITCH = 68;
constexpr uint32_t W1 = 0, W2M = W1 + 2 * CH_W, W2S = W2M + 2 * CH_W, W3 = W2S + 2 * CH_W, W4 = W3 + 2 * CH_W;
constexpr uint32_t A = W4 + 2 * CH_W;     // 128 x 64 operand, 64 rows per warp group
constexpr uint32_t STG = A + 2 * CH_A;    // per warp group: 64 x rows | 64 eps rows, PITCH floats each
constexpr uint32_t PRM = STG + 2 * 2 * 64 * PITCH * 4;  // b1 | b2 (mean) | b2 (std) | b3 | b4 | gamma | beta
constexpr uint32_t BYTES = PRM + 7 * 64 * 4 + 1024;     // + alignment slack
static_assert(BYTES <= 227 * 1024, "latent kernel shared memory exceeds the sm_90 limit");
}  // namespace lat

struct LatParams {
  int B, diag;
  long long n_rows, n_tiles;   // mesh rows; 64-row tiles per batch element
  const float* x;              // (B, n_rows, 64), batch stride x_bs
  const float* eps;            // (B, n_rows, 64), batch stride eps_bs
  long long x_bs, eps_bs;
  FzW w1, w2m, w2s, w3, w4;
  const float *b1, *b2m, *b2s, *b3, *b4, *gamma, *beta;
  float ln_eps;
  float* out;                  // (B, n_rows, 64) dense
};

__global__ void __launch_bounds__(fz::THREADS, 1) tc_latent_kernel(const __grid_constant__ LatParams p) {
  using namespace fz;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* s = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t sb = smem_u32(s);
  uint8_t* sA = s + lat::A;
  float* prm = reinterpret_cast<float*>(s + lat::PRM);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2, gt = tid & 127, bar = 1 + wg;
  const int rq = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // operand row of fragment half 0 (half 1: + 8)
  const int lr = rq - 64 * wg;                              // the same row within the warp group's 64
  const int cq = 2 * (lane & 3);
  const uint32_t aA = sb + lat::A + wg * (CH_A / 2);
  float* sx = reinterpret_cast<float*>(s + lat::STG) + wg * 2 * 64 * lat::PITCH;
  float* se = sx + 64 * lat::PITCH;
  const uint32_t sx_u = smem_u32(sx), se_u = smem_u32(se);

  fz_load_w(s + lat::W1, p.w1, 2, tid);
  fz_load_w(s + lat::W2M, p.w2m, 2, tid);
  if (p.diag) fz_load_w(s + lat::W2S, p.w2s, 2, tid);
  fz_load_w(s + lat::W3, p.w3, 2, tid);
  fz_load_w(s + lat::W4, p.w4, 2, tid);
  for (int i = tid; i < 64; i += THREADS) {
    prm[i] = p.b1[i];
    prm[64 + i] = p.b2m[i];
    prm[128 + i] = p.diag ? p.b2s[i] : 0.f;
    prm[192 + i] = p.b3[i];
    prm[256 + i] = p.b4[i];
    prm[320 + i] = p.gamma[i];
    prm[384 + i] = p.beta[i];
  }
  fence_proxy_async();
  __syncthreads();  // the last CTA-wide barrier: from here on each warp group runs on its own

  const long long n_items = p.n_tiles * p.B, stride = 2LL * gridDim.x;
  const uint64_t pol = policy_evict_first();
  // the x and eps rows of item it -> staging (rows of 64 floats, 16-byte aligned: one span per tensor)
  auto issue = [&](long long it) {
    const int bi = (int)(it / p.n_tiles);
    const long long row0 = (it - (long long)bi * p.n_tiles) * 64;
    const int n = (int)min(64LL, p.n_rows - row0);
    const float* gx = p.x + bi * p.x_bs + row0 * 64;
    const float* ge = p.eps + bi * p.eps_bs + row0 * 64;
    for (int k = gt; k < n * 16; k += 128) {
      const uint32_t o = 4u * (uint32_t)((k >> 4) * lat::PITCH + (k & 15) * 4);
      cp_async_16(sx_u + o, gx + 4 * k, pol);
      cp_async_16(se_u + o, ge + 4 * k, pol);
    }
  };
  float acc[32];
  float v[2][16], z[2][16];
  long long item = 2LL * blockIdx.x + wg;
  if (item < n_items) issue(item);
  for (; item < n_items; item += stride) {
    const int b = (int)(item / p.n_tiles);
    const long long row0 = (item - (long long)b * p.n_tiles) * 64;
    const int nrows = (int)min(64LL, p.n_rows - row0);
    const bool valid0 = lr < nrows, valid1 = lr + 8 < nrows;
    // ---- 1. staged x -> operand (TF32, zero rows past the end); this thread's eps in the accumulator fragment layout
    cp_async_wait_all();
    named_bar_sync(bar, 128);  // every thread's copies have landed; the previous item's MMAs are done with the operand
    for (int g = gt; g < 64 * 16; g += 128) {
      const int i = g >> 4, c = (g & 15) * 4;
      const float4 x = i < nrows ? *reinterpret_cast<const float4*>(sx + i * lat::PITCH + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(sA + fz_off(CH_A, 64 * wg + i, c)) = tf32r4(x);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 e = (i ? valid1 : valid0) ? *reinterpret_cast<const float2*>(se + (lr + 8 * i) * lat::PITCH + 8 * j + cq)
                                               : make_float2(0.f, 0.f);
        z[i][2 * j] = e.x;
        z[i][2 * j + 1] = e.y;
      }
    fence_proxy_async();
    named_bar_sync(bar, 128);  // the operand is complete and the staging buffers free
    if (item + stride < n_items) issue(item + stride);
    // ---- 2. prior latent_param_map: hidden layer
    fz_gemm(acc, aA, sb + lat::W1, 2);
    fz_unpack(acc, v, prm);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t = 0; t < 16; ++t) v[i][t] = silu_fast(v[i][t]);
    fz_store_op(sA, v, rq, wg);
    // ---- 3. eps·std (diagonal: std = 1e-4 + softplus(raw); isotropic: std = 1, eps·1 = eps)
    if (p.diag) {
      fz_gemm(acc, aA, sb + lat::W2S, 2);
      fz_unpack(acc, v, prm + 128);
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int t = 0; t < 16; ++t) {
          const float r = v[i][t];
          const float sp = r > 20.f ? r : log1pf(expf(r));
          z[i][t] = __fmul_rn(z[i][t], __fadd_rn(1e-4f, sp));
        }
    }
    // ---- 4. z = mean + eps·std
    fz_gemm(acc, aA, sb + lat::W2M, 2);
    fz_unpack(acc, v, prm + 64);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t = 0; t < 16; ++t) v[i][t] = __fadd_rn(v[i][t], z[i][t]);
    fz_store_op(sA, v, rq, wg);
    // ---- 5. decoder latent_embedder
    fz_gemm(acc, aA, sb + lat::W3, 2);
    fz_unpack(acc, v, prm + 192);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t = 0; t < 16; ++t) v[i][t] = silu_fast(v[i][t]);
    fz_store_op(sA, v, rq, wg);
    fz_gemm(acc, aA, sb + lat::W4, 2);
    fz_unpack(acc, v, prm + 256);
    fz_layernorm(v, prm + 320, prm + 384, p.ln_eps);
    const long long o = ((long long)b * p.n_rows + row0 + lr) * 64;
    if (valid0) fz_store_row64(p.out + o, v[0]);
    if (valid1) fz_store_row64(p.out + o + 8 * 64, v[1]);
  }
}

// ------------------------------------------------------------------------------------ H = 64 node update
// The node update of an InteractionNet layer, out = res + LN(SiLU([src_0 | src_1]·Wn1ᵀ + bn1)·Wn2ᵀ + bn2) with res one of the
// two 64-wide sources (rec for InteractionNet, aggr for PropagationNet), followed by one of three epilogues:
//   POST_NONE    out                                                  (tc_rowmlp_kernel)
//   POST_PROJ    out, P_s = out·W3ᵀ, P_r = out·W4ᵀ + b4               (tc_node_proj_kernel)
//   POST_OUTMLP  step epilogue of SiLU(out·W3ᵀ + b3)·W4ᵀ + b4, out on chip   (tc_node_out_kernel)
// Every GEMM is m64n64k8 MMAs over 64-row tiles on operands rounded to TF32 (to nearest) as they enter shared memory, with
// the epilogue code of the row kernels above, so POST_PROJ's projections equal tc_rowlinear_kernel's on the same rows, and
// POST_OUTMLP's output equals POST_NONE followed by fused_mlp_kernel's row MLP with the step epilogue, bit for bit.  Work
// items, warp-group ownership and staging are those of tc_latent_kernel:
// an item is 64 rows of one batch element and belongs to one warp group; the item's two source spans (64 x 256 B each,
// contiguous and 16-byte aligned) are copied with cp.async into the warp group's raw staging rows while the previous item's
// GEMMs run.  cp.async does not round, so staging -> operand applies tf32r4 as fz_load_a does; the residual is read from
// staging in fp32 into the accumulator fragment layout before the next item's copies overwrite it.
namespace nod {
using fz::CH_A;
using fz::CH_W;
constexpr int PITCH = 72;  // staged rows: 64 floats + 8 (fragment-layout float2 reads of a half warp hit distinct banks)
constexpr uint32_t WN1 = 0, WN2 = WN1 + 4 * CH_W, W3 = WN2 + 2 * CH_W, W4 = W3 + 2 * CH_W;
constexpr uint32_t A = W4 + 2 * CH_W;                  // 128 x 128 operand [src_0 | src_1], 64 rows per warp group
constexpr uint32_t STG = A + 4 * CH_A;                 // per warp group: 64 src_0 rows | 64 src_1 rows, PITCH floats each
constexpr uint32_t STG_WG = 2 * 64 * PITCH * 4;
constexpr uint32_t PRM = STG + 2 * STG_WG;             // bn1 | bn2 | gamma | beta | b3 | b4
constexpr uint32_t BYTES = PRM + 6 * 64 * 4 + 1024;    // + alignment slack
static_assert(BYTES <= 227 * 1024, "node kernel shared memory exceeds the sm_90 limit");
enum Post { POST_NONE = 0, POST_PROJ = 1, POST_OUTMLP = 2 };
}  // namespace nod

struct NodeParams {
  int B, post, res_src;       // post: nod::Post; res_src: the source that is also the residual
  long long n_rows, n_tiles;  // rows; 64-row tiles per batch element
  const float* src[2];        // (B | 1, n_rows, 64), batch stride bs (0: shared by the batch)
  long long bs[2];
  FzW wn1, wn2, w3, w4;
  const float *bn1, *bn2, *gamma, *beta, *b3, *b4;
  float eps;
  float* out;                 // (B, n_rows, out_w)
  int out_w;
  float *out3, *out4;         // POST_PROJ: (B, n_rows, 64) each
  const float *prev, *bnd, *mask, *dstd, *dmean;  // POST_OUTMLP: the forecast-step epilogue
  float* std_out;             // POST_OUTMLP, STD form: (B, n_rows, out_w / 2) predicted std
};

template <bool STD>  // STD: POST_OUTMLP's step epilogue in its predicted-std form (fz_store_rows)
__global__ void __launch_bounds__(fz::THREADS, 1) tc_node_kernel(const __grid_constant__ NodeParams p) {
  using namespace fz;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* s = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const uint32_t sb = smem_u32(s);
  uint8_t* sA = s + nod::A;
  float* prm = reinterpret_cast<float*>(s + nod::PRM);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warp >> 2, gt = tid & 127, bar = 1 + wg;
  const int rq = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // operand row of fragment half 0 (half 1: + 8)
  const int lr = rq - 64 * wg;                              // the same row within the warp group's 64
  const int cq = 2 * (lane & 3);
  const uint32_t aA = sb + nod::A + wg * (CH_A / 2);
  const float* stg = reinterpret_cast<const float*>(s + nod::STG + wg * nod::STG_WG);
  const float* sres = stg + p.res_src * 64 * nod::PITCH;
  const uint32_t stg_u = smem_u32(stg);

  fz_load_w(s + nod::WN1, p.wn1, 4, tid);
  fz_load_w(s + nod::WN2, p.wn2, 2, tid);
  if (p.post != nod::POST_NONE) {
    fz_load_w(s + nod::W3, p.w3, 2, tid);
    fz_load_w(s + nod::W4, p.w4, 2, tid);
  }
  for (int i = tid; i < 64; i += THREADS) {  // a Linear without bias adds zeros, a LayerNorm without beta too
    prm[i] = p.bn1 ? p.bn1[i] : 0.f;
    prm[64 + i] = p.bn2 ? p.bn2[i] : 0.f;
    prm[128 + i] = p.gamma[i];
    prm[192 + i] = p.beta ? p.beta[i] : 0.f;
    prm[256 + i] = p.b3 ? p.b3[i] : 0.f;
    prm[320 + i] = p.b4 ? p.b4[i] : 0.f;
  }
  fence_proxy_async();
  __syncthreads();  // the last CTA-wide barrier: from here on each warp group runs on its own

  const long long n_items = p.n_tiles * p.B, stride = 2LL * gridDim.x;
  const uint64_t pol_stream = policy_evict_first(), pol_shared = policy_evict_normal();
  // the rows of item it -> staging: source q's 64 rows at float 64 PITCH q, one 16-byte aligned span per source
  auto issue = [&](long long it) {
    const int bi = (int)(it / p.n_tiles);
    const long long row0 = (it - (long long)bi * p.n_tiles) * 64;
    const int n = (int)min(64LL, p.n_rows - row0);
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const float* g = p.src[q] + bi * p.bs[q] + row0 * 64;
      const uint32_t dst = stg_u + 4u * (uint32_t)(q * 64 * nod::PITCH);
      const uint64_t pol = p.bs[q] ? pol_stream : pol_shared;
      for (int k = gt; k < n * 16; k += 128) cp_async_16(dst + 4u * (uint32_t)((k >> 4) * nod::PITCH + (k & 15) * 4), g + 4 * k, pol);
    }
  };
  float acc[32];
  float v[2][16], r[2][16];
  long long item = 2LL * blockIdx.x + wg;
  if (item < n_items) issue(item);
  for (; item < n_items; item += stride) {
    const int b = (int)(item / p.n_tiles);
    const long long row0 = (item - (long long)b * p.n_tiles) * 64;
    const int nrows = (int)min(64LL, p.n_rows - row0);
    const bool valid0 = lr < nrows, valid1 = lr + 8 < nrows;
    // ---- 1. staged rows -> operand (TF32, zero rows past the end); this thread's residual in the fragment layout (fp32)
    cp_async_wait_all();
    named_bar_sync(bar, 128);  // every thread's copies have landed; the previous item's MMAs are done with the operand
    for (int g = gt; g < 64 * 32; g += 128) {
      const int i = g >> 5, c = (g & 31) * 4;
      const float4 x = i < nrows ? *reinterpret_cast<const float4*>(stg + (c >> 6) * 64 * nod::PITCH + i * nod::PITCH + (c & 63))
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(sA + fz_off(CH_A, 64 * wg + i, c)) = tf32r4(x);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 x = (i ? valid1 : valid0) ? *reinterpret_cast<const float2*>(sres + (lr + 8 * i) * nod::PITCH + 8 * j + cq)
                                               : make_float2(0.f, 0.f);
        r[i][2 * j] = x.x;
        r[i][2 * j + 1] = x.y;
      }
    fence_proxy_async();
    named_bar_sync(bar, 128);  // the operand is complete and the staging rows free
    if (item + stride < n_items) issue(item + stride);
    // ---- 2. node MLP on [src_0 | src_1], LayerNorm, residual
    fz_gemm(acc, aA, sb + nod::WN1, 4);
    fz_unpack(acc, v, prm);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t = 0; t < 16; ++t) v[i][t] = silu_fast(v[i][t]);
    fz_store_op(sA, v, rq, wg);
    fz_gemm(acc, aA, sb + nod::WN2, 2);
    fz_unpack(acc, v, prm + 64);
    fz_layernorm(v, prm + 128, prm + 192, p.eps);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int t = 0; t < 16; ++t) v[i][t] += r[i][t];
    const long long r0 = row0 + lr;
    // ---- 3. epilogue
    if (p.post == nod::POST_NONE) {
      fz_store_rows(p, p.out, 64, p.n_rows, false, v, b, r0, valid0, valid1);
    } else if (p.post == nod::POST_PROJ) {
      fz_store_rows(p, p.out, 64, p.n_rows, false, v, b, r0, valid0, valid1);  // the updated node rows
      fz_store_op(sA, v, rq, wg);
      fz_gemm(acc, aA, sb + nod::W3, 2);
      fz_unpack(acc, v, nullptr);
      fz_store_rows(p, p.out3, 64, p.n_rows, false, v, b, r0, valid0, valid1);
      fz_gemm(acc, aA, sb + nod::W4, 2);
      fz_unpack(acc, v, prm + 320);
      fz_store_rows(p, p.out4, 64, p.n_rows, false, v, b, r0, valid0, valid1);
    } else {  // POST_OUTMLP: the updated node rows stay on chip
      fz_store_op(sA, v, rq, wg);
      fz_gemm(acc, aA, sb + nod::W3, 2);
      fz_unpack(acc, v, prm + 256);
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int t = 0; t < 16; ++t) v[i][t] = silu_fast(v[i][t]);
      fz_store_op(sA, v, rq, wg);
      fz_gemm(acc, aA, sb + nod::W4, 2);
      fz_unpack(acc, v, prm + 320);
      fz_store_rows<STD>(p, p.out, p.out_w, p.n_rows, true, v, b, r0, valid0, valid1);
    }
  }
}

// ------------------------------------------------------------------------------------ host
static FzW wslice(const float* w, int ld, int rows, int cols) { return FzW{w, ld, rows, cols}; }

// One launch of the persistent kernel K over `items` work items (none: nothing to launch), `threads` threads and `smem`
// bytes of dynamic shared memory per CTA.  K's dynamic shared-memory limit is raised to smem_limit once per device.  grid
// is the CTA count; 0 asks for as many CTAs as fit on every SM at `smem` bytes, at most one per item, which the occupancy
// calculator can tell only once the limit is raised.
template <auto K, class P>
static int persistent_launch(int threads, size_t smem, size_t smem_limit, long long items, int grid, const char* name,
                             double bytes, cudaStream_t st, const P& p) {
  if (items == 0) return NLAM_OK;
  NLAM_REQUIRE(items < (1LL << 40), NLAM_E_INVALID, "%s: bad work size", name);
  int dev = 0;
  NLAM_CUDA_OK(cudaGetDevice(&dev));
  static unsigned optin = 0;  // one bit per device on which K's limit is raised
  if (!(optin & (1u << (dev & 31)))) {
    NLAM_CUDA_OK(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_limit));
    optin |= 1u << (dev & 31);
  }
  if (grid == 0) {
    int per_sm = 1;
    NLAM_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, K, threads, smem));
    grid = (int)std::min<long long>(items, (long long)num_sms() * std::max(per_sm, 1));
  }
  {
    ProfScope ps(name, st, bytes);
    K<<<grid, threads, smem, st>>>(p);
  }
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

// fused_mlp_kernel: as many CTAs per SM as fit (two for the K = 64 launches); the limit covers the largest layout
template <bool STD = false>
static int fz_launch(const FzParams& p, const char* name, double bytes, cudaStream_t st) {
  const long long n_work = (long long)p.n_tiles * p.B + (p.mode == fz::ROWLIN ? (long long)p.n_tiles1 * p.B1 : 0);
  return persistent_launch<fused_mlp_kernel<STD>>(fz::THREADS, fz::layout(p.kc1, p.mode).bytes, fz::layout(6, fz::EDGE).bytes, n_work,
                                             0, name, bytes, st, p);
}

// The node update every tc_node_kernel launch starts with: [src_0 | src_1] (64 wide each, batch strides bs0 / bs1) through a
// node MLP (node_mlp_ok), plus source res_src as the residual, into out (B, n_rows, 64) unless the epilogue keeps it
static NodeParams node_params(const NlamMlp* m, const float* src0, int64_t bs0, const float* src1, int64_t bs1, int res_src,
                              int64_t n_rows, int B, float* out) {
  NodeParams p;
  memset(&p, 0, sizeof(p));
  p.B = B;
  p.res_src = res_src;
  p.n_rows = n_rows;
  p.n_tiles = (n_rows + 63) / 64;
  p.src[0] = src0;
  p.src[1] = src1;
  p.bs[0] = B > 1 ? bs0 : 0;
  p.bs[1] = B > 1 ? bs1 : 0;
  p.wn1 = wslice(m->w[0], 128, 64, 128);
  p.wn2 = wslice(m->w[1], 64, 64, 64);
  p.bn1 = m->b[0];
  p.bn2 = m->b[1];
  p.gamma = m->ln_gamma;
  p.beta = m->ln_beta;
  p.eps = m->ln_eps;
  p.out = out;
  p.out_w = 64;
  return p;
}

template <bool STD = false>
static int node_launch(const NodeParams& p, const char* name, double bytes, cudaStream_t st) {
  const long long n_items = p.n_tiles * p.B;
  const int grid = (int)std::min<long long>((n_items + 1) / 2, num_sms());  // one CTA per SM, two items at a time
  return persistent_launch<tc_node_kernel<STD>>(fz::THREADS, nod::BYTES, nod::BYTES, n_items, grid, name, bytes, st, p);
}

static void fz_mlp(FzParams& p, const NlamMlp* m, int k_off, int k_cols) {
  // first Linear: columns [k_off, k_off + k_cols) of w[0]; second Linear + LayerNorm
  p.w1 = wslice(m->w[0] + k_off, m->in_dim, 64, k_cols);
  p.kc1 = (k_cols + 31) / 32;
  p.b1 = m->b[0];
  p.act1 = 1;
  p.has_gemm2 = 1;
  p.w2 = wslice(m->w[1], 64, m->out_dim[1], 64);
  p.b2 = m->b[1];
  p.gamma = m->ln_gamma;
  p.beta = m->ln_beta;
  p.eps = m->ln_eps;
}

// node MLP: [rec | aggr] (128) -> 64 -> 64 with an affine LayerNorm
static bool node_mlp_ok(const NlamMlp* m) {
  int no = 0;
  return mlp_shape_ok(m, &no) && no == 64 && m->in_dim == 128 && m->ln_gamma && m->ln_beta;
}

// ---- row MLPs (H = 64): embedders, node updates, output_map (+ step epilogue)
bool tc_rowmlp_supported(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res, const NlamRowSrc* res2,
                         int64_t n_rows) {
  int nout = 0;
  if (res2 || n_rows < 1 || n_rows >= (1LL << 31) - 256 || n_src < 1 || n_src > 4) return false;
  if (!mlp_shape_ok(mlp, &nout)) return false;
  int k = 0;
  for (int s = 0; s < n_src; ++s) {
    // (fz_load_a reads with 16-byte loads only from sources whose width is a multiple of 4)
    if (srcs[s].idx || !aligned16(srcs[s].ptr) || (srcs[s].dim % 4 == 0 && srcs[s].bstride % 4 != 0)) return false;
    k += srcs[s].dim;
  }
  if (k != mlp->in_dim) return false;
  bool all_wide = n_src <= 2;
  for (int s = 0; s < n_src; ++s) all_wide = all_wide && srcs[s].dim == 64;
  if (all_wide) {  // node updates / encoders: the residual is one of the inputs
    if (res) {
      if (nout != 64 || res->idx) return false;
      bool match = false;
      for (int s = 0; s < n_src; ++s) match = match || (srcs[s].ptr == res->ptr && srcs[s].bstride == res->bstride);
      if (!match) return false;
    }
    return true;
  }
  // narrow concatenation (grid embedder, output_map inputs): total width <= 64, no residual
  return !res && mlp->in_dim <= 64;
}

int tc_rowmlp(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res, float* out, int64_t n_rows, int B,
              cudaStream_t st, const StepEpilogue* ep) {
  NLAM_REQUIRE(tc_rowmlp_supported(mlp, srcs, n_src, res, nullptr, n_rows), NLAM_E_UNSUPPORTED, "tc_rowmlp: unsupported shape");
  const int nout = mlp->out_dim[1];
  NLAM_REQUIRE(!ep || (nout < 64 && !mlp->ln_gamma && !res), NLAM_E_UNSUPPORTED,
               "tc_rowmlp: the fused step epilogue needs a narrow output without LayerNorm / residual");
  const bool std_form = ep && ep->std_out;
  NLAM_REQUIRE(!std_form || nout % 2 == 0, NLAM_E_UNSUPPORTED, "tc_rowmlp: the predicted-std form needs 2·d outputs");
  const int nst = std_form ? nout / 2 : nout;  // stored columns per row
  double bytes = 0;
  for (int s = 0; s < n_src; ++s) bytes += 4.0 * n_rows * srcs[s].dim * ((srcs[s].bstride != 0 && B > 1) ? B : 1);
  if (res) bytes += 4.0 * n_rows * 64 * ((res->bstride != 0 && B > 1) ? B : 1);
  bytes += 4.0 * n_rows * B * nst * (std_form ? 2 : 1);
  if (ep) bytes += 4.0 * n_rows * B * nst * (ep->boundary ? 2 : 1);
  // node update: two 64-wide sources, the residual one of them
  if (res && !ep && n_src == 2 && srcs[0].dim == 64 && srcs[1].dim == 64 && node_mlp_ok(mlp)) {
    const int res_src = (srcs[0].ptr == res->ptr && srcs[0].bstride == res->bstride) ? 0 : 1;
    return node_launch(node_params(mlp, srcs[0].ptr, srcs[0].bstride, srcs[1].ptr, srcs[1].bstride, res_src, n_rows, B, out),
                       "tc_rowmlp_kernel", bytes, st);
  }
  FzParams p;
  memset(&p, 0, sizeof(p));
  p.mode = fz::ROWS;
  p.B = B;
  p.n_src = n_src;
  for (int s = 0; s < n_src; ++s) p.src[s] = FzSrc{srcs[s].ptr, srcs[s].idx, B > 1 ? srcs[s].bstride : 0, srcs[s].dim};
  fz_mlp(p, mlp, 0, mlp->in_dim);
  if (res) {
    p.res = res->ptr;
    p.res_bs = B > 1 ? res->bstride : 0;
  }
  p.out = out;
  p.out_w = nout;
  p.n_rows = n_rows;
  p.n_tiles = (int)((n_rows + 127) / 128);
  if (ep) {
    p.step = 1;
    p.prev = ep->prev;
    p.bnd = ep->boundary;
    p.mask = ep->mask;
    p.dstd = ep->std;
    p.dmean = ep->mean;
    p.std_out = ep->std_out;
  }
  return std_form ? fz_launch<true>(p, "tc_rowmlp_kernel", bytes, st) : fz_launch(p, "tc_rowmlp_kernel", bytes, st);
}

// ---- two 64 -> 64 row Linears in one launch: out0 = x0·W0ᵀ (B0 batches), out1 = x1·W1ᵀ + b1 (B1 batches); W0, W1 are
// 64-column slices of the first Linear (in_dim 192) of an edge MLP
static int fz_rowlin2(const float* x0, int64_t x0_bs, int64_t rows0, int B0, const float* w0, float* out0, const float* x1,
                      int64_t x1_bs, int64_t rows1, int B1, const float* w1, const float* b1, float* out1, cudaStream_t st) {
  FzParams p;
  memset(&p, 0, sizeof(p));
  p.mode = fz::ROWLIN;
  p.n_src = 1;
  p.src[0] = FzSrc{x0, nullptr, B0 > 1 ? x0_bs : 0, 64};
  p.w1 = wslice(w0, 192, 64, 64);
  p.kc1 = 2;
  p.out = out0;
  p.out_w = 64;
  p.n_rows = rows0;
  p.n_tiles = (int)((rows0 + 127) / 128);
  p.B = B0;
  p.src1 = FzSrc{x1, nullptr, B1 > 1 ? x1_bs : 0, 64};
  p.w3 = wslice(w1, 192, 64, 64);
  p.b1_1 = b1;
  p.out_1 = out1;
  p.n_rows1 = rows1;
  p.n_tiles1 = (int)((rows1 + 127) / 128);
  p.B1 = B1;
  return fz_launch(p, "tc_rowlinear_kernel", 8.0 * 64 * ((double)rows0 * B0 + (double)rows1 * B1), st);
}

// ---- node projections of the split first edge Linear: P_s = x_s·W1sᵀ (B_s batches), P_r = x_r·W1rᵀ + b1 (B_r batches)
static int fz_projections(const NlamGraph* g, const NlamMlp* em, const float* send, int64_t send_bs, const float* rec,
                          int64_t rec_bs, int B, float* Ps, float* Pr, cudaStream_t st) {
  const int Bs = (send_bs == 0 || B == 1) ? 1 : B, Br = (rec_bs == 0 || B == 1) ? 1 : B;
  return fz_rowlin2(send, send_bs, g->n_send, Bs, em->w[0] + 64, Ps, rec, rec_bs, g->n_rec, Br, em->w[0] + 128, em->b[0], Pr, st);
}

// ---- edge stage: messages, optional edge output, per-receiver aggregate
static bool tc_edge_supported(const NlamGraph* g, const NlamMlp* edge_mlp, int flags) {
  int nout = 0;
  if (flags & NLAM_PROPAGATION) return false;
  if (!g || g->n_tiles <= 0) return false;
  if (!mlp_shape_ok(edge_mlp, &nout) || nout != 64 || edge_mlp->in_dim != 192 || !edge_mlp->ln_gamma) return false;
  return true;
}

// Which form and launch label an edge stage takes: the first rule that applies (DESIGN.md §4.1).  The split form and the
// K = 192 form round differently in TF32, and only tc_edge_rmw_kernel may write its edge output over its edge input, so the
// dispatch and every support query in abi.cu ask here.
//   1. no edge output, uniform in-degree 1..8: split, tc_ell_window_kernel, always with its own projection pass
//   2. E·B >= 2.5·(n_send·Bs + n_rec·Br): the projection pass is small next to the edge work (mesh graphs): split,
//      tc_edge_rmw_kernel without edge output or with it over a dense edge input, else tc_edge3_kernel
//   3. no edge output, edge features and receivers shared by the batch (grid -> mesh): split, tc_edge_bcast_kernel; both
//      projections are far fewer rows than the batch's edges
//   4. otherwise: K = 192 on raw gathered rows, tc_edge_kernel
// Rules 1 and 2 need send / rec 16-byte aligned and both batch strides % 4 == 0, rule 3 send / rec / edge aligned and
// send_bs % 4 == 0.  Bs (Br) is 1 for senders (receivers) shared by the batch, else B.
TcEdgePath tc_edge_path(const NlamGraph* g, const NlamMlp* edge_mlp, int flags, const float* send, int64_t send_bs,
                        const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs, const float* edge_out, int B) {
  if (!tc_edge_supported(g, edge_mlp, flags)) return {};
  const bool aligned = aligned16(send) && aligned16(rec) && send_bs % 4 == 0 && rec_bs % 4 == 0;
  if (!edge_out && g->uniform_degree >= 1 && g->uniform_degree <= 8 && aligned) return {"tc_ell_window_kernel", true, false};
  const double edge_rows = (double)g->n_edges * B;
  const double node_rows = (double)g->n_send * ((send_bs == 0 || B == 1) ? 1 : B) +
                           (double)g->n_rec * ((rec_bs == 0 || B == 1) ? 1 : B);
  if (aligned && edge_rows >= 2.5 * node_rows) {
    const bool rmw = !edge_out || (edge_out == edge && (B == 1 || edge_bs == g->n_edges * 64));
    return {rmw ? "tc_edge_rmw_kernel" : "tc_edge3_kernel", true, true};
  }
  if (!edge_out && (edge_bs == 0 || B == 1) && (rec_bs == 0 || B == 1) && aligned16(send) && aligned16(rec) && aligned16(edge) &&
      send_bs % 4 == 0)
    return {"tc_edge_bcast_kernel", true, true};
  return {"tc_edge_kernel", false, false};
}

size_t tc_edge_split_workspace_floats(const NlamGraph* g, int B) { return (size_t)B * (size_t)(g->n_send + g->n_rec) * 64 + 64; }

// split: A = e, + P_s[src] + P_r[dst] in the GEMM 1 epilogue (projections in ws, or from the previous layer when have_proj);
// otherwise A = [e | x_src | x_dst] (K = 192)
static int fz_edge(const NlamGraph* g, const NlamMlp* em, const float* send, int64_t send_bs, const float* rec, int64_t rec_bs,
                   const float* edge, int64_t edge_bs, float* edge_out, float* aggr_out, int B, int flags, cudaStream_t st,
                   float* ws, bool split, bool have_proj, const char* name) {
  NLAM_REQUIRE(tc_edge_supported(g, em, flags), NLAM_E_UNSUPPORTED, "%s: unsupported shape", name);
  NLAM_REQUIRE(aligned16(send) && aligned16(rec) && aligned16(edge) && aligned16(aggr_out) && (!edge_out || aligned16(edge_out)) &&
                   send_bs % 4 == 0 && rec_bs % 4 == 0 && edge_bs % 4 == 0,
               NLAM_E_INVALID, "%s: pointers / strides must be 16-byte aligned", name);
  const int Bs = (send_bs == 0 || B == 1) ? 1 : B, Br = (rec_bs == 0 || B == 1) ? 1 : B;
  const int64_t eb = B > 1 ? edge_bs : 0;
  const double bytes = edge_algorithmic_bytes(g, B, send_bs, rec_bs, edge_bs, edge_out != nullptr, 64);
  if (split) {
    // ws = [P_s (Bs batches) | P_r (Br batches)], computed here or (have_proj) by an earlier kernel
    float* Ps = ws;
    float* Pr = ws + (size_t)Bs * g->n_send * 64;
    if (!have_proj) {
      int rc = fz_projections(g, em, send, send_bs, rec, rec_bs, B, Ps, Pr, st);
      if (rc) return rc;
    }
    EdgeParams q;
    memset(&q, 0, sizeof(q));
    q.B = B;
    q.n_tiles = g->n_tiles;
    q.mean = (flags & NLAM_AGGR_MEAN) ? 1 : 0;
    q.tile_rec = g->tile_rec;
    q.tile_edge = g->tile_edge;
    q.rowptr = g->rowptr;
    q.src = g->src;
    q.dst = g->dst;
    q.edge = edge;
    q.edge_bs = eb;
    q.edge_out = edge_out;
    q.aggr = aggr_out;
    q.ps = Ps;
    q.pr = Pr;
    q.ps_bs = Bs > 1 ? g->n_send * 64 : 0;
    q.pr_bs = Br > 1 ? g->n_rec * 64 : 0;
    q.w1 = wslice(em->w[0], em->in_dim, 64, 64);  // the edge-feature columns; b1 is carried by P_r
    q.w2 = wslice(em->w[1], 64, em->out_dim[1], 64);
    q.b2 = em->b[1];
    q.gamma = em->ln_gamma;
    q.beta = em->ln_beta;
    q.eps = em->ln_eps;
    q.n_rec = g->n_rec;
    q.n_edges = g->n_edges;
    const long long n_work = (long long)q.n_tiles * B;
    const int grid = (int)std::min<long long>(n_work, num_sms());  // one CTA per SM
    return persistent_launch<tc_edge_split_kernel>(fz::THREADS, edg::BYTES, edg::BYTES, n_work, grid, name, bytes, st, q);
  }
  FzParams p;
  memset(&p, 0, sizeof(p));
  p.mode = fz::EDGE;
  p.B = B;
  p.n_src = 3;
  p.src[0] = FzSrc{edge, nullptr, eb, 64};
  p.src[1] = FzSrc{send, g->src, Bs > 1 ? send_bs : 0, 64};
  p.src[2] = FzSrc{rec, g->dst, Br > 1 ? rec_bs : 0, 64};
  fz_mlp(p, em, 0, 192);
  p.n_tiles = g->n_tiles;
  p.tile_rec = g->tile_rec;
  p.rowptr = g->rowptr;
  p.mean = (flags & NLAM_AGGR_MEAN) ? 1 : 0;
  p.edge = edge;
  p.edge_bs = eb;
  p.edge_out = edge_out;
  p.aggr = aggr_out;
  p.n_rec = g->n_rec;
  p.n_edges = g->n_edges;
  return fz_launch(p, name, bytes, st);
}

int tc_edge_split(const NlamGraph* g, const NlamMlp* edge_mlp, const float* send, int64_t send_bs, const float* rec,
                  int64_t rec_bs, const float* edge, int64_t edge_bs, float* edge_out, float* aggr_out, int B, int flags,
                  cudaStream_t st, float* ws, bool have_proj, const char* label) {
  return fz_edge(g, edge_mlp, send, send_bs, rec, rec_bs, edge, edge_bs, edge_out, aggr_out, B, flags, st, ws, true, have_proj,
                 label);
}

int tc_edge(const NlamGraph* g, const NlamMlp* edge_mlp, const float* send, int64_t send_bs, const float* rec, int64_t rec_bs,
            const float* edge, int64_t edge_bs, float* edge_out, float* aggr_out, int B, int flags, cudaStream_t st) {
  return fz_edge(g, edge_mlp, send, send_bs, rec, rec_bs, edge, edge_bs, edge_out, aggr_out, B, flags, st, nullptr, false, false,
                 "tc_edge_kernel");
}

// ---- node update chained with the next layer's projections / with output_map + step epilogue

bool tc_node_proj_supported(const NlamMlp* node_mlp, const NlamMlp* next_edge_mlp, const float* rec, int64_t rec_bs,
                            const float* aggr, int64_t n_rows, const float* out, const float* proj_out) {
  int no2 = 0;
  if (n_rows < 1 || n_rows >= (1LL << 31) - 256 || !node_mlp_ok(node_mlp)) return false;
  if (!mlp_shape_ok(next_edge_mlp, &no2) || no2 != 64 || next_edge_mlp->in_dim != 192) return false;
  return aligned16(rec) && aligned16(aggr) && aligned16(out) && aligned16(proj_out) && rec_bs % 4 == 0;
}

int tc_node_proj(const NlamMlp* node_mlp, const NlamMlp* next_edge_mlp, const float* rec, int64_t rec_bs, const float* aggr,
                 int64_t n_rows, int B, float* out, float* proj_out, cudaStream_t st) {
  NLAM_REQUIRE(tc_node_proj_supported(node_mlp, next_edge_mlp, rec, rec_bs, aggr, n_rows, out, proj_out), NLAM_E_UNSUPPORTED,
               "tc_node_proj: unsupported shapes");
  NodeParams p = node_params(node_mlp, rec, rec_bs, aggr, n_rows * 64, 0, n_rows, B, out);
  p.post = nod::POST_PROJ;
  p.w3 = wslice(next_edge_mlp->w[0] + 64, 192, 64, 64);
  p.w4 = wslice(next_edge_mlp->w[0] + 128, 192, 64, 64);
  p.b4 = next_edge_mlp->b[0];
  p.out3 = proj_out;
  p.out4 = proj_out + (size_t)B * n_rows * 64;
  const double bytes = 4.0 * n_rows * 64 * (((rec_bs != 0 && B > 1) ? B : 1) + 4.0 * B);
  return node_launch(p, "tc_node_proj_kernel", bytes, st);
}

bool tc_node_out_supported(const NlamMlp* node_mlp, const NlamMlp* out_mlp, const float* rec, int64_t rec_bs, const float* aggr,
                           int64_t n_rows, int B, const float* out, const StepEpilogue* ep) {
  int no2 = 0;
  (void)B;
  if (n_rows < 1 || n_rows >= (1LL << 31) - 256 || !node_mlp_ok(node_mlp)) return false;
  if (!mlp_shape_ok(out_mlp, &no2) || no2 >= 64 || out_mlp->in_dim != 64 || out_mlp->ln_gamma) return false;
  if (!(aligned16(rec) && aligned16(aggr) && rec_bs % 4 == 0 && out)) return false;
  if (ep && ep->std_out && no2 % 2) return false;  // the predicted-std form: 2·d outputs
  return ep && ep->prev && ep->std && ep->mean && (!ep->boundary || ep->mask);
}

int tc_node_out(const NlamMlp* node_mlp, const NlamMlp* out_mlp, const float* rec, int64_t rec_bs, const float* aggr,
                int64_t n_rows, int B, float* out, const StepEpilogue* ep, cudaStream_t st) {
  NLAM_REQUIRE(tc_node_out_supported(node_mlp, out_mlp, rec, rec_bs, aggr, n_rows, B, out, ep), NLAM_E_UNSUPPORTED,
               "tc_node_out: unsupported shapes");
  const int D = out_mlp->out_dim[1];
  NodeParams p = node_params(node_mlp, rec, rec_bs, aggr, n_rows * 64, 0, n_rows, B, out);
  p.post = nod::POST_OUTMLP;
  p.w3 = wslice(out_mlp->w[0], 64, 64, 64);
  p.b3 = out_mlp->b[0];
  p.w4 = wslice(out_mlp->w[1], 64, D, 64);
  p.b4 = out_mlp->b[1];
  p.out_w = D;
  p.prev = ep->prev;
  p.bnd = ep->boundary;
  p.mask = ep->mask;
  p.dstd = ep->std;
  p.dmean = ep->mean;
  p.std_out = ep->std_out;
  // previous / new (/ boundary) state and the std: d = D (D / 2 in the predicted-std form) columns each
  const bool std_form = ep->std_out != nullptr;
  const double bytes = 4.0 * n_rows * (64.0 * (((rec_bs != 0 && B > 1) ? B : 1) + B) + (std_form ? 4.0 * (D / 2) : 3.0 * D) * B);
  return std_form ? node_launch<true>(p, "tc_node_out_kernel", bytes, st) : node_launch(p, "tc_node_out_kernel", bytes, st);
}

// ---- mesh -> grid decoder: edge projections (tc_rowlinear_kernel) + tc_decode_kernel
bool tc_decode_supported(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* node_mlp, const NlamMlp* out_mlp, int flags,
                         const float* send, int64_t send_bs, const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs,
                         int B, const float* out, const StepEpilogue* ep) {
  int no = 0;
  if (flags & (NLAM_PROPAGATION | NLAM_MATH_FP32)) return false;
  if (!g || B < 1 || g->n_rec < 1 || g->n_edges >= (1LL << 31) - 256) return false;
  const int d = g->uniform_degree;
  if (d != 1 && d != 2 && d != 4 && d != 8) return false;
  if (!tc_edge_supported(g, edge_mlp, flags) || !node_mlp_ok(node_mlp)) return false;
  if (!mlp_shape_ok(out_mlp, &no) || no >= 64 || out_mlp->in_dim != 64 || out_mlp->ln_gamma) return false;
  // the kernel reads every bias and LayerNorm parameter: a bias-free Linear or an affine-free LayerNorm is not covered
  for (const NlamMlp* m : {edge_mlp, node_mlp, out_mlp})
    if (!m->b[0] || !m->b[1]) return false;
  if (!edge_mlp->ln_beta || !node_mlp->ln_beta) return false;
  if (!(edge_bs == 0 || B == 1)) return false;  // edge features shared by the batch: P_e is computed once
  if (!(aligned16(send) && aligned16(rec) && aligned16(edge) && send_bs % 4 == 0 && rec_bs % 4 == 0 && out)) return false;
  if (B > 1 && send_bs != 0 && send_bs < g->n_send * 64) return false;
  if (ep && ep->std_out && no % 2) return false;  // the predicted-std form: 2·d outputs
  return ep && ep->prev && ep->std && ep->mean && (!ep->boundary || ep->mask);
}

size_t tc_decode_workspace_floats(const NlamGraph* g, int B) {
  return ((size_t)B * g->n_send + (size_t)g->n_edges) * 64;  // P_s (up to B batches) | P_e
}

int tc_decode(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* node_mlp, const NlamMlp* out_mlp, int flags,
              const float* send, int64_t send_bs, const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs, int B,
              float* out, const StepEpilogue* ep, float* ws, cudaStream_t st) {
  NLAM_REQUIRE(tc_decode_supported(g, edge_mlp, node_mlp, out_mlp, flags, send, send_bs, rec, rec_bs, edge, edge_bs, B, out, ep),
               NLAM_E_UNSUPPORTED, "tc_decode: unsupported shapes");
  const int Bs = (send_bs == 0 || B == 1) ? 1 : B;
  float* Ps = ws;
  float* Pe = ws + (size_t)Bs * g->n_send * 64;
  // P_s = send·W1sᵀ per batch element, P_e = e·W1eᵀ + b1 once for the whole batch
  int rc = fz_rowlin2(send, send_bs, g->n_send, Bs, edge_mlp->w[0] + 64, Ps, edge, 0, g->n_edges, 1, edge_mlp->w[0],
                      edge_mlp->b[0], Pe, st);
  if (rc) return rc;
  DecParams p;
  memset(&p, 0, sizeof(p));
  p.B = B;
  p.d = g->uniform_degree;
  p.mean = (flags & NLAM_AGGR_MEAN) ? 1 : 0;
  p.D = out_mlp->out_dim[1];
  p.n_rec = g->n_rec;
  p.n_blocks = (g->n_rec + 63) / 64;
  p.rec = rec;
  p.rec_bs = B > 1 ? rec_bs : 0;
  p.ps = Ps;
  p.ps_bs = Bs > 1 ? g->n_send * 64 : 0;
  p.pe = Pe;
  p.src = g->src;
  p.w1r = wslice(edge_mlp->w[0] + 128, 192, 64, 64);
  p.w2e = wslice(edge_mlp->w[1], 64, 64, 64);
  p.wn1 = wslice(node_mlp->w[0], 128, 64, 128);
  p.wn2 = wslice(node_mlp->w[1], 64, 64, 64);
  p.wo1 = wslice(out_mlp->w[0], 64, 64, 64);
  p.wo2 = wslice(out_mlp->w[1], 64, p.D, 64);
  p.b2e = edge_mlp->b[1];
  p.gamma_e = edge_mlp->ln_gamma;
  p.beta_e = edge_mlp->ln_beta;
  p.eps_e = edge_mlp->ln_eps;
  p.bn1 = node_mlp->b[0];
  p.bn2 = node_mlp->b[1];
  p.gamma_n = node_mlp->ln_gamma;
  p.beta_n = node_mlp->ln_beta;
  p.eps_n = node_mlp->ln_eps;
  p.bo1 = out_mlp->b[0];
  p.bo2 = out_mlp->b[1];
  p.out = out;
  p.prev = ep->prev;
  p.bnd = ep->boundary;
  p.mask = ep->mask;
  p.dstd = ep->std;
  p.dmean = ep->mean;
  p.std_out = ep->std_out;
  const bool std_form = ep->std_out != nullptr;
  const long long n_items = p.n_blocks * B;
  const int grid = (int)std::min<long long>((n_items + 1) / 2, num_sms());  // one CTA per SM, two items at a time
  // algorithmic bytes: receivers, P_s, P_e and the sender indices once, previous / new (/ boundary) state and the std
  // (Ds columns each), weights
  const int D = p.D, Ds = std_form ? D / 2 : D, Br = (rec_bs != 0 && B > 1) ? B : 1;
  const double bytes = 256.0 * ((double)g->n_rec * Br + (double)g->n_send * Bs + (double)g->n_edges) + 4.0 * g->n_edges +
                       4.0 * (double)g->n_rec * Ds * B * ((ep->boundary ? 3 : 2) + (std_form ? 1 : 0)) +
                       (ep->boundary ? 4.0 * g->n_rec : 0.0) + 4.0 * (7 * 64 * 64 + 64 * D + 9 * 64);
  using Launch = int (*)(int, size_t, size_t, long long, int, const char*, double, cudaStream_t, const DecParams&);
  static const Launch launches[2][4] = {
      {persistent_launch<tc_decode_kernel<1, false>, DecParams>, persistent_launch<tc_decode_kernel<2, false>, DecParams>,
       persistent_launch<tc_decode_kernel<4, false>, DecParams>, persistent_launch<tc_decode_kernel<8, false>, DecParams>},
      {persistent_launch<tc_decode_kernel<1, true>, DecParams>, persistent_launch<tc_decode_kernel<2, true>, DecParams>,
       persistent_launch<tc_decode_kernel<4, true>, DecParams>, persistent_launch<tc_decode_kernel<8, true>, DecParams>}};
  const Launch launch = launches[std_form][p.d == 1 ? 0 : p.d == 2 ? 1 : p.d == 4 ? 2 : 3];
  return launch(dec::THREADS, dec::BYTES, dec::BYTES, n_items, grid, "tc_decode_kernel", bytes, st, p);
}

// ---- grid encoder: grid embedder + g2m node projections + encoding grid MLP (tc_encode_kernel)
static bool enc_mlp_ok(const NlamMlp* m, int in_max) {  // in -> 64 -> 64 with biases and an affine LayerNorm
  int no = 0;
  return mlp_shape_ok(m, &no) && no == 64 && m->in_dim <= in_max && m->b[0] && m->b[1] && m->ln_gamma && m->ln_beta;
}

bool tc_encode_supported(const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src, const NlamMlp* grid_mlp,
                         const NlamMlp* g2m_edge_mlp, const float* mesh, int64_t n_mesh, int64_t n_rows, int B, int flags) {
  if (flags & (NLAM_PROPAGATION | NLAM_MATH_FP32)) return false;
  if (B < 1 || n_rows < 1 || n_rows >= (1LL << 31) - 256 || n_mesh < 1 || n_src < 1 || n_src > 4) return false;
  if (!enc_mlp_ok(embed_mlp, 64) || !enc_mlp_ok(grid_mlp, 64) || grid_mlp->in_dim != 64) return false;
  if (!enc_mlp_ok(g2m_edge_mlp, 192) || g2m_edge_mlp->in_dim != 192) return false;
  int k = 0;
  for (int s = 0; s < n_src; ++s) {
    if (srcs[s].idx || srcs[s].dim < 1 || ((uintptr_t)srcs[s].ptr & 3)) return false;
    k += srcs[s].dim;
  }
  return k == embed_mlp->in_dim && aligned16(mesh);
}

int tc_encode(const NlamMlp* embed_mlp, const NlamRowSrc* srcs, int n_src, const NlamMlp* grid_mlp, const NlamMlp* g2m_edge_mlp,
              const float* mesh, int64_t n_mesh, int64_t n_rows, int B, int flags, float* grid_rep, float* ps, float* pr,
              float* grid_emb, cudaStream_t st, const NlamMlp* g2m_edge_mlp_b, float* ps_b, float* pr_b) {
  NLAM_REQUIRE(tc_encode_supported(embed_mlp, srcs, n_src, grid_mlp, g2m_edge_mlp, mesh, n_mesh, n_rows, B, flags),
               NLAM_E_UNSUPPORTED, "tc_encode: unsupported shapes");
  const bool two = g2m_edge_mlp_b != nullptr;
  NLAM_REQUIRE(!two || (enc_mlp_ok(g2m_edge_mlp_b, 192) && g2m_edge_mlp_b->in_dim == 192), NLAM_E_UNSUPPORTED,
               "tc_encode: unsupported second g2m edge MLP");
  NLAM_REQUIRE(!(two && grid_emb), NLAM_E_INVALID, "tc_encode: grid_emb is not stored with a second g2m edge MLP");
  NLAM_REQUIRE(aligned16(grid_rep) && aligned16(ps) && aligned16(pr) && aligned16(grid_emb) && aligned16(ps_b) &&
                   aligned16(pr_b) && (!two || (ps_b && pr_b)),
               NLAM_E_INVALID, "tc_encode: unaligned or missing outputs");
  EncParams p;
  memset(&p, 0, sizeof(p));
  p.B = B;
  p.n_src = n_src;
  double bytes = 0;
  for (int s = 0; s < n_src; ++s) {
    p.src[s] = FzSrc{srcs[s].ptr, nullptr, B > 1 ? srcs[s].bstride : 0, srcs[s].dim};
    bytes += 4.0 * n_rows * srcs[s].dim * ((srcs[s].bstride != 0 && B > 1) ? B : 1);
  }
  p.n_rows = n_rows;
  p.n_tiles = (n_rows + 63) / 64;
  p.we1 = wslice(embed_mlp->w[0], embed_mlp->in_dim, 64, embed_mlp->in_dim);
  p.we2 = wslice(embed_mlp->w[1], 64, 64, 64);
  p.w1s = wslice(g2m_edge_mlp->w[0] + 64, 192, 64, 64);
  p.wa1 = wslice(grid_mlp->w[0], 64, 64, 64);
  p.wa2 = wslice(grid_mlp->w[1], 64, 64, 64);
  p.w1r = wslice(g2m_edge_mlp->w[0] + 128, 192, 64, 64);
  p.be1 = embed_mlp->b[0];
  p.be2 = embed_mlp->b[1];
  p.gamma_e = embed_mlp->ln_gamma;
  p.beta_e = embed_mlp->ln_beta;
  p.eps_e = embed_mlp->ln_eps;
  p.ba1 = grid_mlp->b[0];
  p.ba2 = grid_mlp->b[1];
  p.gamma_a = grid_mlp->ln_gamma;
  p.beta_a = grid_mlp->ln_beta;
  p.eps_a = grid_mlp->ln_eps;
  p.b1 = g2m_edge_mlp->b[0];
  p.grid_rep = grid_rep;
  p.ps = ps;
  p.grid_emb = grid_emb;
  p.mesh = mesh;
  p.pr = pr;
  p.n_mesh = n_mesh;
  p.n_mesh_tiles = (n_mesh + 63) / 64;
  if (two) {
    p.w1s_b = wslice(g2m_edge_mlp_b->w[0] + 64, 192, 64, 64);
    p.w1r_b = wslice(g2m_edge_mlp_b->w[0] + 128, 192, 64, 64);
    p.b1_b = g2m_edge_mlp_b->b[0];
    p.ps_b = ps_b;
    p.pr_b = pr_b;
  }
  const long long n_items = p.n_tiles * B + (two ? 2 : 1) * p.n_mesh_tiles;
  const int grid = (int)std::min<long long>((n_items + 1) / 2, num_sms());  // one CTA per SM, two items at a time
  // algorithmic bytes: the inputs once, grid_rep and P_s (and grid_emb or P_s_b), the mesh rows and P_r (and P_r_b), the
  // weights
  bytes += ((grid_emb || two) ? 3.0 : 2.0) * 4.0 * 64 * n_rows * B + (two ? 3.0 : 2.0) * 4.0 * 64 * n_mesh +
           4.0 * (embed_mlp->in_dim * 64 + (two ? 7 : 5) * 64 * 64 + (two ? 10 : 9) * 64);
  const size_t smem = two ? enc::Layout<true>::BYTES : enc::Layout<false>::BYTES;
  const auto launch = two        ? persistent_launch<tc_encode_kernel<false, true>, EncParams>
                      : grid_emb ? persistent_launch<tc_encode_kernel<true, false>, EncParams>
                                 : persistent_launch<tc_encode_kernel<false, false>, EncParams>;
  return launch(fz::THREADS, smem, smem, n_items, grid, two ? "tc_encode2_kernel" : "tc_encode_kernel", bytes, st, p);
}

// ---- Graph-EFM latent step: latent_param_map + sample + latent_embedder (tc_latent_kernel)
bool tc_latent_supported(const NlamMlp* param_mlp, const NlamMlp* embed_mlp, const float* x, int64_t x_bs, const float* eps,
                         int64_t eps_bs, const float* out, int64_t n_rows, int B, int flags) {
  if (flags & (NLAM_PROPAGATION | NLAM_MATH_FP32)) return false;
  if (B < 1 || n_rows < 1 || n_rows >= (1LL << 31) - 256) return false;
  // latent_param_map: 64 -> 64 -> 64 (isotropic) or 128 (diagonal), biases, no LayerNorm
  const NlamMlp* m = param_mlp;
  if (m->n_linear != 2 || m->in_dim != 64 || m->out_dim[0] != 64 || (m->out_dim[1] != 64 && m->out_dim[1] != 128)) return false;
  if (m->ln_gamma || !m->b[0] || !m->b[1]) return false;
  if (!aligned16(m->w[0]) || !aligned16(m->w[1]) || !aligned16(m->b[0]) || !aligned16(m->b[1])) return false;
  if (!enc_mlp_ok(embed_mlp, 64) || embed_mlp->in_dim != 64) return false;
  if (!x || !eps || !out || !aligned16(x) || !aligned16(eps) || !aligned16(out)) return false;
  return x_bs >= 0 && eps_bs >= 0 && x_bs % 4 == 0 && eps_bs % 4 == 0;
}

int tc_latent(const NlamMlp* param_mlp, const NlamMlp* embed_mlp, const float* x, int64_t x_bs, const float* eps, int64_t eps_bs,
              float* out, int64_t n_rows, int B, int flags, cudaStream_t st) {
  NLAM_REQUIRE(tc_latent_supported(param_mlp, embed_mlp, x, x_bs, eps, eps_bs, out, n_rows, B, flags), NLAM_E_UNSUPPORTED,
               "tc_latent: unsupported shapes");
  LatParams p;
  memset(&p, 0, sizeof(p));
  p.B = B;
  p.diag = param_mlp->out_dim[1] == 128;
  p.n_rows = n_rows;
  p.n_tiles = (n_rows + 63) / 64;
  p.x = x;
  p.x_bs = B > 1 ? x_bs : 0;
  p.eps = eps;
  p.eps_bs = B > 1 ? eps_bs : 0;
  p.w1 = wslice(param_mlp->w[0], 64, 64, 64);
  p.w2m = wslice(param_mlp->w[1], 64, 64, 64);
  p.w2s = wslice(param_mlp->w[1] + 64 * 64, 64, 64, 64);
  p.w3 = wslice(embed_mlp->w[0], 64, 64, 64);
  p.w4 = wslice(embed_mlp->w[1], 64, 64, 64);
  p.b1 = param_mlp->b[0];
  p.b2m = param_mlp->b[1];
  p.b2s = param_mlp->b[1] + 64;
  p.b3 = embed_mlp->b[0];
  p.b4 = embed_mlp->b[1];
  p.gamma = embed_mlp->ln_gamma;
  p.beta = embed_mlp->ln_beta;
  p.ln_eps = embed_mlp->ln_eps;
  p.out = out;
  const long long n_items = p.n_tiles * B;
  const int grid = (int)std::min<long long>((n_items + 1) / 2, num_sms());  // one CTA per SM, two items at a time
  // algorithmic bytes: x, eps and latent_emb once, the weights
  const double bytes = 3.0 * 4.0 * 64 * n_rows * B + 4.0 * ((p.diag ? 5 : 4) * 64 * 64 + (p.diag ? 8 : 7) * 64);
  return persistent_launch<tc_latent_kernel>(fz::THREADS, lat::BYTES, lat::BYTES, n_items, grid, "tc_latent_kernel", bytes, st, p);
}

}  // namespace nlam

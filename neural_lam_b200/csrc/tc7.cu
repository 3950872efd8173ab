// Generic tensor-core Linear kernel (sm_90a: wgmma TF32) for hidden widths and layer variants the fused kernels do not
// cover:
//
//     Y[r, :] = epi( [X0 | X1][r, :] · Wᵀ + bias + A0[idx0[r], :] + A1[idx1[r], :] )
//     epi: none | SiLU | LayerNorm, then "+ post[idxp[r]]" (PropagationNet's x_j + edge_mlp(...)), a second output before
//     the residual (the message m next to e' = e + m) and "+ residual".
//
// One CTA tile = 128 rows x N (N = the full output width <= 256), K streamed in 32-column chunks through a ring of
// shared-memory stages: the X chunk (16 KB) and the W chunk (N x 128 B, L2 resident) arrive by TMA with 128-byte swizzle,
// the two consumer warp groups round the stage to TF32 in place (to nearest, as fused.cu does: TMA copies raw fp32, which
// the MMA would truncate; each warp group rounds its 64 rows of X and half of the W chunk, then fence.proxy.async and a
// named barrier of both), and each runs `wgmma.mma_async m64nNk8 .tf32` on its 64 rows of the stage, accumulating in
// registers; the epilogue works on the accumulator fragments (a row is spread over the 4 threads of a quad; LayerNorm
// statistics are reduced with two shuffles).  Warp group 0 is the TMA producer.
// An MLP (reference utils/networks.py:27-40) is two launches with the hidden activations in a workspace; an
// InteractionNet (reference gnn_layers.py:110-157) is: node projections of the split first edge Linear, edge layer 1
// (gathered projections added in the epilogue, SiLU), edge layer 2 (LayerNorm, m and e' = e + m), CSR segment sum,
// node layers 1 / 2.
#include "tc_ptx.cuh"
#include "wgmma_tf32.cuh"

namespace nlam {

namespace g7 {
constexpr int THREADS = 384;           // warp group 0: TMA producer (one thread); warp groups 1 / 2: rows 0-63 / 64-127
constexpr int KC = 32;                 // K columns per chunk (128 bytes: one swizzle row)
constexpr uint32_t A_BYTES = 128 * 128;  // 128 rows x 128 B
}  // namespace g7

struct LinParams {
  int n_tiles;       // row tiles per batch
  int B;
  long long n_rows;
  int kc0, kc1;      // chunks of source 0 / source 1
  int a_batched[2];
  int w_batched;
  int n_real;        // real output width (<= N; < N only for direct narrow stores)
  const float* bias;
  int act;           // 0 none, 1 SiLU
  const float* gamma;
  const float* beta;
  float eps;
  // pre-activation gathered addends (rows of width N)
  const float* add[2];
  const int32_t* add_idx[2];
  long long add_bs[2];
  // post-epilogue gathered addend (PropagationNet)
  const float* post;
  const int32_t* post_idx;
  long long post_bs;
  // residual (row r of the residual tensor; batch stride 0 = broadcast)
  const float* res;
  long long res_bs;
  float* out;        // (B, n_rows, n_real)
  float* out2;       // optional: value before the residual
  int stages;
};

__device__ __forceinline__ void add_row2(float* v, const float* row, int N) {
  // v[2j + e] += row[8j + e]: the column pairs one thread holds of a row (row already offset by 2 * (lane & 3))
  for (int j = 0; j < N / 8; ++j) {
    const float2 x = __ldg(reinterpret_cast<const float2*>(row + 8 * j));
    v[2 * j] += x.x;
    v[2 * j + 1] += x.y;
  }
}

template <int N>
__global__ void __launch_bounds__(g7::THREADS, 1)
tc_linear_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                 const __grid_constant__ CUtensorMap tmW, const LinParams p) {
  using namespace g7;
  constexpr uint32_t W_BYTES = N * 128;
  constexpr uint32_t STG_BYTES = A_BYTES + W_BYTES;
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int wg = warp >> 2;
  const int NSTG = p.stages;
  const uint32_t off_misc = (uint32_t)NSTG * STG_BYTES;
  const uint32_t mb = sbase + off_misc;
  const uint32_t bar_full = mb;        // [8] TMA bytes landed
  const uint32_t bar_empty = mb + 64;  // [8] 8 arrivals: every consumer warp has finished its MMAs on the stage
  float* sprm = reinterpret_cast<float*>(smem + off_misc + 256);  // bias | gamma | beta (N each)
  if ((sbase & 1023u) != 0) {
    if (tid == 0) printf("nlam tc_linear: dynamic shared memory not 1024-byte aligned\n");
    __trap();
  }
  if (tid == 0) {
    for (int s = 0; s < NSTG; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA0) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA1) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW) : "memory");
  }
  for (int i = tid; i < N; i += THREADS) {
    sprm[i] = (p.bias && i < p.n_real) ? p.bias[i] : 0.f;
    sprm[N + i] = p.gamma ? p.gamma[i] : 1.f;
    sprm[2 * N + i] = p.beta ? p.beta[i] : 0.f;
  }
  __syncthreads();
  const long long n_work = (long long)p.n_tiles * p.B;
  const int kc_total = p.kc0 + p.kc1;

  if (wg == 0) {
    // =============================== TMA producer ===============================
    if (tid == 0) {
      const uint64_t pol_stream = policy_evict_first();
      const uint64_t pol_keep = policy_evict_last();
      long long c = 0;  // chunk counter over the whole kernel
      for (long long w = blockIdx.x; w < n_work; w += gridDim.x) {
        const int b = (int)(w / p.n_tiles), tile = (int)(w - (long long)b * p.n_tiles);
        for (int kc = 0; kc < kc_total; ++kc, ++c) {
          const int s = (int)(c % NSTG);
          mbar_wait(bar_empty + 8 * s, (uint32_t)(((c / NSTG) & 1) ^ 1));
          const uint32_t full = bar_full + 8 * s;
          mbar_expect_tx(full, STG_BYTES);
          const uint32_t sa = sbase + s * STG_BYTES;
          if (kc < p.kc0)
            tma_load_3d(sa, &tmA0, full, kc * KC, tile * 128, p.a_batched[0] ? b : 0, pol_stream);
          else
            tma_load_3d(sa, &tmA1, full, (kc - p.kc0) * KC, tile * 128, p.a_batched[1] ? b : 0, pol_stream);
          tma_load_3d(sa + A_BYTES, &tmW, full, kc * KC, 0, p.w_batched ? b : 0, pol_keep);
        }
      }
    }
    return;
  }
  // ================= consumers: wgmma (64 rows x N per warp group), then the epilogue from registers =================
  // accumulator fragment of m64nNk8: acc[4j + 2i + e] is row 16 * (warp & 3) + lane / 4 + 8 i, column 8j + 2 (lane & 3) + e
  const int half = wg - 1;
  const int ct = tid - 128, ct128 = tid & 127;  // thread index among the 256 consumer threads / in its warp group
  const int rq = 64 * half + 16 * (warp & 3) + (lane >> 2);
  const int cq = 2 * (lane & 3);
  long long c = 0;
  for (long long w = blockIdx.x; w < n_work; w += gridDim.x) {
    const int b = (int)(w / p.n_tiles), tile = (int)(w - (long long)b * p.n_tiles);
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    for (int kc = 0; kc < kc_total; ++kc, ++c) {
      const int s = (int)(c % NSTG);
      mbar_wait(bar_full + 8 * s, (uint32_t)((c / NSTG) & 1));
      {  // round the stage to TF32 in place: this warp group's 64 rows of A, and its half of the W chunk
        float4* sa = reinterpret_cast<float4*>(smem + s * STG_BYTES + half * (A_BYTES / 2));
#pragma unroll
        for (int i = 0; i < (int)(A_BYTES / 2 / 16 / 128); ++i) sa[ct128 + 128 * i] = tf32r4(sa[ct128 + 128 * i]);
        float4* sw = reinterpret_cast<float4*>(smem + s * STG_BYTES + A_BYTES);
#pragma unroll
        for (int i = 0; i < (int)(W_BYTES / 16 / 256); ++i) sw[ct + 256 * i] = tf32r4(sw[ct + 256 * i]);
        // the rounded values are read by this stage's MMAs (async proxy), and the stage is next overwritten by TMA
        fence_proxy_async();
        named_bar_sync(1, 256);  // both consumer warp groups: the whole W chunk is rounded
      }
      const uint64_t da = gmma_desc(sbase + s * STG_BYTES + half * (A_BYTES / 2));
      const uint64_t db = gmma_desc(sbase + s * STG_BYTES + A_BYTES);
      wgmma_fence(acc, N / 2);
#pragma unroll
      for (int k = 0; k < 4; ++k) Wgmma<N>::mma(acc, da + 2 * k, db + 2 * k, (uint32_t)((kc | k) != 0));
      wgmma_commit();
      wgmma_wait0(acc, N / 2);
      if (lane == 0) mbar_arrive(bar_empty + 8 * s);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const long long r = (long long)tile * 128 + rq + 8 * i;
      const bool valid = r < p.n_rows;
      float v[N / 4];
#pragma unroll
      for (int j = 0; j < N / 8; ++j) {
        v[2 * j] = acc[4 * j + 2 * i] + sprm[8 * j + cq];
        v[2 * j + 1] = acc[4 * j + 2 * i + 1] + sprm[8 * j + cq + 1];
      }
      float mu = 0.f, rstd = 1.f;
      if (p.gamma) quad_row_stats<N / 4>(v, p.eps, mu, rstd);  // LayerNorm statistics of the row (all 4 quad lanes)
      if (!valid) continue;
      for (int a = 0; a < 2; ++a)
        if (p.add[a])
          add_row2(v, p.add[a] + (long long)b * p.add_bs[a] + (long long)(p.add_idx[a] ? __ldg(p.add_idx[a] + r) : r) * N + cq, N);
      if (p.act) {
#pragma unroll
        for (int j = 0; j < N / 4; ++j) v[j] = silu_fast(v[j]);
      }
      if (p.gamma) {
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
          v[2 * j] = fmaf((v[2 * j] - mu) * rstd, sprm[N + 8 * j + cq], sprm[2 * N + 8 * j + cq]);
          v[2 * j + 1] = fmaf((v[2 * j + 1] - mu) * rstd, sprm[N + 8 * j + cq + 1], sprm[2 * N + 8 * j + cq + 1]);
        }
      }
      if (p.post)
        add_row2(v, p.post + (long long)b * p.post_bs + (long long)(p.post_idx ? __ldg(p.post_idx + r) : r) * N + cq, N);
      if (p.out2) {
        float* o2 = p.out2 + ((long long)b * p.n_rows + r) * N + cq;
#pragma unroll
        for (int j = 0; j < N / 8; ++j) *reinterpret_cast<float2*>(o2 + 8 * j) = make_float2(v[2 * j], v[2 * j + 1]);
      }
      if (p.res) add_row2(v, p.res + (long long)b * p.res_bs + r * N + cq, N);
      float* orow = p.out + ((long long)b * p.n_rows + r) * p.n_real;
      if (p.n_real == N) {
#pragma unroll
        for (int j = 0; j < N / 8; ++j) *reinterpret_cast<float2*>(orow + 8 * j + cq) = make_float2(v[2 * j], v[2 * j + 1]);
      } else {
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
          if (8 * j + cq < p.n_real) orow[8 * j + cq] = v[2 * j];
          if (8 * j + cq + 1 < p.n_real) orow[8 * j + cq + 1] = v[2 * j + 1];
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------ host
static int npad(int n) { return n <= 32 ? 32 : n <= 64 ? 64 : n <= 128 ? 128 : 256; }

bool tc_linear_shape_ok(int k0, int k1, int n_out) {
  if (n_out < 1 || n_out > 256) return false;
  if (k0 < 32 || k0 % 32 != 0 || k1 % 32 != 0 || (long long)k0 + k1 > (1LL << 26)) return false;
  return true;
}

int tc_linear(const LinearCall& c, cudaStream_t st) {
  using namespace g7;
  const int N = npad(c.n_out);
  NLAM_REQUIRE(tc_linear_shape_ok(c.k0, c.k1, c.n_out), NLAM_E_UNSUPPORTED, "tc_linear: unsupported shape K=%d+%d N=%d", c.k0,
               c.k1, c.n_out);
  NLAM_REQUIRE(c.n_out == N || (!c.out2 && !c.res && !c.post && !c.add[0] && !c.add[1] && !c.gamma), NLAM_E_UNSUPPORTED,
               "tc_linear: narrow outputs support bias / activation only");
  NLAM_REQUIRE(aligned16(c.x0) && aligned16(c.w) && (!c.x1 || aligned16(c.x1)) && aligned16(c.out) && c.ldw % 4 == 0,
               NLAM_E_INVALID, "tc_linear: pointers must be 16-byte aligned");
  CUtensorMap ma0, ma1, mw;
  const bool b0 = c.x0_bs != 0 && c.B > 1, b1 = c.x1 && c.x1_bs != 0 && c.B > 1;
  const uint64_t pitch0 = c.x0_pitch ? (uint64_t)c.x0_pitch : (uint64_t)c.k0;
  NLAM_REQUIRE(pitch0 % 4 == 0 && c.x0_bs % 4 == 0 && c.w_bs % 4 == 0, NLAM_E_INVALID, "tc_linear: pitches must be multiples of 4");
  int rc = make_map(&ma0, c.x0, (uint64_t)c.k0, (uint64_t)c.n_rows, b0 ? (uint64_t)c.B : 1, pitch0,
                    b0 ? (uint64_t)c.x0_bs : (uint64_t)c.n_rows * pitch0, 128, true);
  if (rc) return rc;
  if (c.x1) {
    rc = make_map(&ma1, c.x1, (uint64_t)c.k1, (uint64_t)c.n_rows, b1 ? (uint64_t)c.B : 1, (uint64_t)c.k1,
                  b1 ? (uint64_t)c.x1_bs : (uint64_t)c.n_rows * c.k1, 128, true);
    if (rc) return rc;
  } else {
    ma1 = ma0;
  }
  // W: (n_out rows, k0 + k1 columns) slice of a row-major matrix with row pitch ldw; rows past n_out read as zero
  const bool wb = c.w_bs != 0 && c.B > 1;
  rc = make_map(&mw, c.w, (uint64_t)(c.w_cols ? c.w_cols : c.k0 + c.k1), (uint64_t)c.n_out, wb ? (uint64_t)c.B : 1, (uint64_t)c.ldw,
                wb ? (uint64_t)c.w_bs : (uint64_t)c.n_out * c.ldw, (uint32_t)N, true);
  if (rc) return rc;
  LinParams p;
  memset(&p, 0, sizeof(p));
  p.n_tiles = (int)((c.n_rows + 127) / 128);
  p.B = c.B;
  p.n_rows = c.n_rows;
  p.kc0 = c.k0 / KC;
  p.kc1 = c.x1 ? c.k1 / KC : 0;
  p.a_batched[0] = b0;
  p.a_batched[1] = b1;
  p.w_batched = wb;
  p.n_real = c.n_out;
  p.bias = c.bias;
  p.act = c.act;
  p.gamma = c.gamma;
  p.beta = c.beta;
  p.eps = c.eps;
  for (int i = 0; i < 2; ++i) {
    p.add[i] = c.add[i];
    p.add_idx[i] = c.add_idx[i];
    p.add_bs[i] = c.B > 1 ? c.add_bs[i] : 0;
  }
  p.post = c.post;
  p.post_idx = c.post_idx;
  p.post_bs = c.B > 1 ? c.post_bs : 0;
  p.res = c.res;
  p.res_bs = c.B > 1 ? c.res_bs : 0;
  p.out = c.out;
  p.out2 = c.out2;
  const uint32_t stg = A_BYTES + (uint32_t)N * 128;
  p.stages = (int)std::min<uint32_t>(8, (220 * 1024 - 4096) / stg);
  const size_t smem = (size_t)p.stages * stg + 256 + 3 * N * sizeof(float) + 64;
  const long long n_work = (long long)p.n_tiles * p.B;
  NLAM_REQUIRE(n_work >= 1 && n_work < (1LL << 40), NLAM_E_INVALID, "tc_linear: bad work size");
  const int grid = (int)std::min<long long>(n_work, num_sms());
  double bytes = 4.0 * c.n_rows * ((double)c.k0 * (b0 ? c.B : 1) + (c.x1 ? (double)c.k1 * (b1 ? c.B : 1) : 0.0)) +
                 4.0 * c.n_rows * c.B * c.n_out * (c.out2 ? 2 : 1) + 4.0 * c.n_out * (c.k0 + c.k1);
  for (int i = 0; i < 2; ++i)
    if (c.add[i]) bytes += 4.0 * c.n_rows * c.B * N;
  if (c.res) bytes += 4.0 * c.n_rows * N * (c.res_bs != 0 ? c.B : 1);
  if (c.post) bytes += 4.0 * c.n_rows * c.B * N;
  int dev = 0;
  NLAM_CUDA_OK(cudaGetDevice(&dev));
#define NLAM_LAUNCH_LIN(NN)                                                                                          \
  {                                                                                                                  \
    static unsigned mask = 0;                                                                                        \
    if (!(mask & (1u << (dev & 31)))) {                                                                              \
      NLAM_CUDA_OK(cudaFuncSetAttribute(tc_linear_kernel<NN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 225 * 1024)); \
      mask |= 1u << (dev & 31);                                                                                      \
    }                                                                                                                \
    ProfScope ps("tc_linear_kernel<" #NN ">", st, bytes);                                                            \
    tc_linear_kernel<NN><<<grid, THREADS, smem, st>>>(ma0, ma1, mw, p);                                              \
  }
  if (N == 32) NLAM_LAUNCH_LIN(32)
  else if (N == 64) NLAM_LAUNCH_LIN(64)
  else if (N == 128) NLAM_LAUNCH_LIN(128)
  else NLAM_LAUNCH_LIN(256)
#undef NLAM_LAUNCH_LIN
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

// Two-Linear MLP (Linear, SiLU, Linear[, LayerNorm]) over up to two dense row blocks, residual optional: two launches,
// hidden activations in `ws` (n_rows * B * hidden floats).
bool tc_mlp2_supported(const NlamMlp* m, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res, const NlamRowSrc* res2) {
  if (m->n_linear != 2 || res2) return false;
  const int H = m->out_dim[0], no = m->out_dim[1];
  if (!(H == 128 || H == 256) || no < 1 || no > 256) return false;
  if (m->ln_gamma && no != npad(no)) return false;
  if (n_src < 1 || n_src > 2) return false;
  int k = 0;
  for (int s = 0; s < n_src; ++s) {
    if (srcs[s].idx || srcs[s].dim % 32 != 0 || srcs[s].dim < 32 || !aligned16(srcs[s].ptr) || srcs[s].bstride % 4 != 0) return false;
    k += srcs[s].dim;
  }
  if (k != m->in_dim || k > 1024) return false;
  if (res && (res->idx || res->dim != no || no != npad(no))) return false;
  return aligned16(m->w[0]) && aligned16(m->w[1]);
}

int tc_mlp2(const NlamMlp* m, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res, float* out, int64_t n_rows, int B,
            cudaStream_t st, float* ws) {
  const int H = m->out_dim[0], no = m->out_dim[1];
  LinearCall c;
  memset(&c, 0, sizeof(c));
  c.x0 = srcs[0].ptr;
  c.x0_bs = srcs[0].bstride;
  c.k0 = srcs[0].dim;
  if (n_src == 2) {
    c.x1 = srcs[1].ptr;
    c.x1_bs = srcs[1].bstride;
    c.k1 = srcs[1].dim;
  }
  // batch-broadcast inputs: the hidden layer is computed once and broadcast
  bool any_batched = false;
  for (int s = 0; s < n_src; ++s) any_batched |= (srcs[s].bstride != 0 && B > 1);
  const int Bh = any_batched ? B : 1;
  c.w = m->w[0];
  c.ldw = m->in_dim;
  c.bias = m->b[0];
  c.n_out = H;
  c.act = 1;
  c.n_rows = n_rows;
  c.B = Bh;
  c.out = ws;
  int rc = tc_linear(c, st);
  if (rc) return rc;
  LinearCall d;
  memset(&d, 0, sizeof(d));
  d.x0 = ws;
  d.x0_bs = Bh > 1 ? (int64_t)n_rows * H : 0;
  d.k0 = H;
  d.w = m->w[1];
  d.ldw = H;
  d.bias = m->b[1];
  d.n_out = no;
  d.gamma = m->ln_gamma;
  d.beta = m->ln_beta;
  d.eps = m->ln_eps;
  if (res) {
    d.res = res->ptr;
    d.res_bs = res->bstride;
  }
  d.n_rows = n_rows;
  d.B = B;
  d.out = out;
  return tc_linear(d, st);
}

// ---- narrow / concatenated inputs (grid embedder: prev | prev_prev | forcing | static, reference graph/base.py:275-283)
// at H = 128 / 256: the sources are packed into one zero-padded dense (rows, Kp) block first, then the two Linear launches
// (a source with a row index gathers: row r of the block is row idx[r] of the source — the [e | x_src | x_dst] rows of an
// edge MLP whose per-chunk weights rule out the fused edge kernels: SplitMLPs, reference gnn_layers.py:274-324)
struct PackIdx {
  const int32_t* i[4];
};
__global__ void pack_rows_kernel(const float* s0, const float* s1, const float* s2, const float* s3, int d0, int d1, int d2,
                                 int d3, long long bs0, long long bs1, long long bs2, long long bs3, float* out, int kp,
                                 long long n_rows, int B, PackIdx ix) {
  const long long total = (long long)B * n_rows * kp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % kp);
    const long long r = (i / kp) % n_rows;
    const int b = (int)(i / ((long long)kp * n_rows));
    float v = 0.f;
    int cc = c;
    if (cc < d0) v = s0[b * bs0 + (ix.i[0] ? (long long)ix.i[0][r] : r) * d0 + cc];
    else if ((cc -= d0) < d1) v = s1[b * bs1 + (ix.i[1] ? (long long)ix.i[1][r] : r) * d1 + cc];
    else if ((cc -= d1) < d2) v = s2[b * bs2 + (ix.i[2] ? (long long)ix.i[2][r] : r) * d2 + cc];
    else if ((cc -= d2) < d3) v = s3[b * bs3 + (ix.i[3] ? (long long)ix.i[3][r] : r) * d3 + cc];
    out[i] = v;
  }
}

bool tc_mlp2_packed_supported(const NlamMlp* m, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res, const NlamRowSrc* res2) {
  if (m->n_linear != 2 || res2 || n_src < 1 || n_src > 4) return false;
  const int H = m->out_dim[0], no = m->out_dim[1];
  if (!(H == 64 || H == 128 || H == 256) || no < 1 || no > 256 || (m->ln_gamma && no != npad(no))) return false;
  if (res && (res->dim != no || no != npad(no) || res->bstride % 4 != 0 || !aligned16(res->ptr))) return false;
  int k = 0;
  for (int s = 0; s < n_src; ++s) k += srcs[s].dim;  // sources may gather (row index)
  return k == m->in_dim && k % 4 == 0 && k <= 1024 && aligned16(m->w[0]) && aligned16(m->w[1]);
}

size_t tc_mlp2_packed_workspace_floats(const NlamMlp* m, int64_t n_rows, int B) {
  const int kp = (m->in_dim + 31) / 32 * 32;
  return (size_t)n_rows * B * (kp + m->out_dim[0]);
}

int tc_mlp2_packed(const NlamMlp* m, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res, float* out, int64_t n_rows, int B,
                   cudaStream_t st, float* ws) {
  const int kp = (m->in_dim + 31) / 32 * 32, H = m->out_dim[0], no = m->out_dim[1];
  float* packed = ws;
  float* hid = ws + (size_t)n_rows * B * kp;
  const float* sp[4] = {nullptr, nullptr, nullptr, nullptr};
  int d[4] = {0, 0, 0, 0};
  long long bs[4] = {0, 0, 0, 0};
  PackIdx ix = {{nullptr, nullptr, nullptr, nullptr}};
  for (int s = 0; s < n_src; ++s) {
    sp[s] = srcs[s].ptr;
    d[s] = srcs[s].dim;
    bs[s] = B > 1 ? srcs[s].bstride : 0;
    ix.i[s] = srcs[s].idx;
  }
  const long long total = (long long)B * n_rows * kp;
  {
    ProfScope ps("pack_rows_kernel", st, 4.0 * total + 4.0 * (double)B * n_rows * m->in_dim);
    pack_rows_kernel<<<(int)std::min<long long>((total + 255) / 256, 132 * 16), 256, 0, st>>>(
        sp[0], sp[1], sp[2], sp[3], d[0], d[1], d[2], d[3], bs[0], bs[1], bs[2], bs[3], packed, kp, n_rows, B, ix);
  }
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  LinearCall c;
  memset(&c, 0, sizeof(c));
  c.x0 = packed; c.x0_bs = (int64_t)n_rows * kp; c.k0 = kp; c.w = m->w[0]; c.ldw = m->in_dim; c.w_cols = m->in_dim;
  c.bias = m->b[0]; c.n_out = H; c.act = 1; c.n_rows = n_rows; c.B = B; c.out = hid;
  int rc = tc_linear(c, st);
  if (rc) return rc;
  memset(&c, 0, sizeof(c));
  c.x0 = hid; c.x0_bs = (int64_t)n_rows * H; c.k0 = H; c.w = m->w[1]; c.ldw = H; c.bias = m->b[1]; c.n_out = no;
  c.gamma = m->ln_gamma; c.beta = m->ln_beta; c.eps = m->ln_eps; c.n_rows = n_rows; c.B = B; c.out = out;
  if (res && res->idx) {  // gathered residual (PropagationNet: + x_src)
    c.post = res->ptr;
    c.post_idx = res->idx;
    c.post_bs = B > 1 ? res->bstride : 0;
  } else if (res) {
    c.res = res->ptr;
    c.res_bs = B > 1 ? res->bstride : 0;
  }
  return tc_linear(c, st);
}

}  // namespace nlam
// zero-padded concatenation of up to four row blocks: out[b, r, :kp] = [s0 | s1 | s2 | s3 | 0...]
extern "C" int nlam_pack_rows(const float* s0, const float* s1, const float* s2, const float* s3, int d0, int d1, int d2, int d3,
                              int64_t bs0, int64_t bs1, int64_t bs2, int64_t bs3, float* out, int kp, int64_t n_rows, int B,
                              void* stream) {
  NLAM_REQUIRE(s0 && out && kp >= d0 + d1 + d2 + d3 && n_rows >= 0 && B >= 1, NLAM_E_INVALID, "nlam_pack_rows: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = (long long)B * n_rows * kp;
  if (total == 0) return NLAM_OK;
  {
    nlam::ProfScope ps("pack_rows_kernel", st, 8.0 * total);
    nlam::pack_rows_kernel<<<(int)std::min<long long>((total + 255) / 256, 132 * 16), 256, 0, st>>>(
        s0, s1, s2, s3, d0, d1, d2, d3, bs0, bs1, bs2, bs3, out, kp, n_rows, B, nlam::PackIdx{{nullptr, nullptr, nullptr, nullptr}});
  }
  nlam::count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}
namespace nlam {

// ---- InteractionNet / PropagationNet (reference gnn_layers.py:110-157, :231-249) from the generic Linear kernel ----
bool tc_inet_gen_supported(const NlamGraph* g, const NlamMlp* em, const NlamMlp* am, int flags, const float* send,
                           int64_t send_bs, const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs) {
  if (!g || em->n_linear != 2 || am->n_linear != 2 || !em->ln_gamma || !am->ln_gamma) return false;
  const int H = em->out_dim[1];
  const bool prop = flags & NLAM_PROPAGATION;
  if (!(H == 128 || H == 256 || (H == 64 && prop))) return false;
  if (em->out_dim[0] != H || am->out_dim[0] != H || am->out_dim[1] != H || em->in_dim != 3 * H || am->in_dim != 2 * H) return false;
  if (!(aligned16(send) && aligned16(rec) && aligned16(edge) && send_bs % 4 == 0 && rec_bs % 4 == 0 && edge_bs % 4 == 0))
    return false;
  for (int l = 0; l < 2; ++l)
    if (!aligned16(em->w[l]) || !aligned16(am->w[l])) return false;
  return true;
}

static size_t rup64(size_t n) { return (n + 63) / 64 * 64; }

size_t tc_inet_gen_workspace_floats(const NlamGraph* g, int B, int H) {
  // Ps | Pr | edge hidden | messages | node hidden
  return rup64((size_t)B * g->n_send * H) + rup64((size_t)B * g->n_rec * H) + 2 * rup64((size_t)B * g->n_edges * H) +
         rup64((size_t)B * g->n_rec * H);
}

int tc_inet_gen(const NlamGraph* g, const NlamMlp* em, const NlamMlp* am, const float* send, int64_t send_bs, const float* rec,
                int64_t rec_bs, const float* edge, int64_t edge_bs, float* rec_out, float* edge_out, float* aggr, int B, int flags,
                float* ws, cudaStream_t st) {
  const int H = em->out_dim[1];
  const bool prop = flags & NLAM_PROPAGATION;
  const int mean = (flags & (NLAM_AGGR_MEAN | NLAM_PROPAGATION)) ? 1 : 0;
  const int64_t ns = g->n_send, nr = g->n_rec, E = g->n_edges;
  const int Bs = (send_bs == 0 || B == 1) ? 1 : B, Br = (rec_bs == 0 || B == 1) ? 1 : B;
  float* Ps = ws;
  float* Pr = Ps + rup64((size_t)B * ns * H);
  float* hid = Pr + rup64((size_t)B * nr * H);
  float* msg = hid + rup64((size_t)B * E * H);
  float* nhid = msg + rup64((size_t)B * E * H);
  const float* w1 = em->w[0];  // (H, 3H): columns [e | sender | receiver]
  LinearCall c;
  // 1 / 2: node projections of the split first Linear
  memset(&c, 0, sizeof(c));
  c.x0 = send; c.x0_bs = send_bs; c.k0 = H; c.w = w1 + H; c.ldw = 3 * H; c.n_out = H; c.n_rows = ns; c.B = Bs; c.out = Ps;
  int rc = tc_linear(c, st);
  if (rc) return rc;
  memset(&c, 0, sizeof(c));
  c.x0 = rec; c.x0_bs = rec_bs; c.k0 = H; c.w = w1 + 2 * H; c.ldw = 3 * H; c.bias = em->b[0]; c.n_out = H; c.n_rows = nr; c.B = Br;
  c.out = Pr;
  rc = tc_linear(c, st);
  if (rc) return rc;
  // 3: edge layer 1: SiLU(W1e·e + Ps[src] + Pr[dst])
  memset(&c, 0, sizeof(c));
  c.x0 = edge; c.x0_bs = edge_bs; c.k0 = H; c.w = w1; c.ldw = 3 * H; c.n_out = H; c.act = 1; c.n_rows = E; c.B = B; c.out = hid;
  c.add[0] = Ps; c.add_idx[0] = g->src; c.add_bs[0] = Bs > 1 ? ns * H : 0;
  c.add[1] = Pr; c.add_idx[1] = g->dst; c.add_bs[1] = Br > 1 ? nr * H : 0;
  rc = tc_linear(c, st);
  if (rc) return rc;
  // 4: edge layer 2: m = LN(W2·h + b2) (+ x_j for PropagationNet); e' = e + m
  memset(&c, 0, sizeof(c));
  c.x0 = hid; c.x0_bs = E * H; c.k0 = H; c.w = em->w[1]; c.ldw = H; c.bias = em->b[1]; c.n_out = H; c.gamma = em->ln_gamma;
  c.beta = em->ln_beta; c.eps = em->ln_eps; c.n_rows = E; c.B = B;
  if (prop) { c.post = send; c.post_idx = g->src; c.post_bs = send_bs; }
  if (edge_out) { c.out = edge_out; c.out2 = msg; c.res = edge; c.res_bs = edge_bs; }
  else c.out = msg;
  rc = tc_linear(c, st);
  if (rc) return rc;
  // 5: CSR segmented sum (deterministic)
  rc = nlam_segment_sum(g->rowptr, nullptr, nr, msg, E * H, aggr, nr * H, B, H, mean, st);
  if (rc) return rc;
  // 6: node update
  NlamRowSrc srcs[2] = {{rec, nullptr, rec_bs, H, 0}, {aggr, nullptr, (int64_t)nr * H, H, 0}};
  NlamRowSrc res = prop ? srcs[1] : srcs[0];
  return tc_mlp2(am, srcs, 2, &res, rec_out, nr, B, st, nhid);
}

}  // namespace nlam

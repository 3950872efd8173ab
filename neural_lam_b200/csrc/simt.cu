// Generic exact-fp32 (FFMA) kernels: any width, any number of hidden layers.
//   rowmlp_simt      make_mlp network over rows with gathered/concatenated inputs
//                    (reference neural_lam/utils/networks.py:27-40; inputs as in
//                    gnn_layers.py:148, :172)
//   segment_sum      CSR-ordered deterministic sum/mean (PyG scatter aggregation reached
//                    from gnn_layers.py:188)
//   gather_rows      x.index_select(-2, idx) (PyG propagate, gnn_layers.py:145)
//   step_epilogue    rescale + residual + boundary mix (graph/base.py:339-342,
//                    forecasters/autoregressive.py:128-131)
// These are the "exact" path and the fallback for shapes the tensor-core kernels do not cover.
#include "common.cuh"

namespace nlam {

constexpr int NT = 256;   // threads per CTA
constexpr int RM = 4;     // rows per thread micro-tile
constexpr int MAXP = 8;   // (row-group, column) pairs per thread
constexpr int KC = 32;    // k-chunk staged through shared memory

struct RowMlpParams {
  int n_src;
  const float* src[NLAM_MAX_SRC];
  const int32_t* sidx[NLAM_MAX_SRC];
  long long sbs[NLAM_MAX_SRC];
  int sdim[NLAM_MAX_SRC];
  int n_linear;
  int in_dim;
  int out_dim[NLAM_MAX_LINEAR];
  const float* w[NLAM_MAX_LINEAR];
  const float* b[NLAM_MAX_LINEAR];
  const float* gamma;
  const float* beta;
  float eps;
  const float* res;
  const int32_t* ridx;
  long long rbs;
  const float* res2;
  long long r2bs;
  float* out;
  float* out2;
  long long n_rows;
  int B;
  int tile_r;
  int pitch_a;  // floats, multiple of 4
  int pitch_b;
  int wpitch;   // floats (odd)
  int tiles_per_batch;
};

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }

__global__ void __launch_bounds__(NT) rowmlp_simt_kernel(const RowMlpParams p) {
  extern __shared__ __align__(16) float smem[];
  float* actA = smem;
  float* actB = actA + (size_t)p.tile_r * p.pitch_a;
  float* Ws = actB + (size_t)p.tile_r * p.pitch_b;
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const long long n_work = (long long)p.tiles_per_batch * p.B;

  for (long long work = blockIdx.x; work < n_work; work += gridDim.x) {
    const int b = (int)(work / p.tiles_per_batch);
    const long long row0 = (work % p.tiles_per_batch) * (long long)p.tile_r;
    const int rows = (int)min((long long)p.tile_r, p.n_rows - row0);

    // ---- load concatenated (optionally gathered) inputs into actA, zero padded ----
    {
      int col0 = 0;
      for (int s = 0; s < p.n_src; ++s) {
        const int d = p.sdim[s];
        const float* base = p.src[s] + (long long)b * p.sbs[s];
        for (int i = tid; i < p.tile_r * d; i += NT) {
          int r = i / d, c = i - r * d;
          float v = 0.f;
          if (r < rows) {
            long long gr = row0 + r;
            if (p.sidx[s]) gr = p.sidx[s][gr];
            v = base[gr * d + c];
          }
          actA[r * p.pitch_a + col0 + c] = v;
        }
        col0 += d;
      }
      // zero the k padding (pitch_a is in_dim rounded up to KC multiple at most)
      const int padw = p.pitch_a - p.in_dim;
      for (int i = tid; i < p.tile_r * padw; i += NT) {
        int r = i / padw, c = i - r * padw;
        actA[r * p.pitch_a + p.in_dim + c] = 0.f;
      }
    }
    __syncthreads();

    float* in = actA;
    float* outb = actB;
    int pin = p.pitch_a, pout = p.pitch_b;
    int K = p.in_dim;
    for (int l = 0; l < p.n_linear; ++l) {
      const int N = p.out_dim[l];
      const float* __restrict__ W = p.w[l];
      const int n_pairs = (p.tile_r / RM) * N;
      float acc[MAXP][RM];
#pragma unroll
      for (int q = 0; q < MAXP; ++q)
#pragma unroll
        for (int i = 0; i < RM; ++i) acc[q][i] = 0.f;

      for (int k0 = 0; k0 < K; k0 += KC) {
        // stage W[:, k0:k0+KC] transposed: Ws[kc][j]
        for (int i = tid; i < N * KC; i += NT) {
          int kc = i & (KC - 1), j = i / KC;
          int k = k0 + kc;
          Ws[kc * p.wpitch + j] = (k < K) ? W[(long long)j * K + k] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < MAXP; ++q) {
          int pr = tid + q * NT;
          if (pr < n_pairs) {
            int rg = pr / N, j = pr - rg * N;
            const float* arow = in + (rg * RM) * pin + k0;
#pragma unroll
            for (int kc = 0; kc < KC; kc += 4) {
              float w0 = Ws[(kc + 0) * p.wpitch + j];
              float w1 = Ws[(kc + 1) * p.wpitch + j];
              float w2 = Ws[(kc + 2) * p.wpitch + j];
              float w3 = Ws[(kc + 3) * p.wpitch + j];
#pragma unroll
              for (int i = 0; i < RM; ++i) {
                float4 a = *reinterpret_cast<const float4*>(arow + i * pin + kc);
                acc[q][i] = fmaf(a.x, w0, acc[q][i]);
                acc[q][i] = fmaf(a.y, w1, acc[q][i]);
                acc[q][i] = fmaf(a.z, w2, acc[q][i]);
                acc[q][i] = fmaf(a.w, w3, acc[q][i]);
              }
            }
          }
        }
        __syncthreads();
      }
      // bias (+ SiLU on all but the last Linear), write to the other buffer
      const bool last = (l == p.n_linear - 1);
#pragma unroll
      for (int q = 0; q < MAXP; ++q) {
        int pr = tid + q * NT;
        if (pr < n_pairs) {
          int rg = pr / N, j = pr - rg * N;
          float bj = p.b[l][j];
#pragma unroll
          for (int i = 0; i < RM; ++i) {
            float v = acc[q][i] + bj;
            if (!last) v = silu_f(v);
            outb[(rg * RM + i) * pout + j] = v;
          }
        }
      }
      // zero k-padding of the new activation (next layer reads in KC chunks)
      {
        const int Kn = N;
        const int kpad = ((Kn + KC - 1) / KC) * KC - Kn;
        for (int i = tid; i < p.tile_r * kpad; i += NT) {
          int r = i / kpad, c = i - r * kpad;
          outb[r * pout + Kn + c] = 0.f;
        }
      }
      __syncthreads();
      // swap
      float* t = in; in = outb; outb = t;
      int tp = pin; pin = pout; pout = tp;
      K = N;
    }
    const int Nf = K;  // final width; result rows are in `in`

    // ---- LayerNorm (two-pass, biased variance, like torch.nn.LayerNorm) ----
    if (p.gamma) {
      for (int r = warp; r < rows; r += NT / 32) {
        float* y = in + r * pin;
        float s = 0.f;
        for (int c = lane; c < Nf; c += 32) s += y[c];
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        float mu = s / Nf;
        float v = 0.f;
        for (int c = lane; c < Nf; c += 32) { float d = y[c] - mu; v += d * d; }
#pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        float rstd = rsqrtf(v / Nf + p.eps);
        for (int c = lane; c < Nf; c += 32) y[c] = (y[c] - mu) * rstd * p.gamma[c] + p.beta[c];
      }
      __syncthreads();
    }

    // ---- epilogue: residual(s) + coalesced store ----
    for (int i = tid; i < rows * Nf; i += NT) {
      int r = i / Nf, c = i - r * Nf;
      long long gr = row0 + r;
      float v = in[r * pin + c];
      if (p.res) {
        long long rr = p.ridx ? (long long)p.ridx[gr] : gr;
        v += p.res[(long long)b * p.rbs + rr * Nf + c];
      }
      long long o = ((long long)b * p.n_rows + gr) * Nf + c;
      if (p.out) p.out[o] = v;
      if (p.out2) p.out2[o] = p.res2[(long long)b * p.r2bs + gr * Nf + c] + v;
    }
    __syncthreads();
  }
}

static int round_up(int x, int m) { return (x + m - 1) / m * m; }

int rowmlp_simt(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const NlamRowSrc* res,
                const NlamRowSrc* res2, float* out, float* out2, int64_t n_rows, int B,
                cudaStream_t stream) {
  NLAM_REQUIRE(mlp && srcs && n_src >= 1 && n_src <= NLAM_MAX_SRC, NLAM_E_INVALID, "rowmlp: bad sources");
  NLAM_REQUIRE(mlp->n_linear >= 1 && mlp->n_linear <= NLAM_MAX_LINEAR, NLAM_E_UNSUPPORTED,
               "rowmlp: %d linear layers unsupported (max %d)", mlp->n_linear, NLAM_MAX_LINEAR);
  NLAM_REQUIRE(n_rows >= 0 && B >= 1, NLAM_E_INVALID, "rowmlp: bad sizes");
  if (n_rows == 0) return NLAM_OK;
  RowMlpParams p;
  memset(&p, 0, sizeof(p));
  p.n_src = n_src;
  int in_dim = 0;
  for (int s = 0; s < n_src; ++s) {
    p.src[s] = srcs[s].ptr;
    p.sidx[s] = srcs[s].idx;
    p.sbs[s] = srcs[s].bstride;
    p.sdim[s] = srcs[s].dim;
    NLAM_REQUIRE(srcs[s].ptr && srcs[s].dim >= 1, NLAM_E_INVALID, "rowmlp: bad source %d", s);
    in_dim += srcs[s].dim;
  }
  NLAM_REQUIRE(in_dim == mlp->in_dim, NLAM_E_INVALID, "rowmlp: sources give width %d, MLP expects %d", in_dim, mlp->in_dim);
  p.n_linear = mlp->n_linear;
  p.in_dim = in_dim;
  int nmax = 0;
  for (int l = 0; l < mlp->n_linear; ++l) {
    p.out_dim[l] = mlp->out_dim[l];
    p.w[l] = mlp->w[l];
    p.b[l] = mlp->b[l];
    NLAM_REQUIRE(mlp->w[l] && mlp->b[l] && mlp->out_dim[l] >= 1, NLAM_E_INVALID, "rowmlp: bad layer %d", l);
    nmax = std::max(nmax, mlp->out_dim[l]);
  }
  const int nf = mlp->out_dim[mlp->n_linear - 1];
  p.gamma = mlp->ln_gamma;
  p.beta = mlp->ln_beta;
  p.eps = mlp->ln_eps;
  NLAM_REQUIRE((p.gamma == nullptr) == (p.beta == nullptr), NLAM_E_INVALID, "rowmlp: gamma/beta must both be set or null");
  if (res) {
    NLAM_REQUIRE(res->dim == nf, NLAM_E_INVALID, "rowmlp: residual width %d != output width %d", res->dim, nf);
    p.res = res->ptr; p.ridx = res->idx; p.rbs = res->bstride;
  }
  if (res2) {
    NLAM_REQUIRE(res2->dim == nf && res2->idx == nullptr && out2, NLAM_E_INVALID, "rowmlp: bad second residual");
    p.res2 = res2->ptr; p.r2bs = res2->bstride;
  }
  p.out = out; p.out2 = out2; p.n_rows = n_rows; p.B = B;
  // buffer A holds the input (width in_dim) and every odd layer's output; B the even ones
  int wa = round_up(in_dim, KC), wb = KC;
  for (int l = 0; l < mlp->n_linear; ++l) {
    int w = round_up(mlp->out_dim[l], KC);
    if (l % 2 == 0) wb = std::max(wb, w); else wa = std::max(wa, w);
  }
  p.pitch_a = wa; p.pitch_b = wb;
  p.wpitch = nmax | 1;
  int tile_r = std::min(64, (MAXP * NT * RM) / nmax);
  const size_t smem_budget = 160 * 1024;
  size_t ws_bytes = (size_t)KC * p.wpitch * sizeof(float);
  while (tile_r > RM && (size_t)tile_r * (wa + wb) * sizeof(float) + ws_bytes > smem_budget) tile_r /= 2;
  tile_r = std::max(RM, tile_r / RM * RM);
  NLAM_REQUIRE((tile_r / RM) * nmax <= MAXP * NT, NLAM_E_UNSUPPORTED, "rowmlp: layer width %d too large", nmax);
  p.tile_r = tile_r;
  size_t smem = (size_t)tile_r * (wa + wb) * sizeof(float) + ws_bytes;
  NLAM_REQUIRE(smem <= 220 * 1024, NLAM_E_UNSUPPORTED, "rowmlp: widths too large for shared memory (%zu B)", smem);
  p.tiles_per_batch = (int)((n_rows + tile_r - 1) / tile_r);
  long long n_work = (long long)p.tiles_per_batch * B;
  NLAM_CUDA_OK(cudaFuncSetAttribute(rowmlp_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int occ = std::max<int>(1, (int)((220 * 1024) / (smem + 1024)));
  int grid = (int)std::min<long long>(n_work, (long long)132 * std::min(occ, 4));
  {
    ProfScope ps("rowmlp_simt_kernel", stream, rowmlp_algorithmic_bytes(mlp, srcs, n_src, res, res2, n_rows, B, out2 != nullptr, nullptr));
    rowmlp_simt_kernel<<<grid, NT, smem, stream>>>(p);
  }
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

// ---------------------------------------------------------------------------------------
// segment sum: one thread per (segment, float4 column); CSR order, deterministic
// ---------------------------------------------------------------------------------------
template <int VEC>
__global__ void segment_sum_kernel(const int32_t* __restrict__ ptr, const int32_t* __restrict__ order,
                                   long long n_seg, const float* __restrict__ x, long long xbs,
                                   float* __restrict__ out, long long obs, int B, int H, int mean) {
  const int hv = H / VEC;
  const long long total = (long long)B * n_seg * hv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % hv);
    long long n = (i / hv) % n_seg;
    int b = (int)(i / (hv * n_seg));
    int k0 = ptr[n], k1 = ptr[n + 1];
    float acc[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = 0.f;
    const float* xb = x + (long long)b * xbs + (long long)c * VEC;
    for (int k = k0; k < k1; ++k) {
      long long row = order ? order[k] : k;
      if (VEC == 4) {
        float4 t = *reinterpret_cast<const float4*>(xb + row * H);
        acc[0] += t.x; acc[1] += t.y; acc[2] += t.z; acc[3] += t.w;
      } else {
        acc[0] += xb[row * H];
      }
    }
    if (mean) {
      float sc = 1.0f / (float)max(k1 - k0, 1);
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc[v] = acc[v] * sc;
    }
    float* o = out + (long long)b * obs + n * H + (long long)c * VEC;
    if (VEC == 4) *reinterpret_cast<float4*>(o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    else o[0] = acc[0];
  }
}

template <int VEC>
__global__ void gather_rows_kernel(const float* __restrict__ x, long long xbs, const int32_t* __restrict__ idx,
                                   long long n_rows, float* __restrict__ out, long long obs, int B, int H,
                                   const int32_t* __restrict__ deg_ptr) {
  const int hv = H / VEC;
  const long long total = (long long)B * n_rows * hv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int c = (int)(i % hv);
    long long r = (i / hv) % n_rows;
    int b = (int)(i / (hv * n_rows));
    long long srow = idx[r];
    float sc = 1.f;
    if (deg_ptr) sc = 1.0f / (float)max(deg_ptr[srow + 1] - deg_ptr[srow], 1);
    const float* xp = x + (long long)b * xbs + srow * H + (long long)c * VEC;
    float* op = out + (long long)b * obs + r * H + (long long)c * VEC;
    if (VEC == 4) {
      float4 t = *reinterpret_cast<const float4*>(xp);
      t.x *= sc; t.y *= sc; t.z *= sc; t.w *= sc;
      *reinterpret_cast<float4*>(op) = t;
    } else {
      op[0] = xp[0] * sc;
    }
  }
}

__global__ void step_epilogue_kernel(const float* __restrict__ net_out, const float* __restrict__ prev,
                                     const float* __restrict__ boundary, const float* __restrict__ bmask,
                                     const float* __restrict__ dstd, const float* __restrict__ dmean,
                                     float* __restrict__ new_state, long long B, long long G, long long D) {
  const long long total = B * G * D;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int d = (int)(i % D);
    long long gidx = (i / D) % G;
    float pred = prev[i] + (net_out[i] * dstd[d] + dmean[d]);
    if (boundary) {
      float m = bmask[gidx];
      pred = m * boundary[i] + (1.0f - m) * pred;
    }
    new_state[i] = pred;
  }
}

// Clamped state update (reference models/step_predictors/base.py:296-334, :366-396; utils/tensor.py:7-81): per state
// variable kind 0 = plain residual, 1 = scaled sigmoid between (lo, up), 2 = softplus above lo, 3 = mirrored softplus
// below up; X' = f(f^-1(X) + delta), sharpness 1, centre 0, softplus threshold 20 and the reference's clamps of the
// inverse functions.
__device__ __forceinline__ float softplus20(float x) { return x > 20.f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float inv_softplus(float y) {
  const float yc = fminf(fmaxf(y, 9.5367386e-07f), 20.f);  // float32(log(1 + 1e-6)), threshold 20
  return y <= 20.f ? logf(expm1f(yc)) : y;
}

__global__ void step_epilogue_clamped_kernel(const float* __restrict__ net_out, const float* __restrict__ prev,
                                             const float* __restrict__ boundary, const float* __restrict__ bmask,
                                             const float* __restrict__ dstd, const float* __restrict__ dmean,
                                             const int32_t* __restrict__ kind, const float* __restrict__ lo,
                                             const float* __restrict__ up, float* __restrict__ new_state, long long B,
                                             long long G, long long D) {
  const long long total = B * G * D;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(i % D);
    const long long gidx = (i / D) % G;
    const float x = prev[i];
    const float delta = net_out[i] * dstd[d] + dmean[d];
    float pred;
    const int k = kind[d];
    if (k == 1) {
      const float a = lo[d], w = up[d] - lo[d];
      const float xc = fminf(fmaxf((x - a) / w, 1e-6f), 1.f - 1e-6f);
      const float z = logf(xc / (1.f - xc)) + delta;
      pred = a + w * (1.f / (1.f + expf(-z)));
    } else if (k == 2) {
      pred = lo[d] + softplus20(inv_softplus(x - lo[d]) + delta);
    } else if (k == 3) {
      pred = up[d] - softplus20(inv_softplus(up[d] - x) - delta);
    } else {
      pred = x + delta;
    }
    if (boundary) {
      const float m = bmask[gidx];
      pred = m * boundary[i] + (1.0f - m) * pred;
    }
    new_state[i] = pred;
  }
}

static int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  return (int)std::max<long long>(1, std::min<long long>(g, 132LL * 16));
}

}  // namespace nlam

using namespace nlam;

extern "C" int nlam_segment_sum(const int32_t* ptr, const int32_t* order, int64_t n_seg, const float* x,
                                int64_t x_bstride, float* out, int64_t out_bstride, int B, int H, int mean,
                                void* stream) {
  NLAM_REQUIRE(ptr && x && out && n_seg >= 0 && B >= 1 && H >= 1, NLAM_E_INVALID, "segment_sum: bad arguments");
  if (n_seg == 0) return NLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  bool vec = (H % 4 == 0) && (x_bstride % 4 == 0) && (out_bstride % 4 == 0) &&
             ((uintptr_t)x % 16 == 0) && ((uintptr_t)out % 16 == 0);
  ProfScope ps("segment_sum_kernel", st, 4.0 * H * B * (double)n_seg * 2 + 4.0 * n_seg);  // + the rows it reads (unknown here)
  if (vec) {
    long long total = (long long)B * n_seg * (H / 4);
    segment_sum_kernel<4><<<grid_for(total, 256), 256, 0, st>>>(ptr, order, n_seg, x, x_bstride, out, out_bstride, B, H, mean);
  } else {
    long long total = (long long)B * n_seg * H;
    segment_sum_kernel<1><<<grid_for(total, 256), 256, 0, st>>>(ptr, order, n_seg, x, x_bstride, out, out_bstride, B, H, mean);
  }
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

extern "C" int nlam_gather_rows(const float* x, int64_t x_bstride, const int32_t* idx, int64_t n_rows,
                                float* out, int64_t out_bstride, int B, int H, const int32_t* deg_ptr,
                                void* stream) {
  NLAM_REQUIRE(x && idx && out && n_rows >= 0 && B >= 1 && H >= 1, NLAM_E_INVALID, "gather_rows: bad arguments");
  if (n_rows == 0) return NLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  bool vec = (H % 4 == 0) && (x_bstride % 4 == 0) && (out_bstride % 4 == 0) &&
             ((uintptr_t)x % 16 == 0) && ((uintptr_t)out % 16 == 0);
  ProfScope ps("gather_rows_kernel", st, 4.0 * H * B * (double)n_rows * 2 + 4.0 * n_rows);
  if (vec) {
    long long total = (long long)B * n_rows * (H / 4);
    gather_rows_kernel<4><<<grid_for(total, 256), 256, 0, st>>>(x, x_bstride, idx, n_rows, out, out_bstride, B, H, deg_ptr);
  } else {
    long long total = (long long)B * n_rows * H;
    gather_rows_kernel<1><<<grid_for(total, 256), 256, 0, st>>>(x, x_bstride, idx, n_rows, out, out_bstride, B, H, deg_ptr);
  }
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

extern "C" int nlam_step_epilogue(const float* net_out, const float* prev, const float* boundary,
                                  const float* bmask, const float* diff_std, const float* diff_mean,
                                  float* new_state, int64_t B, int64_t G, int64_t D, void* stream) {
  NLAM_REQUIRE(net_out && prev && diff_std && diff_mean && new_state, NLAM_E_INVALID, "step_epilogue: null argument");
  NLAM_REQUIRE((boundary == nullptr) || bmask, NLAM_E_INVALID, "step_epilogue: boundary without mask");
  long long total = B * G * D;
  if (total == 0) return NLAM_OK;
  {
    ProfScope ps("step_epilogue_kernel", (cudaStream_t)stream, 4.0 * total * (boundary ? 4 : 3));
    step_epilogue_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(net_out, prev, boundary, bmask, diff_std,
                                                                                 diff_mean, new_state, B, G, D);
  }
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

extern "C" int nlam_step_epilogue_clamped(const float* net_out, const float* prev, const float* boundary, const float* bmask,
                                          const float* diff_std, const float* diff_mean, const int32_t* clamp_kind,
                                          const float* clamp_lo, const float* clamp_up, float* new_state, int64_t B, int64_t G,
                                          int64_t D, void* stream) {
  NLAM_REQUIRE(net_out && prev && diff_std && diff_mean && new_state && clamp_kind && clamp_lo && clamp_up, NLAM_E_INVALID,
               "step_epilogue_clamped: null argument");
  NLAM_REQUIRE((boundary == nullptr) || bmask, NLAM_E_INVALID, "step_epilogue_clamped: boundary without mask");
  long long total = B * G * D;
  if (total == 0) return NLAM_OK;
  {
    ProfScope ps("step_epilogue_clamped_kernel", (cudaStream_t)stream, 4.0 * total * (boundary ? 4 : 3));
    step_epilogue_clamped_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
        net_out, prev, boundary, bmask, diff_std, diff_mean, clamp_kind, clamp_lo, clamp_up, new_state, B, G, D);
  }
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

// ---------------------------------------------------------------------------------------------------
// Halo push (node-partitioned rollout, SURVEY 8e): ONE launch copies this rank's OWN sender rows into the front of
// its extended buffer [own rows | halo rows] and stores the boundary rows its peers need DIRECTLY into their halo
// regions — `peer_ext[p]` are the peers' extended buffers mapped into this process (CUDA IPC / symmetric memory), so
// the stores travel over NVLink / NVSwitch from this kernel; no pack buffer, no NCCL send/recv, no concatenation.
// The consumer side only needs a cross-rank barrier before it reads its extended buffer.
__global__ void halo_push_kernel(const float* __restrict__ own, long long own_bs, long long n_own, float* ext_local,
                                 long long ext_bs, float* const* __restrict__ peer_ext, const int32_t* __restrict__ send_rows,
                                 const int32_t* __restrict__ send_ptr, const int32_t* __restrict__ peer_dst_off, int world,
                                 int B, int H4) {
  const long long n_send = send_ptr[world];
  const long long per_b = (n_own + n_send) * H4;
  const long long total = (long long)B * per_b;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / per_b);
    const long long j = i - (long long)b * per_b;
    const long long r = j / H4;
    const int c = (int)(j - r * H4);
    if (r < n_own) {
      reinterpret_cast<float4*>(ext_local + b * ext_bs)[r * H4 + c] = reinterpret_cast<const float4*>(own + b * own_bs)[r * H4 + c];
    } else {
      const long long k = r - n_own;  // index into the concatenated send lists
      int p = 0;
      while (k >= send_ptr[p + 1]) ++p;  // world <= 8
      const long long dst_row = peer_dst_off[p] + (k - send_ptr[p]);
      reinterpret_cast<float4*>(peer_ext[p] + b * ext_bs)[dst_row * H4 + c] =
          reinterpret_cast<const float4*>(own + b * own_bs)[(long long)send_rows[k] * H4 + c];
    }
  }
}

extern "C" int nlam_halo_push(const float* own, int64_t own_bs, int64_t n_own, float* ext_local, int64_t ext_bs,
                              float* const* peer_ext, const int32_t* send_rows, const int32_t* send_ptr,
                              const int32_t* peer_dst_off, int64_t n_send_total, int world, int B, int H, void* stream) {
  NLAM_REQUIRE(own && ext_local && peer_ext && send_ptr && peer_dst_off && world >= 1 && B >= 1 && H >= 4 && H % 4 == 0,
               NLAM_E_INVALID, "halo_push: bad arguments");
  NLAM_REQUIRE(own_bs % 4 == 0 && ext_bs % 4 == 0 && ((uintptr_t)own % 16 == 0) && ((uintptr_t)ext_local % 16 == 0),
               NLAM_E_INVALID, "halo_push: rows must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = (long long)B * (n_own + n_send_total) * (H / 4);
  if (total == 0) return NLAM_OK;
  {
    ProfScope ps("halo_push_kernel", st, 8.0 * total * 4);
    halo_push_kernel<<<grid_for(total, 256), 256, 0, st>>>(own, own_bs, n_own, ext_local, ext_bs, peer_ext, send_rows, send_ptr,
                                                           peer_dst_off, world, B, H / 4);
  }
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

// One strided host<->device copy per tensor and forecast step (ARForecaster.rollout_from_host): the step-i slice of a
// (B, T, G, F) host tensor is B rows of G*F floats with pitch T*G*F — one cudaMemcpy2DAsync instead of B small copies.
// depth x height rows of width_bytes; row pitch and rows-per-slice (slice stride = pitch * rows) on either side: the
// boundary frame of a forecast step (the strips left and right of the interior: runs of nodes one grid row apart,
// for every sample) in ONE cudaMemcpy3DAsync
extern "C" int nlam_memcpy3d_async(void* dst, size_t dpitch, size_t drows, const void* src, size_t spitch, size_t srows,
                                   size_t width_bytes, size_t height, size_t depth, int host_to_device, void* stream) {
  NLAM_REQUIRE(dst && src && height <= drows && height <= srows && width_bytes <= dpitch && width_bytes <= spitch,
               NLAM_E_INVALID, "memcpy3d: bad arguments");
  cudaMemcpy3DParms q;
  memset(&q, 0, sizeof(q));
  q.srcPtr = make_cudaPitchedPtr(const_cast<void*>(src), spitch, spitch, srows);
  q.dstPtr = make_cudaPitchedPtr(dst, dpitch, dpitch, drows);
  q.extent = make_cudaExtent(width_bytes, height, depth);
  q.kind = host_to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost;
  NLAM_CUDA_OK(cudaMemcpy3DAsync(&q, (cudaStream_t)stream));
  return NLAM_OK;
}

extern "C" int nlam_memcpy2d_async(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width_bytes,
                                   size_t height, int host_to_device, void* stream) {
  NLAM_REQUIRE(dst && src, NLAM_E_INVALID, "memcpy2d: null pointer");
  NLAM_CUDA_OK(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width_bytes, height,
                                 host_to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return NLAM_OK;
}

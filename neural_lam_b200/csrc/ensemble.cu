// Ensemble statistics of K forecast members (DESIGN §4.5): per point (b, g, v), with x_1 .. x_K the members and y the
// target,
//   m   = (1/K) Σ_k x_k                                 ensemble mean
//   s²  = (1/(K-1)) Σ_k (x_k - m)²                      unbiased variance (torch.var)
//   SE  = (m - y)²                                      squared error of the mean
//   A   = (1/K) Σ_k |x_k - y|                           mean absolute error term of the CRPS
//   D   = (1/(K(K-1))) Σ_{k≠l} |x_k - x_l|              mean pair difference, summed over the pairs directly
// m and s = sqrt(s²) are stored per point; SE, s², A and D are averaged per (b, v) over the interior grid nodes.
//
// ens_stats_kernel: one point per thread (K values G·d floats apart: each load coalesces across the warp), the K values
// held in registers (compile-time indices: the loops are unrolled to the bucket KMAX and leave at K), exact fp32.  Each
// CTA writes its per-variable interior partial sums (SE, s², A, D and the interior count) summed in point order;
// ens_reduce_kernel then sums the partials of one (b, v, quantity) in a fixed order.  No atomics: the results are
// bit-reproducible run to run, and initial condition b's results do not depend on the other rows of the batch.
#include "common.cuh"

namespace nlam {

constexpr int kEnsThreads = 256;
constexpr int kEnsQ = 5;  // SE, s², A, D, interior count

template <int KMAX>
__global__ void __launch_bounds__(kEnsThreads) ens_stats_kernel(const float* __restrict__ x, long long x_bs, long long x_ks, int K,
                                                                const float* __restrict__ y, long long y_bs,
                                                                const float* __restrict__ interior, long long n_pts, int d,
                                                                float* __restrict__ mean, float* __restrict__ std,
                                                                float* __restrict__ part, int n_cta) {
  __shared__ float red[kEnsQ][kEnsThreads];
  const int b = blockIdx.y;
  const long long p0 = (long long)blockIdx.x * kEnsThreads;
  const long long p = p0 + threadIdx.x;
  const bool live = p < n_pts;
  float v[KMAX];
  const float* xp = x + b * x_bs + (live ? p : 0);
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    if (k >= K) break;
    v[k] = live ? __ldg(xp + k * x_ks) : 0.f;
  }
  // two passes on the values shifted by the first member: identical members give m = x and s² = 0 exactly
  const float c = v[0];
  float su = 0.f;
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    if (k >= K) break;
    su += v[k] - c;
  }
  const float mu = su / (float)K;
  const float m = c + mu;
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    if (k >= K) break;
    const float e = (v[k] - c) - mu;
    ss = fmaf(e, e, ss);
  }
  const float var = ss / (float)(K - 1);
  if (live) {
    mean[b * n_pts + p] = m;
    std[b * n_pts + p] = sqrtf(var);
  }
  if (part == nullptr) return;

  // interior scores of this point (zero for boundary nodes and for the threads past the end)
  const bool in = live && interior[p / d] != 0.f;
  float se = 0.f, a = 0.f, dd = 0.f;
  if (in) {
    const float t = y[b * y_bs + p];
    se = (m - t) * (m - t);
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
      if (k >= K) break;
      a += fabsf(v[k] - t);
    }
    a = a / (float)K;
    // Σ_{k<l} |x_k - x_l| in four interleaved accumulators (pair l's terms go to accumulator l % 4), combined in a fixed
    // order; Σ_{k≠l} is twice that
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int l = 1; l < KMAX; ++l) {
      if (l >= K) break;
#pragma unroll
      for (int k = 0; k < l; ++k) acc[l & 3] += fabsf(v[k] - v[l]);
    }
    dd = 2.f * ((acc[0] + acc[1]) + (acc[2] + acc[3])) / ((float)K * (float)(K - 1));
  }
  red[0][threadIdx.x] = se;
  red[1][threadIdx.x] = in ? var : 0.f;
  red[2][threadIdx.x] = a;
  red[3][threadIdx.x] = dd;
  red[4][threadIdx.x] = in ? 1.f : 0.f;
  __syncthreads();
  // per (quantity, variable): the CTA's points of variable v in increasing point order
  const int v0 = (int)(p0 % d);
  const int n_here = n_pts - p0 < kEnsThreads ? (int)(n_pts - p0) : kEnsThreads;
  for (int j = threadIdx.x; j < kEnsQ * d; j += kEnsThreads) {
    const int q = j / d, var_i = j - q * d;
    int first = var_i - v0;
    if (first < 0) first += d;
    float s = 0.f;
    for (int i = first; i < n_here; i += d) s += red[q][i];
    part[(((long long)b * kEnsQ + q) * d + var_i) * n_cta + blockIdx.x] = s;
  }
}

// out[b, v, q] = Σ_cta part[b, q, v, cta] / Σ_cta count[b, v, cta] for q < 4: one CTA per (b, v, q), each thread sums a
// strided slice of the partials in order, then a fixed-shape tree over the threads
__global__ void __launch_bounds__(kEnsThreads) ens_reduce_kernel(const float* __restrict__ part, int n_cta, int d,
                                                                 float* __restrict__ out) {
  __shared__ float sv[kEnsThreads];
  __shared__ int sc[kEnsThreads];
  const int q = blockIdx.x % 4, var_i = (blockIdx.x / 4) % d, b = blockIdx.x / (4 * d);
  const float* pv = part + (((long long)b * kEnsQ + q) * d + var_i) * n_cta;
  const float* pc = part + (((long long)b * kEnsQ + 4) * d + var_i) * n_cta;
  float s = 0.f;
  int c = 0;
  for (int i = threadIdx.x; i < n_cta; i += kEnsThreads) {
    s += pv[i];
    c += (int)pc[i];
  }
  sv[threadIdx.x] = s;
  sc[threadIdx.x] = c;
  __syncthreads();
  for (int w = kEnsThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      sv[threadIdx.x] += sv[threadIdx.x + w];
      sc[threadIdx.x] += sc[threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[((long long)b * d + var_i) * 4 + q] = sv[0] / (float)sc[0];
}

static long long ens_ctas(long long n_pts) { return (n_pts + kEnsThreads - 1) / kEnsThreads; }

size_t ens_stats_workspace_bytes(int B, int64_t G, int d) {
  return (size_t)B * kEnsQ * d * ens_ctas(G * d) * sizeof(float);
}

int ens_stats(const float* x, int64_t x_bs, int64_t x_ks, int B, int K, int64_t G, int d, const float* y, int64_t y_bs,
              const float* interior, float* mean, float* std, float* scores, void* ws, size_t ws_bytes, cudaStream_t st) {
  NLAM_REQUIRE(K >= 2 && K <= 64, NLAM_E_UNSUPPORTED, "nlam_ensemble_stats: K = %d members outside 2 .. 64", K);
  const long long n_pts = (long long)G * d, n_cta = ens_ctas(n_pts);
  NLAM_REQUIRE(n_cta <= 0x7fffffff && B <= 65535, NLAM_E_UNSUPPORTED, "nlam_ensemble_stats: G = %lld, d = %d, B = %d too large",
               (long long)G, d, B);
  float* part = nullptr;
  if (scores) {
    NLAM_REQUIRE(ws && ws_bytes >= ens_stats_workspace_bytes(B, G, d), NLAM_E_WORKSPACE,
                 "nlam_ensemble_stats: workspace of %zu bytes, %zu needed", ws_bytes, ens_stats_workspace_bytes(B, G, d));
    part = (float*)ws;
  }
  const dim3 grid((unsigned)n_cta, (unsigned)B);
  {
    // algorithmic bytes: the K members and the target read once, m and s written once
    const double bytes = 4.0 * B * n_pts * (K + (scores ? 1 : 0) + 2);
    ProfScope ps("ens_stats_kernel", st, bytes);
#define NLAM_ENS_LAUNCH(KM) \
  ens_stats_kernel<KM><<<grid, kEnsThreads, 0, st>>>(x, x_bs, x_ks, K, y, y_bs, interior, n_pts, d, mean, std, part, (int)n_cta)
    if (K <= 4) NLAM_ENS_LAUNCH(4);
    else if (K <= 8) NLAM_ENS_LAUNCH(8);
    else if (K <= 16) NLAM_ENS_LAUNCH(16);
    else if (K <= 32) NLAM_ENS_LAUNCH(32);
    else NLAM_ENS_LAUNCH(64);
#undef NLAM_ENS_LAUNCH
  }
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  if (scores) {
    {
      ProfScope ps("ens_reduce_kernel", st, 4.0 * B * kEnsQ * d * n_cta + 16.0 * B * d);
      ens_reduce_kernel<<<B * d * 4, kEnsThreads, 0, st>>>(part, (int)n_cta, d, scores);
    }
    count_launch();
    NLAM_CUDA_OK(cudaGetLastError());
  }
  return NLAM_OK;
}

}  // namespace nlam

// Building blocks of the hand-written BACKWARD of the path (reference: autograd through gnn_layers.py:110-157 and
// utils/networks.py:27-40; tests/test_gnn_layers.py section F).  The dense products of the backward —
//   dX = dY · W          (Linear with the transposed weight)
//   dW = dYᵀ · X         (reduction over the rows: split-K partial products on the tensor cores + a deterministic
//                         reduction of the partials)
// run on the generic wgmma Linear kernel (tc7.cu); this file holds the elementwise / reduction / layout kernels
// around them: SiLU forward / backward, LayerNorm forward / backward (with the dγ / dβ column reductions), column
// sums (bias gradients), zero-padded transposes (the K-major operands of the dW products), the reduction of partial
// products, and the gather-add that assembles the message gradient g_m[e] = g_e'[e] + g_aggr[dst(e)] / deg.
// All reductions are two-stage and ordered: results are bit-reproducible run to run (no floating-point atomics).
#include "common.cuh"

namespace nlam {

static int grid_1d(long long total, int block, int cap = 132 * 8) {
  long long g = (total + block - 1) / block;
  return (int)std::max<long long>(1, std::min<long long>(g, cap));
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }

__global__ void silu_fwd_kernel(const float* __restrict__ z, float* __restrict__ h, long long n4) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = reinterpret_cast<const float4*>(z)[i];
    v.x *= sigmoidf_(v.x);
    v.y *= sigmoidf_(v.y);
    v.z *= sigmoidf_(v.z);
    v.w *= sigmoidf_(v.w);
    reinterpret_cast<float4*>(h)[i] = v;
  }
}

__device__ __forceinline__ float dsilu(float z) {
  const float s = sigmoidf_(z);
  return s * (1.0f + z * (1.0f - s));
}

__global__ void silu_bwd_kernel(const float* __restrict__ gh, const float* __restrict__ z, float* __restrict__ gz, long long n4) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 g = reinterpret_cast<const float4*>(gh)[i];
    const float4 v = reinterpret_cast<const float4*>(z)[i];
    reinterpret_cast<float4*>(gz)[i] = make_float4(g.x * dsilu(v.x), g.y * dsilu(v.y), g.z * dsilu(v.z), g.w * dsilu(v.w));
  }
}

// one warp per row; H <= 256 (8 values per lane)
template <int VPL>
__device__ __forceinline__ void row_stats(const float (&v)[VPL], int H, float eps, float& mu, float& rstd) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) s += v[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  mu = s / H;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const float d = v[i] - mu;
    q += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  rstd = rsqrtf(q / H + eps);
}

template <int VPL>
__global__ void ln_fwd_kernel(const float* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ beta,
                              float eps, float* __restrict__ out, long long rows) {
  constexpr int H = VPL * 32;
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < rows; r += n_warps) {
    float v[VPL];
#pragma unroll
    for (int i = 0; i < VPL; ++i) v[i] = y[r * H + lane + 32 * i];
    float mu, rstd;
    row_stats<VPL>(v, H, eps, mu, rstd);
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int c = lane + 32 * i;
      out[r * H + c] = (v[i] - mu) * rstd * gamma[c] + beta[c];
    }
  }
}

// g_y = rstd * (γ g − mean(γ g) − x̂ · mean(γ g x̂)); per-warp partial dγ = Σ g x̂, dβ = Σ g  ->  part[warp][2H]
template <int VPL>
__global__ void ln_bwd_kernel(const float* __restrict__ g, const float* __restrict__ y, const float* __restrict__ gamma,
                              float eps, float* __restrict__ gy, float* __restrict__ part, long long rows) {
  constexpr int H = VPL * 32;
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  float dg[VPL], db[VPL], gm[VPL];
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    dg[i] = 0.f;
    db[i] = 0.f;
    gm[i] = gamma[lane + 32 * i];
  }
  for (long long r = warp; r < rows; r += n_warps) {
    float v[VPL], gg[VPL];
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      v[i] = y[r * H + lane + 32 * i];
      gg[i] = g[r * H + lane + 32 * i];
    }
    float mu, rstd;
    row_stats<VPL>(v, H, eps, mu, rstd);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const float xh = (v[i] - mu) * rstd;
      const float gx = gg[i] * gm[i];
      s1 += gx;
      s2 += gx * xh;
      dg[i] += gg[i] * xh;
      db[i] += gg[i];
      v[i] = xh;
      gg[i] = gx;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    s1 /= H;
    s2 /= H;
#pragma unroll
    for (int i = 0; i < VPL; ++i) gy[r * H + lane + 32 * i] = rstd * (gg[i] - s1 - v[i] * s2);
  }
  if (warp < n_warps) {
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      part[warp * 2 * H + lane + 32 * i] = dg[i];
      part[warp * 2 * H + H + lane + 32 * i] = db[i];
    }
  }
}

// per-warp column sums of g (rows x C, C <= 1024): part[warp][C]
__global__ void colsum_kernel(const float* __restrict__ g, long long rows, int C, float* __restrict__ part) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (int c0 = 0; c0 < C; c0 += 32) {
    const int c = c0 + lane;
    float s = 0.f;
    if (c < C)
      for (long long r = warp; r < rows; r += n_warps) s += g[r * C + c];
    if (c < C) part[warp * C + c] = s;
  }
}

// out[r][c] (+)= Σ_p part[p][r][c]   (ordered: deterministic)
__global__ void reduce_partials_kernel(const float* __restrict__ part, int P, long long R, int C, float* __restrict__ out,
                                       long long out_pitch, int accumulate) {
  const long long total = R * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C;
    const int c = (int)(i - r * C);
    float s = 0.f;
    for (int p = 0; p < P; ++p) s += part[(long long)p * total + i];
    float* o = out + r * out_pitch + c;
    *o = accumulate ? *o + s : s;
  }
}

// same sum for FEW outputs and MANY partials (column reductions: thousands of per-warp partial rows, <= 2H columns):
// block = 32 output elements x 8 slices of the partial range, fixed-order combine through shared memory
__global__ void reduce_partials_tall_kernel(const float* __restrict__ part, int P, long long total, int C, float* __restrict__ out,
                                            long long out_pitch, int accumulate) {
  __shared__ float sm[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const long long i = (long long)blockIdx.x * 32 + tx;
  float s = 0.f;
  if (i < total)
    for (int p = ty; p < P; p += 8) s += part[(long long)p * total + i];
  sm[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && i < total) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += sm[k][tx];
    const long long r = i / C;
    float* o = out + r * out_pitch + (i - r * C);
    *o = accumulate ? *o + t : t;
  }
}

static void launch_reduce_partials(const float* part, int P, long long R, int C, float* out, long long out_pitch, int accumulate,
                                   cudaStream_t st) {
  const long long total = R * C;
  if (total <= 8192 && P >= 32)
    reduce_partials_tall_kernel<<<(int)((total + 31) / 32), 256, 0, st>>>(part, P, total, C, out, out_pitch, accumulate);
  else
    reduce_partials_kernel<<<grid_1d(total, 256), 256, 0, st>>>(part, P, R, C, out, out_pitch, accumulate);
}

// XT[c][r] = X[r][c] for r < rows, 0 for rows <= r < rows_pad   (32 x 32 tiles through shared memory)
__global__ void transpose_pad_kernel(const float* __restrict__ x, long long rows, int C, long long x_pitch, float* __restrict__ xt,
                                     long long rows_pad) {
  __shared__ float tile[32][33];
  const long long tiles_r = (rows_pad + 31) / 32;
  const int tiles_c = (C + 31) / 32;
  for (long long t = blockIdx.x; t < tiles_r * tiles_c; t += gridDim.x) {
    const long long tr = t / tiles_c;
    const int tc = (int)(t - tr * tiles_c);
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8 threads
    for (int j = ty; j < 32; j += 8) {
      const long long r = tr * 32 + j;
      const int c = tc * 32 + tx;
      tile[j][tx] = (r < rows && c < C) ? x[r * x_pitch + c] : 0.f;
    }
    __syncthreads();
    for (int j = ty; j < 32; j += 8) {
      const int c = tc * 32 + j;
      const long long r = tr * 32 + tx;
      if (c < C && r < rows_pad) xt[(long long)c * rows_pad + r] = tile[tx][j];
    }
    __syncthreads();
  }
}

// out[b, e, :] = (a ? a[b, e, :] : 0) + scale_e * v[b, idx[e], :],  scale_e = 1 or 1 / max(deg(idx[e]), 1)
__global__ void add_gather_kernel(const float* __restrict__ a, const float* __restrict__ v, const int32_t* __restrict__ idx,
                                  const int32_t* __restrict__ deg_ptr, long long n_e, long long n_v, int H4, int B,
                                  float* __restrict__ out) {
  const long long total = (long long)B * n_e * H4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % H4);
    const long long e = (i / H4) % n_e;
    const long long b = i / ((long long)H4 * n_e);
    const int j = idx[e];
    float sc = 1.f;
    if (deg_ptr) sc = 1.0f / (float)max(deg_ptr[j + 1] - deg_ptr[j], 1);
    float4 x = reinterpret_cast<const float4*>(v)[(b * n_v + j) * H4 + c];
    x.x *= sc; x.y *= sc; x.z *= sc; x.w *= sc;
    if (a) {
      const float4 y = reinterpret_cast<const float4*>(a)[i];
      x.x += y.x; x.y += y.y; x.z += y.z; x.w += y.w;
    }
    reinterpret_cast<float4*>(out)[i] = x;
  }
}

}  // namespace nlam

using namespace nlam;

extern "C" int nlam_silu(const float* z, const float* gh, float* out, int64_t n, void* stream) {
  NLAM_REQUIRE(z && out && n % 4 == 0, NLAM_E_INVALID, "nlam_silu: bad arguments");
  if (n == 0) return NLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope ps(gh ? "silu_bwd_kernel" : "silu_fwd_kernel", st, 4.0 * n * (gh ? 3 : 2));
  if (gh) silu_bwd_kernel<<<grid_1d(n / 4, 256), 256, 0, st>>>(gh, z, out, n / 4);
  else silu_fwd_kernel<<<grid_1d(n / 4, 256), 256, 0, st>>>(z, out, n / 4);
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

extern "C" int nlam_layernorm_fwd(const float* y, const float* gamma, const float* beta, float eps, float* out, int64_t rows,
                                  int H, void* stream) {
  NLAM_REQUIRE(y && gamma && beta && out && (H == 32 || H == 64 || H == 128 || H == 256), NLAM_E_UNSUPPORTED,
               "nlam_layernorm_fwd: width %d unsupported", H);
  if (rows == 0) return NLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_1d(rows * 32, 256);
  ProfScope ps("ln_fwd_kernel", st, 8.0 * rows * H);
  if (H == 32) ln_fwd_kernel<1><<<grid, 256, 0, st>>>(y, gamma, beta, eps, out, rows);
  else if (H == 64) ln_fwd_kernel<2><<<grid, 256, 0, st>>>(y, gamma, beta, eps, out, rows);
  else if (H == 128) ln_fwd_kernel<4><<<grid, 256, 0, st>>>(y, gamma, beta, eps, out, rows);
  else ln_fwd_kernel<8><<<grid, 256, 0, st>>>(y, gamma, beta, eps, out, rows);
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

extern "C" size_t nlam_bwd_scratch_floats(int C) { return (size_t)(132 * 8 * 8 + 2) * 2 * (size_t)C; }

extern "C" int nlam_layernorm_bwd(const float* g, const float* y, const float* gamma, float eps, float* gy, float* dgamma,
                                  float* dbeta, int64_t rows, int H, float* scratch, void* stream) {
  NLAM_REQUIRE(g && y && gamma && gy && dgamma && dbeta && scratch && (H == 32 || H == 64 || H == 128 || H == 256),
               NLAM_E_UNSUPPORTED, "nlam_layernorm_bwd: width %d unsupported", H);
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_1d(std::max<int64_t>(rows, 1) * 32, 256);
  const int n_warps = grid * 8;
  {
    ProfScope ps("ln_bwd_kernel", st, 12.0 * rows * H);
    if (H == 32) ln_bwd_kernel<1><<<grid, 256, 0, st>>>(g, y, gamma, eps, gy, scratch, rows);
    else if (H == 64) ln_bwd_kernel<2><<<grid, 256, 0, st>>>(g, y, gamma, eps, gy, scratch, rows);
    else if (H == 128) ln_bwd_kernel<4><<<grid, 256, 0, st>>>(g, y, gamma, eps, gy, scratch, rows);
    else ln_bwd_kernel<8><<<grid, 256, 0, st>>>(g, y, gamma, eps, gy, scratch, rows);
  }
  count_launch();
  // partials (n_warps, 2H): columns [0,H) -> dgamma, [H,2H) -> dbeta
  launch_reduce_partials(scratch, n_warps, 1, 2 * H, scratch + (size_t)n_warps * 2 * H, 2 * H, 0, st);
  count_launch();
  NLAM_CUDA_OK(cudaMemcpyAsync(dgamma, scratch + (size_t)n_warps * 2 * H, H * sizeof(float), cudaMemcpyDeviceToDevice, st));
  NLAM_CUDA_OK(cudaMemcpyAsync(dbeta, scratch + (size_t)n_warps * 2 * H + H, H * sizeof(float), cudaMemcpyDeviceToDevice, st));
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

extern "C" int nlam_colsum(const float* g, int64_t rows, int C, float* out, float* scratch, void* stream) {
  NLAM_REQUIRE(g && out && scratch && C >= 1 && C <= 1024, NLAM_E_INVALID, "nlam_colsum: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_1d(std::max<int64_t>(rows, 1) * 32, 256, 132 * 4);
  const int n_warps = grid * 8;
  {
    ProfScope ps("colsum_kernel", st, 4.0 * rows * C);
    colsum_kernel<<<grid, 256, 0, st>>>(g, rows, C, scratch);
  }
  count_launch();
  launch_reduce_partials(scratch, n_warps, 1, C, out, C, 0, st);
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

extern "C" int nlam_reduce_partials(const float* part, int P, int64_t R, int C, float* out, int64_t out_pitch, int accumulate,
                                    void* stream) {
  NLAM_REQUIRE(part && out && P >= 1 && R >= 1 && C >= 1, NLAM_E_INVALID, "nlam_reduce_partials: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  {
    ProfScope ps("reduce_partials_kernel", st, 4.0 * P * R * C);
    launch_reduce_partials(part, P, R, C, out, out_pitch, accumulate, st);
  }
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

extern "C" int nlam_transpose_pad(const float* x, int64_t rows, int C, int64_t x_pitch, float* xt, int64_t rows_pad, void* stream) {
  NLAM_REQUIRE(x && xt && rows >= 0 && rows_pad >= rows && C >= 1, NLAM_E_INVALID, "nlam_transpose_pad: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const long long tiles = ((rows_pad + 31) / 32) * ((C + 31) / 32);
  {
    ProfScope ps("transpose_pad_kernel", st, 4.0 * C * (rows + rows_pad));
    transpose_pad_kernel<<<(int)std::min<long long>(tiles, 132 * 16), 256, 0, st>>>(x, rows, C, x_pitch, xt, rows_pad);
  }
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

extern "C" int nlam_add_gather(const float* a, const float* v, const int32_t* idx, const int32_t* deg_ptr, int64_t n_e,
                               int64_t n_v, int H, int B, float* out, void* stream) {
  NLAM_REQUIRE(v && idx && out && H % 4 == 0, NLAM_E_INVALID, "nlam_add_gather: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = (long long)B * n_e * (H / 4);
  if (total == 0) return NLAM_OK;
  {
    ProfScope ps("add_gather_kernel", st, 4.0 * B * n_e * H * (a ? 3 : 2));
    add_gather_kernel<<<grid_1d(total, 256), 256, 0, st>>>(a, v, idx, deg_ptr, n_e, n_v, H / 4, B, out);
  }
  count_launch();
  NLAM_CUDA_OK(cudaGetLastError());
  return NLAM_OK;
}

// Generic wgmma Linear through the C ABI (LinearCall fields flattened; see common.cuh / tc7.cu)
extern "C" int nlam_linear(const float* x0, int64_t x0_bs, int k0, int64_t x0_pitch, const float* x1, int64_t x1_bs, int k1,
                           const float* w, int ldw, int w_cols, int64_t w_bs, const float* bias, int n_out, int act,
                           const float* gamma, const float* beta, float eps, const float* add0, const int32_t* add0_idx,
                           int64_t add0_bs, const float* add1, const int32_t* add1_idx, int64_t add1_bs, const float* post,
                           const int32_t* post_idx, int64_t post_bs, const float* res, int64_t res_bs, int64_t n_rows, int B,
                           float* out, float* out2, void* stream) {
  NLAM_REQUIRE(x0 && w && out && n_rows >= 1 && B >= 1, NLAM_E_INVALID, "nlam_linear: bad arguments");
  LinearCall c;
  memset(&c, 0, sizeof(c));
  c.x0 = x0; c.x0_bs = x0_bs; c.k0 = k0; c.x0_pitch = x0_pitch; c.x1 = x1; c.x1_bs = x1_bs; c.k1 = k1;
  c.w = w; c.ldw = ldw; c.w_cols = w_cols; c.w_bs = w_bs; c.bias = bias; c.n_out = n_out; c.act = act;
  c.gamma = gamma; c.beta = beta; c.eps = eps;
  c.add[0] = add0; c.add_idx[0] = add0_idx; c.add_bs[0] = add0_bs;
  c.add[1] = add1; c.add_idx[1] = add1_idx; c.add_bs[1] = add1_bs;
  c.post = post; c.post_idx = post_idx; c.post_bs = post_bs; c.res = res; c.res_bs = res_bs;
  c.n_rows = n_rows; c.B = B; c.out = out; c.out2 = out2;
  return tc_linear(c, (cudaStream_t)stream);
}

// =====================================================================================================================
// nlam_mlp_bwd / nlam_inet_bwd: the backward chains composed on the host side of the ABI (one call per layer; all
// temporaries in the caller's workspace; same sequence of launches as neural_lam_b200/backward.py, which remains as the
// readable restatement and is tested against this).
// =====================================================================================================================
namespace nlam {
namespace {

struct Arena {  // stack allocator over the caller's workspace; dry = size the workspace without touching memory
  float* base;
  size_t off, cap;
  bool dry;
  size_t peak = 0;
  bool overflow = false;
  float* get(size_t n) {
    n = (n + 63) / 64 * 64;
    float* p = dry ? nullptr : base + off;
    off += n;
    peak = std::max(peak, off);
    if (!dry && off > cap) overflow = true;
    return p;
  }
  size_t mark() const { return off; }
  void release(size_t m) { off = m; }
  void note() {}
};

struct Ctx {
  Arena a;
  cudaStream_t st;
  int rc = NLAM_OK;
  bool ok() const { return rc == NLAM_OK && !a.overflow; }
};

#define BW_TRY(expr)                  \
  do {                                \
    if (!c.a.dry && c.ok()) c.rc = (expr); \
  } while (0)

// out (B, n, n_out) = epi(x0 (+x1) · w[:, w_off ..]ᵀ ...)
struct LinArgs {
  const float* x0 = nullptr; int64_t x0_bs = 0; int k0 = 0; int64_t x0_pitch = 0;
  const float* x1 = nullptr; int64_t x1_bs = 0; int k1 = 0;
  const float* w = nullptr; int ldw = 0; int w_cols = 0; int64_t w_bs = 0;
  const float* bias = nullptr; int n_out = 0;
  const float* add0 = nullptr; const int32_t* idx0 = nullptr; int64_t add0_bs = 0;
  const float* add1 = nullptr; const int32_t* idx1 = nullptr; int64_t add1_bs = 0;
  const float* res = nullptr; int64_t res_bs = 0;
  int64_t n = 0; int B = 1;
};

static void lin(Ctx& c, const LinArgs& a, float* out) {
  if (c.a.dry || !c.ok()) return;
  LinearCall q;
  memset(&q, 0, sizeof(q));
  q.x0 = a.x0; q.x0_bs = a.x0_bs; q.k0 = a.k0; q.x0_pitch = a.x0_pitch; q.x1 = a.x1; q.x1_bs = a.x1_bs; q.k1 = a.k1;
  q.w = a.w; q.ldw = a.ldw; q.w_cols = a.w_cols; q.w_bs = a.w_bs; q.bias = a.bias; q.n_out = a.n_out;
  q.add[0] = a.add0; q.add_idx[0] = a.idx0; q.add_bs[0] = a.add0_bs; q.add[1] = a.add1; q.add_idx[1] = a.idx1; q.add_bs[1] = a.add1_bs;
  q.res = a.res; q.res_bs = a.res_bs; q.n_rows = a.n; q.B = a.B; q.out = out;
  c.rc = tc_linear(q, c.st);
}

// xt (C, rows_pad) = transpose of x rows (row r reads x[(r % mod_rows) * pitch + col]); zero padded
__global__ void transpose_mod_kernel(const float* __restrict__ x, long long rows, long long mod_rows, int C, long long x_pitch,
                                     float* __restrict__ xt, long long rows_pad) {
  __shared__ float tile[32][33];
  const long long tiles_r = (rows_pad + 31) / 32;
  const int tiles_c = (C + 31) / 32;
  for (long long t = blockIdx.x; t < tiles_r * tiles_c; t += gridDim.x) {
    const long long tr = t / tiles_c;
    const int tc = (int)(t - tr * tiles_c);
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int j = ty; j < 32; j += 8) {
      const long long r = tr * 32 + j;
      const int col = tc * 32 + tx;
      tile[j][tx] = (r < rows && col < C) ? x[(mod_rows >= rows ? r : r % mod_rows) * x_pitch + col] : 0.f;
    }
    __syncthreads();
    for (int j = ty; j < 32; j += 8) {
      const int col = tc * 32 + j;
      const long long r = tr * 32 + tx;
      if (col < C && r < rows_pad) xt[(long long)col * rows_pad + r] = tile[tx][j];
    }
    __syncthreads();
  }
}

static void transpose(Ctx& c, const float* x, int64_t rows, int64_t mod_rows, int C, int64_t pitch, float* xt, int64_t rows_pad) {
  if (c.a.dry || !c.ok()) return;
  const long long tiles = ((rows_pad + 31) / 32) * ((C + 31) / 32);
  {
    ProfScope ps("transpose_pad_kernel", c.st, 4.0 * C * (rows + rows_pad));
    transpose_mod_kernel<<<(int)std::min<long long>(tiles, 132 * 16), 256, 0, c.st>>>(x, rows, mod_rows, C, pitch, xt, rows_pad);
  }
  count_launch();
  if (cudaGetLastError() != cudaSuccess) c.rc = NLAM_E_CUDA;
}

// out[:, off .. off+K) (pitch out_pitch) = gyᵀ (R x N, dense) · x (R x K; rows repeat with period x_mod, pitch x_pitch)
static void grad_weight(Ctx& c, const float* gy, int64_t R, int N, const float* x, int64_t x_mod, int K, int64_t x_pitch,
                        float* out, int64_t out_pitch) {
  const int n_tiles = (N + 127) / 128;
  const int64_t S = std::max<int64_t>(1, std::min<int64_t>(296 / n_tiles, (R + 511) / 512));
  const int64_t k_per = (((R + S - 1) / S) + 31) / 32 * 32;
  const int64_t rows_pad = S * k_per;
  const size_t m = c.a.mark();
  float* gyT = c.a.get((size_t)N * rows_pad);
  transpose(c, gy, R, R, N, N, gyT, rows_pad);
  for (int c0 = 0; c0 < K; c0 += 256) {
    const int kc = std::min(256, K - c0);
    const size_t m2 = c.a.mark();
    float* xT = c.a.get((size_t)kc * rows_pad);
    float* part = c.a.get((size_t)S * N * kc);
    c.a.note();
    transpose(c, x + c0, R, x_mod, kc, x_pitch, xT, rows_pad);
    LinArgs a;
    a.x0 = gyT; a.x0_bs = k_per; a.k0 = (int)k_per; a.x0_pitch = rows_pad; a.w = xT; a.ldw = (int)rows_pad; a.w_cols = (int)k_per;
    a.w_bs = k_per; a.n_out = kc; a.n = N; a.B = (int)S;
    lin(c, a, part);
    if (!c.a.dry && c.ok()) c.rc = nlam_reduce_partials(part, (int)S, N, kc, out + c0, out_pitch, 0, c.st);
    c.a.release(m2);
  }
  c.a.release(m);
}

// out (B, n, n_in) = gy (B, n, N dense) · W[:, w_off .. w_off + n_in)  (+ res dense).  The Linear kernel's output is at
// most 256 wide: a wider n_in (an MLP input of more than 256 columns) runs one Linear per 256-column block of W into a
// temporary that is copied into its column slice of out; res is only supported with n_in <= 256.
static void grad_input(Ctx& c, const float* gy, int64_t n, int B, int N, const float* w, int ldw, int n_in, const float* res,
                       float* out) {
  const int Np = (N + 31) / 32 * 32, N4 = (N + 3) / 4 * 4;
  const bool chunked = n_in > 256;
  if (chunked && res) {
    if (!c.a.dry && c.ok()) {
      set_error("grad_input: a residual needs n_in <= 256 (got %d)", n_in);
      c.rc = NLAM_E_UNSUPPORTED;
    }
    return;
  }
  const size_t m = c.a.mark();
  const float* x0 = gy;
  if (Np != N) {
    float* pk = c.a.get((size_t)B * n * Np);
    if (!c.a.dry && c.ok())
      c.rc = nlam_pack_rows(gy, nullptr, nullptr, nullptr, N, 0, 0, 0, n * N, 0, 0, 0, pk, Np, n, B, c.st);
    x0 = pk;
  }
  for (int c0 = 0; c0 < n_in; c0 += 256) {
    const int kc = std::min(256, n_in - c0);
    const size_t m2 = c.a.mark();
    float* wT = c.a.get((size_t)kc * N4);
    float* dst = chunked ? c.a.get((size_t)B * n * kc) : out;
    c.a.note();
    transpose(c, w + c0, N, N, kc, ldw, wT, N4);
    LinArgs a;
    a.x0 = x0; a.x0_bs = n * Np; a.k0 = Np; a.w = wT; a.ldw = N4; a.w_cols = N; a.n_out = kc; a.res = res; a.res_bs = n * kc;
    a.n = n; a.B = B;
    lin(c, a, dst);
    if (chunked && !c.a.dry && c.ok() &&
        cudaMemcpy2DAsync(out + c0, (size_t)n_in * 4, dst, (size_t)kc * 4, (size_t)kc * 4, (size_t)B * n, cudaMemcpyDeviceToDevice,
                          c.st) != cudaSuccess)
      c.rc = NLAM_E_CUDA;
    c.a.release(m2);
  }
  c.a.release(m);
}

static void silu_(Ctx& c, const float* z, const float* gh, float* out, int64_t n) { BW_TRY(nlam_silu(z, gh, out, n, c.st)); }
static void colsum_(Ctx& c, const float* g, int64_t rows, int C, float* out) {
  const size_t m = c.a.mark();
  float* sc = c.a.get(nlam_bwd_scratch_floats(C));
  c.a.note();
  BW_TRY(nlam_colsum(g, rows, C, out, sc, c.st));
  c.a.release(m);
}
static void ln_bwd_(Ctx& c, const float* g, const float* y, const float* gamma, float eps, float* gy, float* dgamma, float* dbeta,
                    int64_t rows, int H) {
  const size_t m = c.a.mark();
  float* sc = c.a.get(nlam_bwd_scratch_floats(H));
  c.a.note();
  BW_TRY(nlam_layernorm_bwd(g, y, gamma, eps, gy, dgamma, dbeta, rows, H, sc, c.st));
  c.a.release(m);
}

struct MlpBwdArgs {
  const NlamMlp* mlp;
  const NlamRowSrc* srcs;
  int n_src;
  const float* g_out;   // (B, n, n_out) dense
  float* const* g_srcs; // per source (B, n, dim) dense or NULL
  const NlamMlpGrads* grads;
  int64_t n;
  int B;
};

static void mlp_bwd_impl(Ctx& c, const MlpBwdArgs& q) {
  const NlamMlp* m = q.mlp;
  const int K = m->in_dim, H = m->out_dim[0], no = m->out_dim[1];
  const int Kp = (K + 31) / 32 * 32, K4 = (K + 3) / 4 * 4;
  const int64_t n = q.n;
  const int B = q.B;
  const int64_t rows = n * B;
  const size_t mk = c.a.mark();
  // packed, zero-padded input (B, n, Kp)
  const float* x = nullptr;
  int64_t x_bs = 0;
  if (q.n_src == 1 && K == Kp) {
    x = q.srcs[0].ptr;
    x_bs = q.srcs[0].bstride;
  } else {
    float* pk = c.a.get((size_t)rows * Kp);
    const NlamRowSrc* s = q.srcs;
    if (!c.a.dry && c.ok())
      c.rc = nlam_pack_rows(s[0].ptr, q.n_src > 1 ? s[1].ptr : nullptr, q.n_src > 2 ? s[2].ptr : nullptr,
                            q.n_src > 3 ? s[3].ptr : nullptr, s[0].dim, q.n_src > 1 ? s[1].dim : 0, q.n_src > 2 ? s[2].dim : 0,
                            q.n_src > 3 ? s[3].dim : 0, B > 1 ? s[0].bstride : 0, (q.n_src > 1 && B > 1) ? s[1].bstride : 0,
                            (q.n_src > 2 && B > 1) ? s[2].bstride : 0, (q.n_src > 3 && B > 1) ? s[3].bstride : 0, pk, Kp, n, B, c.st);
    x = pk;
    x_bs = n * Kp;
  }
  const float* W1 = m->w[0];
  int ldw1 = K;
  if (K % 4) {  // 16-byte row pitch for TMA
    float* wp = c.a.get((size_t)H * K4);
    if (!c.a.dry && c.ok()) c.rc = nlam_pack_rows(m->w[0], nullptr, nullptr, nullptr, K, 0, 0, 0, 0, 0, 0, 0, wp, K4, H, 1, c.st);
    W1 = wp;
    ldw1 = K4;
  }
  float* z = c.a.get((size_t)rows * H);
  float* h = c.a.get((size_t)rows * H);
  {
    LinArgs a;
    a.x0 = x; a.x0_bs = x_bs; a.k0 = Kp; a.w = W1; a.ldw = ldw1; a.w_cols = K; a.bias = m->b[0]; a.n_out = H; a.n = n; a.B = B;
    lin(c, a, z);
  }
  silu_(c, z, nullptr, h, rows * H);
  const float* g_y = q.g_out;
  if (m->ln_gamma) {
    float* y = c.a.get((size_t)rows * no);
    float* gy = c.a.get((size_t)rows * no);
    LinArgs a;
    a.x0 = h; a.x0_bs = n * H; a.k0 = H; a.w = m->w[1]; a.ldw = H; a.bias = m->b[1]; a.n_out = no; a.n = n; a.B = B;
    lin(c, a, y);
    ln_bwd_(c, q.g_out, y, m->ln_gamma, m->ln_eps, gy, q.grads->ln_gamma, q.grads->ln_beta, rows, no);
    g_y = gy;
  }
  colsum_(c, g_y, rows, no, q.grads->b[1]);
  grad_weight(c, g_y, rows, no, h, rows, H, H, q.grads->w[1], H);
  float* g_h = c.a.get((size_t)rows * H);
  grad_input(c, g_y, n, B, no, m->w[1], H, H, nullptr, g_h);
  silu_(c, z, g_h, g_h, rows * H);  // in place: g_z
  colsum_(c, g_h, rows, H, q.grads->b[0]);
  grad_weight(c, g_h, rows, H, x, (x_bs == 0 && B > 1) ? n : rows, K, Kp == K && q.n_src == 1 ? K : Kp, q.grads->w[0], K);
  bool need_src = false;
  for (int s = 0; s < q.n_src; ++s) need_src |= q.g_srcs && q.g_srcs[s];
  if (need_src) {
    float* gx = c.a.get((size_t)rows * K);
    grad_input(c, g_h, n, B, H, m->w[0], K, K, nullptr, gx);
    // split the columns back into the sources (strided device-to-device copies)
    int col = 0;
    for (int s = 0; s < q.n_src; ++s) {
      const int d = q.srcs[s].dim;
      if (q.g_srcs[s] && !c.a.dry && c.ok()) {
        if (cudaMemcpy2DAsync(q.g_srcs[s], (size_t)d * 4, gx + col, (size_t)K * 4, (size_t)d * 4, (size_t)rows,
                              cudaMemcpyDeviceToDevice, c.st) != cudaSuccess)
          c.rc = NLAM_E_CUDA;
      }
      col += d;
    }
  }
  c.a.note();
  c.a.release(mk);
}

struct InetBwdArgs {
  const NlamGraph* g;
  const NlamMlp* em;
  const NlamMlp* am;
  const float* send; int64_t send_bs;
  const float* rec; int64_t rec_bs;
  const float* edge; int64_t edge_bs;
  const float* g_rec_out;
  const float* g_edge_out;
  float* g_send; float* g_rec; float* g_edge;
  const NlamMlpGrads* eg;
  const NlamMlpGrads* ag;
  int B;
  int flags;
};

static void inet_bwd_impl(Ctx& c, const InetBwdArgs& q) {
  const NlamGraph* g = q.g;
  const int H = q.em->out_dim[1], B = q.B;
  const bool prop = q.flags & NLAM_PROPAGATION;
  const int mean = (q.flags & (NLAM_AGGR_MEAN | NLAM_PROPAGATION)) ? 1 : 0;
  const int64_t Ns = g->n_send, Nr = g->n_rec, E = g->n_edges;
  const int64_t sbs = B > 1 ? q.send_bs : 0, rbs = B > 1 ? q.rec_bs : 0, ebs = B > 1 ? q.edge_bs : 0;
  const int64_t s_mod = (sbs == 0 && B > 1) ? Ns : Ns * B, r_mod = (rbs == 0 && B > 1) ? Nr : Nr * B,
                e_mod = (ebs == 0 && B > 1) ? E : E * B;
  // dense-batch views are required for the transposes (rows of all batches contiguous)
  const float* W1 = q.em->w[0];
  const float* W2 = q.em->w[1];
  const float* Wn1 = q.am->w[0];
  const float* Wn2 = q.am->w[1];
  const size_t mk = c.a.mark();
  float* Ps = c.a.get((size_t)B * Ns * H);
  float* Pr = c.a.get((size_t)B * Nr * H);
  float* z1 = c.a.get((size_t)B * E * H);
  float* h1 = c.a.get((size_t)B * E * H);
  float* y2 = c.a.get((size_t)B * E * H);
  float* msg = c.a.get((size_t)B * E * H);
  float* aggr = c.a.get((size_t)B * Nr * H);
  float* nz = c.a.get((size_t)B * Nr * H);
  float* nh = c.a.get((size_t)B * Nr * H);
  float* ny = c.a.get((size_t)B * Nr * H);
  float* t_n1 = c.a.get((size_t)B * Nr * H);  // g_ny, later g_Pr
  float* t_n2 = c.a.get((size_t)B * Nr * H);  // g_nh / g_nz
  float* g_aggr = c.a.get((size_t)B * Nr * H);
  float* g_rec0 = c.a.get((size_t)B * Nr * H);
  float* g_Ps = c.a.get((size_t)B * Ns * H);
  float* g_sp = prop ? c.a.get((size_t)B * Ns * H) : nullptr;
  c.a.note();
  // ---- forward recompute
  {
    LinArgs a;
    a.x0 = q.send; a.x0_bs = sbs; a.k0 = H; a.w = W1 + H; a.ldw = 3 * H; a.n_out = H; a.n = Ns; a.B = B;
    lin(c, a, Ps);
    LinArgs b;
    b.x0 = q.rec; b.x0_bs = rbs; b.k0 = H; b.w = W1 + 2 * H; b.ldw = 3 * H; b.bias = q.em->b[0]; b.n_out = H; b.n = Nr; b.B = B;
    lin(c, b, Pr);
    LinArgs e;
    e.x0 = q.edge; e.x0_bs = ebs; e.k0 = H; e.w = W1; e.ldw = 3 * H; e.n_out = H; e.n = E; e.B = B;
    e.add0 = Ps; e.idx0 = g->src; e.add0_bs = Ns * H; e.add1 = Pr; e.idx1 = g->dst; e.add1_bs = Nr * H;
    lin(c, e, z1);
  }
  silu_(c, z1, nullptr, h1, (int64_t)B * E * H);
  {
    LinArgs a;
    a.x0 = h1; a.x0_bs = E * H; a.k0 = H; a.w = W2; a.ldw = H; a.bias = q.em->b[1]; a.n_out = H; a.n = E; a.B = B;
    lin(c, a, y2);
  }
  BW_TRY(nlam_layernorm_fwd(y2, q.em->ln_gamma, q.em->ln_beta, q.em->ln_eps, msg, (int64_t)B * E, H, c.st));
  if (prop) {
    // m += x_j: gather of the (dense-batch) sender rows
    if (sbs == 0 && B > 1) {
      for (int b = 0; b < B; ++b)
        BW_TRY(nlam_add_gather(msg + (size_t)b * E * H, q.send, g->src, nullptr, E, Ns, H, 1, msg + (size_t)b * E * H, c.st));
    } else {
      BW_TRY(nlam_add_gather(msg, q.send, g->src, nullptr, E, Ns, H, B, msg, c.st));
    }
  }
  BW_TRY(nlam_segment_sum(g->rowptr, nullptr, Nr, msg, E * H, aggr, Nr * H, B, H, mean, c.st));
  {
    LinArgs a;
    a.x0 = q.rec; a.x0_bs = rbs; a.k0 = H; a.x1 = aggr; a.x1_bs = Nr * H; a.k1 = H; a.w = Wn1; a.ldw = 2 * H; a.bias = q.am->b[0];
    a.n_out = H; a.n = Nr; a.B = B;
    lin(c, a, nz);
  }
  silu_(c, nz, nullptr, nh, (int64_t)B * Nr * H);
  {
    LinArgs a;
    a.x0 = nh; a.x0_bs = Nr * H; a.k0 = H; a.w = Wn2; a.ldw = H; a.bias = q.am->b[1]; a.n_out = H; a.n = Nr; a.B = B;
    lin(c, a, ny);
  }
  // ---- node update backward
  ln_bwd_(c, q.g_rec_out, ny, q.am->ln_gamma, q.am->ln_eps, t_n1, q.ag->ln_gamma, q.ag->ln_beta, (int64_t)B * Nr, H);
  colsum_(c, t_n1, (int64_t)B * Nr, H, q.ag->b[1]);
  grad_weight(c, t_n1, (int64_t)B * Nr, H, nh, (int64_t)B * Nr, H, H, q.ag->w[1], H);
  grad_input(c, t_n1, Nr, B, H, Wn2, H, H, nullptr, t_n2);
  silu_(c, nz, t_n2, t_n2, (int64_t)B * Nr * H);  // g_nz
  colsum_(c, t_n2, (int64_t)B * Nr, H, q.ag->b[0]);
  grad_weight(c, t_n2, (int64_t)B * Nr, H, q.rec, r_mod, H, H, q.ag->w[0], 2 * H);
  grad_weight(c, t_n2, (int64_t)B * Nr, H, aggr, (int64_t)B * Nr, H, H, q.ag->w[0] + H, 2 * H);
  grad_input(c, t_n2, Nr, B, H, Wn1, 2 * H, H, prop ? nullptr : q.g_rec_out, g_rec0);
  grad_input(c, t_n2, Nr, B, H, Wn1 + H, 2 * H, H, prop ? q.g_rec_out : nullptr, g_aggr);
  // ---- message gradient and the edge MLP
  float* g_m = msg;  // the messages themselves are no longer needed
  BW_TRY(nlam_add_gather(q.g_edge_out, g_aggr, g->dst, mean ? g->rowptr : nullptr, E, Nr, H, B, g_m, c.st));
  float* g_y2 = c.a.get((size_t)B * E * H);
  c.a.note();
  ln_bwd_(c, g_m, y2, q.em->ln_gamma, q.em->ln_eps, g_y2, q.eg->ln_gamma, q.eg->ln_beta, (int64_t)B * E, H);
  if (prop) BW_TRY(nlam_segment_sum(g->sptr, g->sperm, Ns, g_m, E * H, g_sp, Ns * H, B, H, 0, c.st));
  colsum_(c, g_y2, (int64_t)B * E, H, q.eg->b[1]);
  grad_weight(c, g_y2, (int64_t)B * E, H, h1, (int64_t)B * E, H, H, q.eg->w[1], H);
  float* g_z1 = y2;  // y2 is dead once g_y2 exists
  grad_input(c, g_y2, E, B, H, W2, H, H, nullptr, g_z1);
  silu_(c, z1, g_z1, g_z1, (int64_t)B * E * H);
  grad_weight(c, g_z1, (int64_t)B * E, H, q.edge, e_mod, H, H, q.eg->w[0], 3 * H);
  grad_input(c, g_z1, E, B, H, W1, 3 * H, H, q.g_edge_out, q.g_edge);
  BW_TRY(nlam_segment_sum(g->sptr, g->sperm, Ns, g_z1, E * H, g_Ps, Ns * H, B, H, 0, c.st));
  float* g_Pr = t_n1;
  BW_TRY(nlam_segment_sum(g->rowptr, nullptr, Nr, g_z1, E * H, g_Pr, Nr * H, B, H, 0, c.st));
  colsum_(c, g_Pr, (int64_t)B * Nr, H, q.eg->b[0]);
  grad_weight(c, g_Ps, (int64_t)B * Ns, H, q.send, s_mod, H, H, q.eg->w[0] + H, 3 * H);
  grad_weight(c, g_Pr, (int64_t)B * Nr, H, q.rec, r_mod, H, H, q.eg->w[0] + 2 * H, 3 * H);
  grad_input(c, g_Ps, Ns, B, H, W1 + H, 3 * H, H, g_sp, q.g_send);
  grad_input(c, g_Pr, Nr, B, H, W1 + 2 * H, 3 * H, H, g_rec0, q.g_rec);
  c.a.note();
  c.a.release(mk);
}

}  // namespace
}  // namespace nlam

static bool bwd_shapes_ok(const NlamMlp* m) {
  if (!m || m->n_linear != 2) return false;
  const int H = m->out_dim[0], no = m->out_dim[1];
  return H % 32 == 0 && H <= 256 && no >= 1 && no <= 256 && (!m->ln_gamma || no == 32 || no == 64 || no == 128 || no == 256);
}

extern "C" size_t nlam_mlp_bwd_workspace_bytes(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, int64_t n_rows, int B) {
  if (!bwd_shapes_ok(mlp) || !srcs || n_src < 1 || n_src > 4) return 0;
  Ctx c;
  c.a = Arena{nullptr, 0, 0, true};
  c.st = nullptr;
  NlamMlpGrads dummy;
  memset(&dummy, 0, sizeof(dummy));
  float* gs[4] = {(float*)16, (float*)16, (float*)16, (float*)16};
  MlpBwdArgs q{mlp, srcs, n_src, nullptr, gs, &dummy, n_rows, B};
  mlp_bwd_impl(c, q);
  return (c.a.peak + 64) * sizeof(float);
}

extern "C" int nlam_mlp_bwd(const NlamMlp* mlp, const NlamRowSrc* srcs, int n_src, const float* g_out, float* const* g_srcs,
                            const NlamMlpGrads* grads, int64_t n_rows, int B, void* workspace, size_t ws_bytes, void* stream) {
  NLAM_REQUIRE(mlp && srcs && g_out && grads && workspace && n_src >= 1 && n_src <= 4, NLAM_E_INVALID, "nlam_mlp_bwd: null argument");
  NLAM_REQUIRE(bwd_shapes_ok(mlp), NLAM_E_UNSUPPORTED, "nlam_mlp_bwd: MLP shape not covered (two Linear layers, hidden width a multiple of 32 <= 256)");
  for (int s = 0; s < n_src; ++s) NLAM_REQUIRE(!srcs[s].idx, NLAM_E_UNSUPPORTED, "nlam_mlp_bwd: gathered sources unsupported");
  NLAM_REQUIRE(ws_bytes >= nlam_mlp_bwd_workspace_bytes(mlp, srcs, n_src, n_rows, B), NLAM_E_WORKSPACE, "nlam_mlp_bwd: workspace too small");
  Ctx c;
  c.a = Arena{(float*)workspace, 0, ws_bytes / sizeof(float), false};
  c.st = (cudaStream_t)stream;
  MlpBwdArgs q{mlp, srcs, n_src, g_out, g_srcs, grads, n_rows, B};
  mlp_bwd_impl(c, q);
  NLAM_REQUIRE(!c.a.overflow, NLAM_E_WORKSPACE, "nlam_mlp_bwd: workspace overflow");
  return c.rc;
}

extern "C" size_t nlam_inet_bwd_workspace_bytes(const NlamGraph* g, int B, int H, int flags) {
  if (!g) return 0;
  Ctx c;
  c.a = Arena{nullptr, 0, 0, true};
  c.st = nullptr;
  NlamMlp em, am;
  memset(&em, 0, sizeof(em));
  memset(&am, 0, sizeof(am));
  em.n_linear = am.n_linear = 2;
  em.in_dim = 3 * H; am.in_dim = 2 * H;
  em.out_dim[0] = em.out_dim[1] = am.out_dim[0] = am.out_dim[1] = H;
  NlamMlpGrads d;
  memset(&d, 0, sizeof(d));
  InetBwdArgs q{g, &em, &am, nullptr, 1, nullptr, 1, nullptr, 1, nullptr, nullptr, nullptr, nullptr, nullptr, &d, &d, B, flags};
  inet_bwd_impl(c, q);
  return (c.a.peak + 64) * sizeof(float);
}

extern "C" int nlam_inet_bwd(const NlamGraph* g, const NlamMlp* edge_mlp, const NlamMlp* aggr_mlp, const float* send,
                             int64_t send_bs, const float* rec, int64_t rec_bs, const float* edge, int64_t edge_bs,
                             const float* g_rec_out, const float* g_edge_out, float* g_send, float* g_rec, float* g_edge,
                             const NlamMlpGrads* edge_grads, const NlamMlpGrads* aggr_grads, int B, int flags, void* workspace,
                             size_t ws_bytes, void* stream) {
  NLAM_REQUIRE(g && edge_mlp && aggr_mlp && send && rec && edge && g_rec_out && g_send && g_rec && g_edge && edge_grads &&
                   aggr_grads && workspace,
               NLAM_E_INVALID, "nlam_inet_bwd: null argument");
  const int H = edge_mlp->out_dim[1];
  NLAM_REQUIRE(bwd_shapes_ok(edge_mlp) && bwd_shapes_ok(aggr_mlp) && edge_mlp->ln_gamma && aggr_mlp->ln_gamma &&
                   (H == 64 || H == 128 || H == 256) && edge_mlp->in_dim == 3 * H && aggr_mlp->in_dim == 2 * H &&
                   edge_mlp->out_dim[0] == H && aggr_mlp->out_dim[0] == H && aggr_mlp->out_dim[1] == H,
               NLAM_E_UNSUPPORTED, "nlam_inet_bwd: layer shape not covered (hidden_layers = 1, H in {64, 128, 256})");
  NLAM_REQUIRE(ws_bytes >= nlam_inet_bwd_workspace_bytes(g, B, H, flags), NLAM_E_WORKSPACE, "nlam_inet_bwd: workspace too small");
  Ctx c;
  c.a = Arena{(float*)workspace, 0, ws_bytes / sizeof(float), false};
  c.st = (cudaStream_t)stream;
  InetBwdArgs q{g, edge_mlp, aggr_mlp, send, send_bs, rec, rec_bs, edge, edge_bs, g_rec_out, g_edge_out, g_send, g_rec, g_edge,
                edge_grads, aggr_grads, B, flags};
  inet_bwd_impl(c, q);
  NLAM_REQUIRE(!c.a.overflow, NLAM_E_WORKSPACE, "nlam_inet_bwd: workspace overflow");
  return c.rc;
}

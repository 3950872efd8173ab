// Shared device-side PTX wrappers (mbarrier, TMA, wgmma, cp.async) and host-side tensor-map helpers for the sm_90a
// tensor-core kernels.
#pragma once
#include <cuda.h>
#include <stdlib.h>

#include <mutex>

#include "common.cuh"

namespace nlam {

// ------------------------------------------------------------------------------------ PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  // try_wait suspends the thread in hardware until the phase completes or the time hint expires
  uint32_t done = 0;
  uint32_t spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(1000000u)
        : "memory");
    if (done) break;
    if (++spins > (1u << 20)) {  // bounded: a protocol bug must not hang the GPU
      printf("nlam tc kernel: mbarrier timeout (block %d thread %d bar %u parity %u)\n", blockIdx.x, threadIdx.x, bar,
             parity);
      __trap();
    }
  }
}
// mbar_wait without the diagnostic printf, for kernels whose MMAs must stay pipelined: a call (printf) anywhere in a kernel
// makes ptxas wait for every wgmma before issuing the next (C7510)
__device__ __forceinline__ void mbar_wait_nocall(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  uint32_t spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(1000000u)
        : "memory");
    if (done) break;
    if (++spins > (1u << 20)) __trap();  // bounded: a protocol bug must not hang the GPU
  }
}
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done != 0;
}
// one elected lane of a converged warp (the warp stays in uniform control flow, so TMA operands live in
// uniform registers instead of going through an R2UR + waterfall loop per instruction)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
// warp-uniform barrier test (every lane tests; lane 0's answer is taken so the compiler sees a uniform value)
__device__ __forceinline__ bool mbar_test_u(uint32_t bar, uint32_t parity) {
  return __shfl_sync(0xffffffffu, (int)mbar_test(bar, parity), 0) != 0;
}
// Programmatic dependent launch: a kernel launched with the programmatic-stream-serialization attribute (launch_pdl below)
// may start while the previous kernel in the stream is still draining; it must not touch anything that kernel writes before
// pdl_wait() (= the previous grid has completed and its writes are visible).  pdl_launch_dependents() lets the NEXT kernel begin
// to launch as this grid's CTAs exit.  Both are no-ops for a kernel launched without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int n) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}

// One warp of a warp group polls the mbarrier; the others block on a hardware named barrier, which
// costs no issue slots (26 warps all polling measurably slowed the working warps down).
__device__ __forceinline__ void group_wait(bool leader, uint32_t bar, uint32_t parity, int bar_id, int nthreads) {
  if (leader) mbar_wait(bar, parity);
  named_bar_sync(bar_id, nthreads);
}

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// L2 eviction policies: the streamed edge tiles (hundreds of MB per layer at the bench batch) must
// not push the small, heavily re-read node rows (gather sources) out of the 50 MB L2.
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t policy_evict_normal() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                            uint64_t pol) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "l"(pol)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
// e'[box] += smem tile (fp32 add performed in L2; element type and swizzle come from the tensor map)
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
// 1-D bulk copy global -> shared (16-byte aligned addresses, size a multiple of 16), completion on an mbarrier
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// 1-D bulk copy shared -> global (16-byte aligned addresses, size a multiple of 16), bulk-group completion
__device__ __forceinline__ void bulk_store_1d(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void tma_prefetch_3d(const CUtensorMap* map, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];"
               ::"l"(map), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
// bring one 128-byte line into L2 without holding a register
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src, uint64_t pol) {
  asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async_4(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
// arrive on an mbarrier once all cp.async of this thread issued so far have landed (the arrival counts against the
// barrier's expected count)
__device__ __forceinline__ void cp_async_mbar_arrive(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// wait until at most N of this thread's committed cp.async groups are pending
template <int N>
__device__ __forceinline__ void cp_async_wait_group() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

// wgmma shared-memory matrix descriptor (sm_90): K-major, 128-byte swizzle, 8-row groups 1024 B apart
// (start >> 4 at [0,14), LBO >> 4 at [16,30) (unused for swizzled K-major), SBO >> 4 at [32,46), layout [62,64): 1 = SWIZZLE_128B).
// Advancing K by 8 tf32 elements inside the 128-byte swizzle row adds 32 B (= 2 in the start field).
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// the accumulator registers are written asynchronously between wgmma issue and wgmma.wait_group: the empty asm statements
// pin every read and write of them on the right side of the fence / wait
__device__ __forceinline__ void wgmma_fence(float* acc, int n) {
  for (int i = 0; i < n; ++i) asm volatile("" : "+f"(acc[i])::"memory");
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0(float* acc, int n) {
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
  for (int i = 0; i < n; ++i) asm volatile("" : "+f"(acc[i])::"memory");
}

// wgmma operands are rounded to TF32 (round to nearest, ties away from zero) in shared memory before the MMA reads them;
// the MMA would otherwise drop the low 13 mantissa bits (truncation: every product biased toward zero, by about 7e-4
// relative on average)
__device__ __forceinline__ float tf32r(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
__device__ __forceinline__ float4 tf32r4(float4 v) { return make_float4(tf32r(v.x), tf32r(v.y), tf32r(v.z), tf32r(v.w)); }

// byte offset of 16-byte chunk `ch` (0..7) of row `row` inside a 128B-swizzled [128][32 float] block
__device__ __forceinline__ uint32_t swz(int row, int ch) { return (uint32_t)(row * 128 + ((ch ^ (row & 7)) << 4)); }

__device__ __forceinline__ float silu_fast(float x) {
  // x*sigmoid(x) = h + h*tanh(h), h = x/2: one MUFU op (tanh.approx.f32, rel. error ~2^-11 — the
  // size of the TF32 rounding the value undergoes anyway as the second GEMM's operand)
  const float h = 0.5f * x;
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
  return fmaf(h, t, h);
}

// shared-memory read the compiler may not hoist or keep live across loop iterations (register pressure)
__device__ __forceinline__ float4 lds128(const void* ptr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"(smem_u32(ptr)));
  return v;
}
__device__ __forceinline__ float tanh_fast(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(x));
  return t;
}

// ------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)ptr;
  });
  return fn;
}

// rows x cols fp32 tensor with an optional batch dim; box = 32 cols x box_rows rows, 128B swizzle
inline int make_map(CUtensorMap* m, const void* ptr, uint64_t cols, uint64_t rows, uint64_t batch, uint64_t row_pitch_elems,
                    uint64_t bstride_elems, uint32_t box_rows, bool three_d) {
  EncodeTiledFn enc = get_encode();
  NLAM_REQUIRE(enc, NLAM_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[3] = {cols, rows, batch};
  cuuint64_t strides[2] = {row_pitch_elems * 4, bstride_elems * 4};
  cuuint32_t box[3] = {32, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, three_d ? 3 : 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  NLAM_REQUIRE(r == CUDA_SUCCESS, NLAM_E_CUDA, "cuTensorMapEncodeTiled failed (%d) ptr=%p cols=%llu rows=%llu", (int)r, ptr,
               (unsigned long long)cols, (unsigned long long)rows);
  return NLAM_OK;
}

// kernel<<<grid, block, smem, st>>>(args...) with the programmatic-stream-serialization attribute (NLAM_NO_PDL=1: without)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), int grid, int block, size_t smem, cudaStream_t st, Args&&... args) {
  static int pdl = -1;
  if (pdl < 0) pdl = getenv("NLAM_NO_PDL") ? 0 : 1;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)grid, 1, 1);
  cfg.blockDim = dim3((unsigned)block, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

inline bool mlp_shape_ok(const NlamMlp* m, int* nout) {
  if (m->n_linear != 2 || m->out_dim[0] != 64) return false;
  const int no = m->out_dim[1];
  if (no < 1 || no > 64) return false;
  if (m->ln_gamma && no != 64) return false;
  if (m->in_dim % 4 != 0 || m->in_dim > 192) return false;
  if (!aligned16(m->w[0]) || !aligned16(m->w[1]) || !aligned16(m->b[0]) || !aligned16(m->b[1])) return false;
  if (m->ln_gamma && (!aligned16(m->ln_gamma) || !aligned16(m->ln_beta))) return false;
  *nout = no;
  return true;
}

inline int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

}  // namespace nlam

// Shared device/host helpers for the sm_90a ProPainter kernels.
// PTX wrappers for mbarrier, cp.async, bulk async copy (TMA engine) and wgmma.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#define PP_OK 0
#define PP_ERR_CUDA 1
#define PP_ERR_ARG 2
#define PP_ERR_STATE 3

void pp_set_error(const char* fmt, ...);

#define PP_CUDA_CHECK(expr)                                                                   \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      pp_set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return PP_ERR_CUDA;                                                                     \
    }                                                                                         \
  } while (0)

#define PP_REQUIRE(cond, ...)        \
  do {                               \
    if (!(cond)) {                   \
      pp_set_error(__VA_ARGS__);     \
      return PP_ERR_ARG;             \
    }                                \
  } while (0)

#define PP_TRY(expr)                 \
  do {                               \
    int _r = (expr);                 \
    if (_r != PP_OK) return _r;      \
  } while (0)

static inline int pp_ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline long long pp_ceil_div64(long long a, long long b) { return (a + b - 1) / b; }

#ifdef __CUDACC__

namespace ppx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
// Bounded wait: a pipeline that never completes (bad tensor map, transaction-byte mismatch) traps instead of hanging
// the GPU; the host then sees cudaErrorLaunchFailure from the next CUDA call.  The bound is an iteration count of the
// (potentially blocking) try_wait -- 2^26 tries are >= 1 s even if every try returned at once -- so the retry path is
// three extra integer instructions and the satisfied path is unchanged (a globaltimer-based bound cost 10 % on the
// launch-latency-bound recurrent layers).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      ".reg .u32 n;\n"
      "mov.u32 n, 0;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "add.u32 n, n, 1;\n"
      "setp.lt.u32 p, n, 0x4000000;\n"
      "@p bra WAIT_LOOP;\n"
      "trap;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(addr),
      "r"(parity)
      : "memory");
}

// ------------------------------------------------------------------ grid-wide barrier (persistent kernels)
// All CTAs of a co-resident grid (cooperative launch) meet here: `counter` counts arrivals since it was zeroed, the
// k-th barrier of a kernel passes when it reaches k * gridDim.x.  Writes made before the barrier by any thread of the
// grid are visible to every thread after it (read them with ld.global.cg / __ldcg: L1 is not coherent across SMs).
__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    unsigned int v, spins = 0;
    uint64_t t0 = 0;
    for (;;) {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
      if (v >= target) break;
      if ((++spins & 0xFFFu) == 0) {     // a CTA that never arrives must not hang the GPU: trap after ~2 s
        uint64_t now;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
        if (t0 == 0) t0 = now;
        else if (now - t0 > 2000000000ull) __trap();
      }
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------ async copies
// 16-byte cp.async (LDGSTS) with zero-fill when src_bytes == 0.
__device__ __forceinline__ void cp_async16(uint32_t dst_smem, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(src_bytes)
               : "memory");
}
// Arrive on `bar` once all cp.async issued so far by this thread have landed (counts as one expected arrival).
__device__ __forceinline__ void cp_async_arrive_noinc(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
// generic-proxy writes -> visible to the async proxy (wgmma / TMA reads of shared memory)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// the same for generic-proxy writes to global memory that a later TMA load reads
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// Bulk async copy global -> shared through the TMA engine (SASS: UBLKCP), completion on an mbarrier.
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// TMA tensor loads (global -> shared, box and swizzle given by the CUtensorMap at `tmap`), completion on an mbarrier.
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* tmap, int c0, int c1, int c2, int c3, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// TMA tensor store (shared -> global) into this thread's bulk group; tma_store_commit closes the group, and
// tma_store_wait_read<N> / tma_store_wait<N> wait until at most N groups still read shared memory / are incomplete.
__device__ __forceinline__ void tma_store_2d(const void* tmap, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(tmap), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const void* tmap, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(tmap), "r"(src),
               "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// The 1024-byte aligned base of the dynamic shared memory (128B-swizzled TMA / wgmma tiles need that alignment).
// Launches reserve 1024 bytes of slack for it.
__device__ __forceinline__ uint8_t* dyn_smem_1024() {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  return smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
}

// ------------------------------------------------------------------ wgmma (warpgroup MMA, accumulators in registers)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from touching accumulator registers across a wgmma_wait
template <int N>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Accumulator fragment of m64nNk16 (fp32): register i of thread t of the warpgroup holds
//   row 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2),  column 8 * (i / 4) + 2 * (t % 4) + i % 2.

// Shared-memory matrix descriptor (wgmma), 128-byte swizzle (16-byte chunk index XOR address bits 7-9), so a view
// that starts at any 128-byte row of a swizzled tile reads what TMA / the producers wrote there.
// K-major tile: rows of 64 fp16 (128 B); `sbo` = bytes between 8-row groups (1024 for a dense tile).
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);       // start address, 16-byte units
  d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;        // leading byte offset
  d |= (uint64_t)((sbo >> 4) & 0x3FFF) << 32;        // stride byte offset
  d |= (uint64_t)1 << 62;                            // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ uint64_t gmma_desc_sw128_kmajor(uint32_t smem_addr, uint32_t sbo = 1024) {
  return gmma_desc_sw128(smem_addr, 16, sbo);        // LBO unused for swizzled K-major
}
// MN-major B operand ([K rows][64 N-elements] panels of 128-byte rows, e.g. V[key][d] for P.V):
// 8-row K groups are 1024 B apart (SBO), consecutive 64-element N panels are `panel_bytes` apart (LBO).
__device__ __forceinline__ uint64_t gmma_desc_sw128_mnmajor(uint32_t smem_addr, uint32_t panel_bytes) {
  return gmma_desc_sw128(smem_addr, panel_bytes, 1024);
}

// warpgroup-wide register reallocation (all threads of the warpgroup execute it)
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// named barrier over `n` threads (multiple of 32)
__device__ __forceinline__ void named_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// true on exactly one lane of the (converged) warp
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "elect.sync _|p, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// x rounded to tf32 (10 explicit mantissa bits, nearest, ties away): the hi half of a split-tf32 pair (conv_igemm.cuh);
// the lo half x - hi is exact in fp32
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

// fp32-accurate forms for the fp32 RAFT path.  The library is built with --use_fast_math, which turns tanhf into
// tanh.approx.f32 (MUFU.TANH, relative error ~2^-11) and expf into ex2.approx of a rounded x*log2(e) (relative error
// growing with |x|); these stay within a few fp32 ulp.  No IEEE-division slow paths: tanh_acc sits in the conv
// epilogues.  (sigmoidf_ needs no such form: the error of its rounded x*log2(e) is of the order of the fp32 rounding of
// x itself, and the split GRU z|r epilogue measures as accurate as torch's fp32 sigmoid.)
// 1 / d for 1 <= d < 2^126 (finite: at d = inf the Newton step gives NaN): rcp.approx + one Newton step
__device__ __forceinline__ float rcp_acc(float d) {
  const float r = __fdividef(1.f, d);
  return fmaf(fmaf(-d, r, 1.f), r, r);
}
// exp(x): the product x*log2(e) is carried to ~2^-48 (fma residual), only ex2.approx's own ~2 ulp remain
__device__ __forceinline__ float exp_acc(float x) {
  const float t = x * 1.44269502f;
  const float r = fmaf(x, 1.44269502f, -t) + x * 1.92596303e-8f;   // x*log2(e) - t
  return exp2f(t) * fmaf(r, 0.693147181f, 1.f);
}
// tanh|x| = expm1(2|x|) / (expm1(2|x|) + 2): no cancellation near 0 (expm1f is not affected by --use_fast_math);
// tanh(9) rounds to 1 in fp32 (above 9 the quotient, NaN from d = inf, is not selected)
__device__ __forceinline__ float tanh_acc(float x) {
  const float a = fabsf(x);
  const float e = expm1f(2.f * a), d = e + 2.f;
  float q = e * rcp_acc(d);
  q = fmaf(fmaf(-q, d, e), rcp_acc(d), q);     // one residual correction of the quotient
  return copysignf(a > 9.f ? 1.f : q, x);
}

}  // namespace ppx

#endif  // __CUDACC__

// wgmma implicit-GEMM convolution for sm_90a.  See conv_igemm.cuh for the contract.
//
// Persistent CTA (one per SM, 384 threads) looping over 128 x BN output tiles:
//   warpgroups 0-1  consumers: warpgroup w issues wgmma (M=64 rows 64w.., N=BN, K=16 x4 per 64-wide K chunk) into
//                   register accumulators, then runs the fused epilogue of its 64 rows (conv_epilogue.cuh)
//   warpgroup 2     im2col producers: 16-byte cp.async gathers into a 128B-swizzled K-major A tile; thread 0 also
//                   streams the pre-swizzled weight tile with a single cp.async.bulk (TMA engine) per stage
// Pipeline: `stages` smem slots (full/empty mbarriers) that keep filling across tile boundaries, so the producers run
// ahead through the consumers' epilogue.
// conv_igemm_tf32_kernel is the split-tf32 form (PPConvParams::split): the same body with tf32 MMAs (k8 per 32-byte
// k-step instead of k16) and the split epilogue.
// The file also holds pp_launch_conv, which picks the kernel of every convolution, and the host plumbing that the
// halo and GEMM kernels share with this one (SM count, tensor maps).
#include <stdlib.h>

#include "conv_igemm.cuh"
#include "conv_epilogue.cuh"

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KiB
constexpr int NUM_CONSUMERS = 256;  // warpgroups 0-1
constexpr int NUM_PRODUCERS = 128;  // warpgroup 2
constexpr int NUM_THREADS = 384;
constexpr int MAX_STAGES = 8;
constexpr int SMEM_BUDGET = 192 * 1024;

template <int BN, bool TF32>
__device__ __forceinline__ void igemm_consume(const PPConvParams& p, uint8_t* smem, int stage_bytes, uint64_t* full_bar,
                                              uint64_t* empty_bar, float* stg, int wg, int t128) {
  using namespace ppx;
  const int S = p.stages;
  const int num_kc = p.num_kc;
  const int m_tiles = (p.M_total + BM - 1) / BM;
  const int n_tiles = p.Cout_g_pad / p.BN;
  const int total_tiles = m_tiles * n_tiles * p.groups;
  float acc[BN / 2];
  int s = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int n_idx = tile % n_tiles;
    const int rest = tile / n_tiles;
    const int m0 = (rest % m_tiles) * BM;
    const int g = rest / m_tiles;
    const int n0 = n_idx * p.BN;
    int prev = -1;
    for (int kc = 0; kc < num_kc; ++kc) {
      mbar_wait(&full_bar[s], phase);
      fence_proxy_async();   // the A tile was written by cp.async (generic proxy)
      wgmma_fence();
      const uint32_t a_addr = smem_u32(smem + s * stage_bytes);
      const uint64_t adesc = gmma_desc_sw128_kmajor(a_addr + wg * (A_STAGE_BYTES / 2));
      const uint64_t bdesc = gmma_desc_sw128_kmajor(a_addr + A_STAGE_BYTES);
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        if constexpr (TF32) wgmma_tf32<BN>(acc, adesc + 2 * k, bdesc + 2 * k, (kc | k) != 0 ? 1u : 0u);
        else wgmma_f16<BN>(acc, adesc + 2 * k, bdesc + 2 * k, (kc | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();   // the previous chunk's MMAs are done: its slot may be refilled
      if (prev >= 0) mbar_arrive(&empty_bar[prev]);
      prev = s;
      if (++s == S) { s = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    mbar_arrive(&empty_bar[prev]);
    ppconv::drain_acc<BN>(acc, stg, t128, 4 + wg, [&](const float* src, int r, int c) {
      const int m = m0 + wg * 64 + r;
      if (m < p.M_total && n0 + c < p.Cout_g)
        ppconv::epilogue_from_stage<TF32>(p, src, m, g, n0 + c);
    });
  }
}

template <bool TF32>
__device__ __forceinline__ void igemm_body(const PPConvParams& p) {
  using namespace ppx;
  uint8_t* smem = dyn_smem_1024();

  const int S = p.stages;
  const int b_stage_bytes = p.BN * 128;
  const int stage_bytes = A_STAGE_BYTES + b_stage_bytes;
  float* stg = reinterpret_cast<float*>(smem + S * stage_bytes);     // 2 x STG_BYTES accumulator staging
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S * stage_bytes + 2 * ppconv::STG_BYTES);
  uint64_t* empty_bar = full_bar + MAX_STAGES;

  const int tid = threadIdx.x;
  const int num_kc = p.num_kc;
  const int m_tiles = (p.M_total + BM - 1) / BM;
  const int n_tiles = p.Cout_g_pad / p.BN;
  const int total_tiles = m_tiles * n_tiles * p.groups;

  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], NUM_PRODUCERS + 1);
      mbar_init(&empty_bar[s], NUM_CONSUMERS);
    }
    mbar_fence_init();
  }
  __syncthreads();
  // Programmatic dependent launch: everything above (barrier init) overlapped the tail of the previous kernel in the
  // stream; from here on we read its outputs.  Let our own dependents start their prologue.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  // 168 registers per thread at launch; the producers give theirs to the accumulator-holding consumers.  An increase
  // can only use what this CTA's warpgroups released: 2 x 128 x (216 - 168) <= 128 x (168 - 64).
  if (tid < NUM_CONSUMERS) {
    setmaxnreg_inc<216>();
    const int wg = tid >> 7;
    ppconv::with_tile_width<256>(p.BN, [&](auto bn) {
      igemm_consume<decltype(bn)::value, TF32>(p, smem, stage_bytes, full_bar, empty_bar, stg + wg * (ppconv::STG_BYTES / 4), wg,
                                         tid & 127);
    });
  } else {
    // ------------------------------------------------------------------ im2col producers (+ weight tile loader)
    setmaxnreg_dec<64>();
    const int ptid = tid - NUM_CONSUMERS;
    const int j = ptid & 7;    // 16-byte chunk inside the 128-byte K row
    const int rb = ptid >> 3;  // rows rb, rb+16, ..., rb+112
    const uint32_t a_off = rb * 128 + ((j ^ (rb & 7)) << 4);
    int s = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int n0 = (tile % n_tiles) * p.BN;
      const int rest = tile / n_tiles;
      const int m0 = (rest % m_tiles) * BM;
      const int g = rest / m_tiles;
      const __half* wsrc = p.wpacked + ((long long)g * num_kc * p.Cout_g_pad + n0) * BK;
      int rpix[8], riy[8], rix[8];
      uint32_t rvalid = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int m = m0 + rb + 16 * i;
        if (m < p.M_total) {
          const int ox = m % p.OW;
          const int t = m / p.OW;
          const int oy = t % p.OH;
          const int img = t / p.OH;
          rpix[i] = img * p.H * p.W;
          riy[i] = oy * p.sh - p.ph;
          rix[i] = ox * p.sw - p.pw;
          rvalid |= 1u << i;
        } else {
          rpix[i] = 0; riy[i] = 0; rix[i] = 0;
        }
      }
      // this thread's position inside the K range: channel ci of tap (ky, kx); advances by 64 per chunk
      int k = j * 8;
      int tap0 = k / p.Cin;
      int ci = k - tap0 * p.Cin;
      int ky = tap0 / p.kw;
      int kx = tap0 - ky * p.kw;
      for (int kc = 0; kc < num_kc; ++kc) {
        mbar_wait(&empty_bar[s], phase ^ 1);
        if (ptid == 0) {
          mbar_arrive_expect_tx(&full_bar[s], (uint32_t)b_stage_bytes);
          bulk_g2s(smem_u32(smem + s * stage_bytes + A_STAGE_BYTES), wsrc + (long long)kc * p.Cout_g_pad * BK,
                   (uint32_t)b_stage_bytes, &full_bar[s]);
        }
        const bool kvalid = k < p.K_total;
        const int q = pp_seg_of(p, ci);
        const __half* sbase = p.seg[q].ptr + p.seg[q].coff + g * p.seg[q].gstep + (ci - p.seg[q].cbegin);
        const long long cs = p.seg[q].cstride;
        const int dy = ky * p.dh, dx = kx * p.dw;
        const uint32_t a_dst = smem_u32(smem + s * stage_bytes) + a_off;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          int iy = riy[i] + dy, ix = rix[i] + dx;
          bool v = kvalid && ((rvalid >> i) & 1u);
          if (p.pad_replicate) {
            iy = min(max(iy, 0), p.H - 1);
            ix = min(max(ix, 0), p.W - 1);
          } else {
            v = v && ((unsigned)iy < (unsigned)p.H) && ((unsigned)ix < (unsigned)p.W);
          }
          const __half* src = v ? sbase + (long long)(rpix[i] + iy * p.W + ix) * cs : p.seg[0].ptr;
          cp_async16(a_dst + i * (16 * 128), src, v ? 16u : 0u);
        }
        k += BK;
        ci += BK;
        while (ci >= p.Cin) {
          ci -= p.Cin;
          if (++kx == p.kw) { kx = 0; ++ky; }
        }
        // asynchronous arrival: fires when this thread's copies for the stage have landed, so up to `stages`
        // K chunks (across tile boundaries) are in flight without any wait in the producer loop
        cp_async_arrive_noinc(&full_bar[s]);
        if (++s == S) { s = 0; phase ^= 1; }
      }
    }
  }
}

__global__ void __launch_bounds__(NUM_THREADS, 1) conv_igemm_kernel(const __grid_constant__ PPConvParams p) {
  igemm_body<false>(p);
}

__global__ void __launch_bounds__(NUM_THREADS, 1) conv_igemm_tf32_kernel(const __grid_constant__ PPConvParams p) {
  igemm_body<true>(p);
}

}  // namespace

namespace {
thread_local PPConvPlan g_last_plan = {'?', 0, 0, 0, 0, 0, 0, 0};
}
PPConvPlan& pp_last_conv_plan() { return g_last_plan; }

int pp_launch_conv(const PPConvParams& pin, cudaStream_t stream) {
  PPConvParams p = pin;
  PP_REQUIRE(p.BN >= 16 && p.BN <= 256 && p.BN % 16 == 0, "conv: BN=%d must be a multiple of 16 in [16,256]", p.BN);
  PP_REQUIRE(p.Cout_g_pad % p.BN == 0, "conv: Cout_g_pad=%d not a multiple of BN=%d", p.Cout_g_pad, p.BN);
  PP_REQUIRE(p.Cin % 8 == 0, "conv: Cin=%d must be a multiple of 8", p.Cin);
  PP_REQUIRE(p.nseg >= 1 && p.nseg <= PP_MAX_SEGS, "conv: nseg=%d", p.nseg);
  PP_REQUIRE(p.seg[p.nseg - 1].cend == p.Cin && p.seg[0].cbegin == 0, "conv: segments do not cover Cin=%d", p.Cin);
  for (int i = 0; i < p.nseg; ++i) {
    PP_REQUIRE(p.seg[i].cstride % 8 == 0 && p.seg[i].coff % 8 == 0 && p.seg[i].gstep % 8 == 0 &&
                   p.seg[i].cbegin % 8 == 0 && p.seg[i].cend % 8 == 0,
               "conv: segment %d is not 16-byte aligned (cstride=%d coff=%d)", i, p.seg[i].cstride, p.seg[i].coff);
    PP_REQUIRE((reinterpret_cast<uintptr_t>(p.seg[i].ptr) & 15) == 0, "conv: segment %d pointer misaligned", i);
  }
  PP_REQUIRE((reinterpret_cast<uintptr_t>(p.wpacked) & 15) == 0, "conv: weight pointer misaligned");
  p.K_total = p.kh * p.kw * p.Cin;
  p.num_kc = pp_ceil_div(p.K_total, BK);
  p.M_total = p.N * p.OH * p.OW;
  if (p.M_total <= 0) return PP_OK;
  if (p.split) {
    // every epilogue tensor is fp32: 16-byte runs need 4-float aligned pointers, strides, offsets and hi -> lo distances
    auto al = [](const void* ptr, long long cs, long long co, long long gs, long long lo) {
      return ptr == nullptr || ((reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && cs % 4 == 0 && co % 4 == 0 && gs % 4 == 0 &&
                                lo % 4 == 0);
    };
    bool ok = al(p.out, p.out_cstride, p.out_coff, p.out_gstep, p.out_fp32 ? 0 : p.out_lo) &&
              al(p.aux0, p.aux0_cstride, p.aux0_coff, 0, p.aux0_lo) && al(p.aux1, p.aux1_cstride, p.aux1_coff, 0, p.aux1_lo) &&
              al(p.out2, p.out2_cstride, p.out2_coff, 0, p.out2_lo);
    if (p.epi == PP_EPI_GRU_ZR) ok = ok && ((p.Cout_g >> 1) % 16 == 0);
    p.vec_ok = ok ? 1 : 0;
  } else {
    const int esz = p.out_fp32 ? 4 : 2, per16 = 16 / esz;
    auto al = [](const void* ptr, long long cs, long long co, long long gs, int per) {
      return ptr == nullptr || ((reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && cs % per == 0 && co % per == 0 && gs % per == 0);
    };
    bool ok = al(p.out, p.out_cstride, p.out_coff, p.out_gstep, per16) && al(p.aux0, p.aux0_cstride, p.aux0_coff, 0, 8) &&
              al(p.aux1, p.aux1_cstride, p.aux1_coff, 0, 8) && al(p.out2, p.out2_cstride, p.out2_coff, 0, 8);
    if (p.bias != nullptr) ok = ok && (reinterpret_cast<uintptr_t>(p.bias) & 15) == 0 && (p.groups == 1 || p.Cout_g % 4 == 0);
    if (p.epi == PP_EPI_GRU_ZR) ok = ok && ((p.Cout_g >> 1) % 16 == 0);
    p.vec_ok = ok ? 1 : 0;
  }
  g_last_plan = PPConvPlan{'?', 0, 0, 0, 0, 0, 0, 0};
  if (pp_prog_recording()) {
    PP_REQUIRE(!p.split, "conv program: split-tf32 layers are not supported");
    g_last_plan.kind = 'p';
    return pp_prog_record_conv(p);
  }
  if (pp_conv_gemm_eligible(p)) return pp_launch_conv_gemm(p, stream);   // both launchers record their plan
  if (pp_conv_halo_eligible(p)) return pp_launch_conv_halo(p, stream);
  for (int i = 0; i < p.nseg; ++i)
    PP_REQUIRE(p.seg[i].cvalid == 0, "conv: zero-extended input channels (cvalid=%d of %d) need the TMA halo kernel "
               "(stride 1, zero padding, Cin %% 64 == 0)", p.seg[i].cvalid, p.seg[i].cend - p.seg[i].cbegin);   // stride-1 k>1 layers: TMA halo-tile kernel
  const int stage_bytes = A_STAGE_BYTES + p.BN * 128;
  int stages = SMEM_BUDGET / stage_bytes;
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  p.stages = stages;
  g_last_plan = PPConvPlan{'i', 0, p.BN, 0, 0, 0, stages, stages};
  const size_t smem = (size_t)stages * stage_bytes + 2 * ppconv::STG_BYTES + 1024 + 256;
  static bool smem_limit_set = false;
  if (!smem_limit_set) {
    PP_CUDA_CHECK(cudaFuncSetAttribute(conv_igemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    PP_CUDA_CHECK(cudaFuncSetAttribute(conv_igemm_tf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    smem_limit_set = true;
  }
  int num_sms = 0;
  PP_TRY(pp_num_sms(&num_sms));
  const long long total_tiles = (long long)pp_ceil_div(p.M_total, BM) * (p.Cout_g_pad / p.BN) * p.groups;
  PP_REQUIRE(total_tiles < (1LL << 31), "conv: too many tiles");
  const int grid = (int)(total_tiles < num_sms ? total_tiles : num_sms);
  return pp_conv_launch(p.split ? conv_igemm_tf32_kernel : conv_igemm_kernel, p, grid, NUM_THREADS, smem, stream);
}

// ---- host plumbing shared with conv_halo.cu and conv_gemm.cu ----------------------------------------------------------
int pp_num_sms(int* n) {
  static int num_sms = 0;
  if (num_sms == 0) {
    int dev = 0, v = 0;
    PP_CUDA_CHECK(cudaGetDevice(&dev));
    PP_CUDA_CHECK(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev));
    num_sms = v;
  }
  *n = num_sms;
  return PP_OK;
}

int pp_conv_noepi() {
  const char* e = getenv("PP_CONV_NOEPI");
  return (e != nullptr && atoi(e) != 0) ? 1 : 0;
}

namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    cudaDriverEntryPointQueryResult qr;
    void* ptr = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

}  // namespace

bool pp_tmap_supported() { return encode_fn() != nullptr; }

int pp_conv_input_tmaps(const PPConvParams& p, int bw, int bh, bool flat, CUtensorMap* maps) {
  EncodeTiledFn enc = encode_fn();
  PP_REQUIRE(enc != nullptr, "conv: cuTensorMapEncodeTiled is not available");
  for (int i = 0; i < p.nseg; ++i) {
    const PPConvSeg& s = p.seg[i];
    const cuuint64_t cacc = (cuuint64_t)(p.groups - 1) * s.gstep + (s.cvalid > 0 ? s.cvalid : s.cend - s.cbegin);
    cuuint64_t dims[4] = {cacc, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.N};
    cuuint64_t strides[3] = {(cuuint64_t)s.cstride * 2, (cuuint64_t)p.W * s.cstride * 2, (cuuint64_t)p.H * p.W * s.cstride * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)bw, (cuuint32_t)bh, 1};
    if (flat) {   // pixels as one flat dimension; the last tile's tail is out of bounds -> zero-filled
      dims[1] = (cuuint64_t)p.M_total; dims[2] = 1; dims[3] = 1;
      strides[1] = strides[2] = (cuuint64_t)p.M_total * s.cstride * 2;
    }
    cuuint32_t es[4] = {1, 1, 1, 1};
    const CUresult r = enc(&maps[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<__half*>(s.ptr + s.coff), dims, strides, box,
                           es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PP_REQUIRE(r == CUDA_SUCCESS, "conv: cuTensorMapEncodeTiled failed (%d) for segment %d (cstride=%d W=%d H=%d N=%d)",
               (int)r, i, s.cstride, p.W, p.H, p.N);
  }
  return PP_OK;
}

int pp_tmap_2d_f16(CUtensorMap* map, const __half* base, int cols, long long rows, int ld, int box_rows) {
  EncodeTiledFn enc = encode_fn();
  PP_REQUIRE(enc != nullptr, "conv: cuTensorMapEncodeTiled is not available");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t es[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  PP_REQUIRE(r == CUDA_SUCCESS, "conv: cuTensorMapEncodeTiled (2-D, %d x %lld, ld %d) failed (%d)", cols, rows, ld, (int)r);
  return PP_OK;
}

int pp_tmap_pixels_f16(CUtensorMap* map, const __half* base, int cols, int cstride, long long w, int h, int n, int box_c,
                       int box_w, int box_h) {
  EncodeTiledFn enc = encode_fn();
  PP_REQUIRE(enc != nullptr, "conv: cuTensorMapEncodeTiled is not available");
  const cuuint64_t pix = (cuuint64_t)cstride * 2;
  cuuint64_t dims[4] = {(cuuint64_t)cols, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  cuuint64_t strides[3] = {pix, (cuuint64_t)w * pix, (cuuint64_t)w * h * pix};
  cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  const CUtensorMapSwizzle swz = box_c == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : box_c == 32 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                                                        : CU_TENSOR_MAP_SWIZZLE_32B;
  PP_REQUIRE(box_c == 64 || box_c == 32 || box_c == 16, "conv: pixel tensor map box of %d channels", box_c);
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<__half*>(base), dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  PP_REQUIRE(r == CUDA_SUCCESS, "conv: cuTensorMapEncodeTiled (%d ch x %lld x %d x %d, cstride %d) failed (%d)", cols, w, h, n,
             cstride, (int)r);
  return PP_OK;
}

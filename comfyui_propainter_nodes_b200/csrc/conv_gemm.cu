// Wide-tile wgmma GEMM for the flat layers (1x1 convolutions and linear layers) on sm_90a:
//   out[M x Cout] = epilogue( A[M x Cin] * W[Cout x Cin]^T ),  A = the flattened N*H*W pixels of the input segments.
//
// The halo kernel's flat mode runs these with 256 x <=128 tiles and drains the accumulators through a shared-memory
// staging tile 32 columns at a time (two named barriers per chunk, 32-byte per-thread global stores); the tensor cores
// idle meanwhile.  Here:
//   * tiles are 128 x 256 (MB = 1: each consumer warpgroup owns 64 rows x 256 columns, wgmma m64n256k16) or, for layers
//     with Cout <= 128, 256 x 128 (MB = 2: two m64 blocks of 128 columns), 128 accumulator registers per thread either
//     way.  Per 64-channel K chunk a stage holds the A rows (one 2-D TMA box per segment view, zero-filled past M and
//     past the last segment's channels) and the pre-swizzled weight tile (cp.async.bulk), 48 KB in both shapes.
//   * the epilogue runs on the wgmma fragments (ppconv::frag_epilogue, shared with conv_halo_kernel's TMA path): bias,
//     act1, scale, residual, act2 in the order of conv_epilogue16's PP_EPI_STD branch, fp16 into a 128B-swizzled
//     staging tile of 64-channel panels that span both warpgroups' rows, from which one thread per warpgroup issues TMA
//     stores (rows / columns past the tensor are clipped).  The stores drain while the next tile's main loop runs; the staging
//     tile is only waited for (cp.async.bulk.wait_group.read) before it is written again.  A residual tile (the in-place
//     transformer proj) is TMA-loaded into the staging tile, read and overwritten in place by the same threads.
//     The tile's bias columns are copied to shared memory once per tile and act1 is a compile-time case, so the loop
//     over the fragments is straight-line code: with a global bias load per fragment column and a runtime activation
//     switch it took ~9.5 us of a 128 x 256 tile (measured on H100), more than the tile's main loop.
//   * the stage ring keeps running across tiles, so the producer loads the next tile during the epilogue.  Tiles are
//     ordered N-fastest: the CTAs in flight share their A rows in L2.
// Warp roles (384 threads, one persistent CTA per SM): warpgroups 0-1 consumers, warp 8 producer (one elected thread
// issues both loads of a stage), warps 9-11 idle (setmaxnreg works per warpgroup).
#include <string.h>

#include "conv_epilogue.cuh"
#include "conv_igemm.cuh"

namespace {

constexpr int NUM_THREADS = 384;
constexpr int NUM_CONSUMERS = 256;
constexpr int WARP_PRODUCER = 8;
constexpr int STAGE_BYTES = 48 * 1024;        // A [128*MB rows][128 B] + B [256/MB rows][128 B]
constexpr int STAGES = 3;
constexpr int OUT_BYTES = 64 * 1024;          // fp16 staging tile [256/MB / 64 panels][128*MB rows][128 B]
constexpr int BIAS_BYTES = 2 * 256 * 4;       // the tile's bias columns, one copy per consumer warpgroup
constexpr int SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + OUT_BYTES + 1024 + BIAS_BYTES;   // alignment slack, barriers

struct GemmParams {
  PPConvParams c;
  CUtensorMap tmap_a[PP_MAX_SEGS];
  CUtensorMap tmap_out;   // [M][Cout] at out + out_coff, boxes of 64 columns x 64*MB rows (one warpgroup's rows)
  CUtensorMap tmap_res;   // the same for the residual (aux0), when there is one
  int m_tiles, n_tiles, chunks;
  int debug;              // bit 0: skip the epilogue math/stores (PP_CONV_NOEPI=1, mainloop-only timing experiments)
};

struct Smem {
  uint8_t* stages;
  uint8_t* out;
  uint64_t *full, *empty, *res;   // res: one barrier per consumer warpgroup
  float* bias;                    // [2][256]
};
__device__ __forceinline__ Smem gemm_smem() {
  uint8_t* base = ppx::dyn_smem_1024();
  Smem m;
  m.stages = base;
  m.out = base + STAGES * STAGE_BYTES;
  m.full = reinterpret_cast<uint64_t*>(m.out + OUT_BYTES);
  m.empty = m.full + STAGES;
  m.res = m.empty + STAGES;
  m.bias = reinterpret_cast<float*>(m.out + OUT_BYTES + 1024);
  return m;
}

// One tile of one consumer warpgroup: main loop into acc[MB][BN / 2], then the fragment epilogue into the staging tile
// and this warpgroup's TMA stores.  The ring position (s, ph) runs on across tiles.
template <int MB, int BN>
__device__ __forceinline__ void gemm_tile(const GemmParams& h, const Smem& m, int tile, int& s, uint32_t& ph, uint32_t& rph,
                                          int wg, int t128) {
  using namespace ppx;
  const PPConvParams& p = h.c;
  constexpr int A_BYTES = 128 * MB * 128;
  constexpr int WG_ROWS = 64 * MB;
  constexpr int PANEL = 128 * MB * 128;        // one 64-column panel of the staging tile
  const int n0 = (tile % h.n_tiles) * BN;
  const int m0 = (tile / h.n_tiles) * (128 * MB);
  float acc[MB][BN / 2];
  int prev = -1;
  for (int c = 0; c < h.chunks; ++c) {
    mbar_wait(&m.full[s], ph);
    const uint32_t a = smem_u32(m.stages + s * STAGE_BYTES);
    uint64_t adesc[MB];
#pragma unroll
    for (int b = 0; b < MB; ++b) adesc[b] = gmma_desc_sw128_kmajor(a + (wg * MB + b) * 64 * 128);
    const uint64_t bdesc = gmma_desc_sw128_kmajor(a + A_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int b = 0; b < MB; ++b) wgmma_f16<BN>(acc[b], adesc[b] + 2 * k, bdesc + 2 * k, (c | k) != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0) mbar_arrive(&m.empty[prev]);
    prev = s;
    if (++s == STAGES) { s = 0; ph ^= 1; }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int b = 0; b < MB; ++b) wgmma_fence_acc(acc[b]);
  mbar_arrive(&m.empty[prev]);
  if (h.debug & 1) return;

  // ---- epilogue: this warpgroup's rows [wg * WG_ROWS, +WG_ROWS) of every panel of the staging tile
  const int bar_id = 2 + wg, row0 = m0 + wg * WG_ROWS;
  const int npanel = (min(BN, p.Cout_g - n0) + 63) / 64;
  uint8_t* so = m.out + wg * WG_ROWS * 128;
  const bool issuer = t128 == 0;
  // the tile's bias columns; the previous tile's readers of this copy have passed its last named barrier
  float* bs = m.bias + wg * 256;
  ppconv::stage_bias<BN>(p, bs, 0, n0, t128);
  if (issuer) tma_store_wait_read<0>();   // the previous tile's stores have read it
  named_bar(bar_id, 128);
  const bool has_res = p.aux0 != nullptr;
  if (has_res) {
    if (issuer) {
      mbar_arrive_expect_tx(&m.res[wg], (uint32_t)(npanel * WG_ROWS * 128));
      for (int pnl = 0; pnl < npanel; ++pnl) tma_load_2d(smem_u32(so + pnl * PANEL), &h.tmap_res, n0 + pnl * 64, row0, &m.res[wg]);
    }
    mbar_wait(&m.res[wg], rph);
    rph ^= 1;
  }
  // 64-channel panels of all the tile's rows (both warpgroups')
  auto epilogue = [&](auto act1) {
    ppconv::frag_epilogue<MB, BN, 64, PANEL, PP_EPI_STD, decltype(act1)::value>(p, acc, so, nullptr, bs, has_res, false, 0,
                                                                                t128);
  };
  switch (p.act1) {
    case PP_ACT_RELU: epilogue(ppconv::IntC<PP_ACT_RELU>{}); break;
    case PP_ACT_LRELU: epilogue(ppconv::IntC<PP_ACT_LRELU>{}); break;
    case PP_ACT_SIGMOID: epilogue(ppconv::IntC<PP_ACT_SIGMOID>{}); break;
    case PP_ACT_TANH: epilogue(ppconv::IntC<PP_ACT_TANH>{}); break;
    case PP_ACT_GELU: epilogue(ppconv::IntC<PP_ACT_GELU>{}); break;
    default: epilogue(ppconv::IntC<PP_ACT_NONE>{}); break;
  }
  fence_proxy_async();           // generic-proxy smem writes -> visible to the TMA store
  named_bar(bar_id, 128);
  if (issuer) {
    for (int pnl = 0; pnl < npanel; ++pnl) tma_store_2d(&h.tmap_out, smem_u32(so + pnl * PANEL), n0 + pnl * 64, row0);
    tma_store_commit();
  }
}

template <int MB>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_gemm_kernel(const __grid_constant__ GemmParams h) {
  using namespace ppx;
  constexpr int BN = 256 / MB;
  constexpr int A_BYTES = 128 * MB * 128;
  const Smem m = gemm_smem();
  const PPConvParams& p = h.c;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int total_tiles = h.m_tiles * h.n_tiles;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&m.full[s], 1); mbar_init(&m.empty[s], NUM_CONSUMERS); }
    mbar_init(&m.res[0], 1);
    mbar_init(&m.res[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  // as in the halo kernel: the producer warpgroup gives its registers to the accumulator holders
  if (warp < 8) setmaxnreg_inc<232>();
  else setmaxnreg_dec<40>();
  if (warp < 8) {
    const int wg = tid >> 7, t128 = tid & 127;
    int s = 0;
    uint32_t ph = 0, rph = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) gemm_tile<MB, BN>(h, m, tile, s, ph, rph, wg, t128);
    if (t128 == 0) tma_store_wait<0>();   // this warpgroup's stores complete
  } else if (warp == WARP_PRODUCER) {
    if (elect_one()) {
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n0 = (tile % h.n_tiles) * BN;
        const int m0 = (tile / h.n_tiles) * (128 * MB);
        // columns >= bnt of the last N tile keep stale weights: computed, never stored
        const uint32_t b_bytes = (uint32_t)(min(BN, p.Cout_g_pad - n0) * 128);
        for (int c = 0; c < h.chunks; ++c) {
          const int ci = c * 64;
          const int q = pp_seg_of(p, ci);
          mbar_wait(&m.empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&m.full[s], (uint32_t)A_BYTES + b_bytes);
          const uint32_t dst = smem_u32(m.stages + s * STAGE_BYTES);
          tma_load_4d(dst, &h.tmap_a[q], ci - p.seg[q].cbegin, m0, 0, 0, &m.full[s]);
          bulk_g2s(dst + A_BYTES, p.wpacked + ((long long)c * p.Cout_g_pad + n0) * 64, b_bytes, &m.full[s]);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  }
}

// MB (m64 blocks per consumer warpgroup) of a layer: 256 x 128 tiles when all output channels fit one 128-wide tile
int gemm_mb(const PPConvParams& p) { return p.Cout_g_pad <= 128 && p.M_total >= 256 ? 2 : 1; }

long long gemm_tiles(const PPConvParams& p, int mb) {
  return pp_ceil_div64(p.M_total, 128 * mb) * pp_ceil_div(p.Cout_g_pad, 256 / mb);
}

}  // namespace

int pp_conv_gemm_eligible(const PPConvParams& p) {
  if (p.kh != 1 || p.kw != 1 || p.sh != 1 || p.sw != 1 || p.ph != 0 || p.pw != 0 || p.pad_replicate) return 0;
  if (p.groups != 1 || p.split || p.epi != PP_EPI_STD || p.out_fp32 || p.M_total < 128) return 0;
  if (!pp_conv_segs_chunked(p, true)) return 0;
  // TMA stores (and residual loads): 16-byte aligned rows
  if (!aligned16(p.out, p.out_cstride, p.out_coff)) return 0;
  // TMA stores clip the channel dimension at 16-byte granularity (measured on H100: layers of 2, 10 and 126 channels
  // written into a wider tensor overwrote the channels up to the next multiple of 8), so a channel count that ends
  // inside a 16-byte unit would overwrite its neighbours; such layers run on the halo kernel's drain epilogue
  if (p.Cout_g % 8 != 0) return 0;
  if (p.aux0 != nullptr && !aligned16(p.aux0, p.aux0_cstride, p.aux0_coff)) return 0;
  if (p.bias != nullptr && (reinterpret_cast<uintptr_t>(p.bias) & 7) != 0) return 0;
  // launches of less than one wave keep the halo kernel, which narrows its tiles to fill the SMs
  int num_sms = 0;
  if (pp_num_sms(&num_sms) != PP_OK || gemm_tiles(p, gemm_mb(p)) < num_sms) return 0;
  return pp_tmap_supported() ? 1 : 0;
}

int pp_launch_conv_gemm(const PPConvParams& pin, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    PP_CUDA_CHECK(cudaFuncSetAttribute(conv_gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    PP_CUDA_CHECK(cudaFuncSetAttribute(conv_gemm_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    attr_set = true;
  }
  GemmParams h;
  memset(&h, 0, sizeof(h));
  h.c = pin;
  const PPConvParams& p = h.c;
  const int mb = gemm_mb(p);
  h.m_tiles = (int)pp_ceil_div64(p.M_total, 128 * mb);
  h.n_tiles = pp_ceil_div(p.Cout_g_pad, 256 / mb);
  h.chunks = pp_ceil_div(p.Cin, 64);
  PP_REQUIRE((long long)h.m_tiles * h.n_tiles < (1LL << 31), "conv_gemm: too many tiles");
  h.debug = pp_conv_noepi();
  PP_TRY(pp_conv_input_tmaps(p, 128 * mb, 1, true, h.tmap_a));
  PP_TRY(pp_tmap_2d_f16(&h.tmap_out, static_cast<const __half*>(p.out) + p.out_coff, p.Cout_g, p.M_total, p.out_cstride, 64 * mb));
  if (p.aux0 != nullptr)
    PP_TRY(pp_tmap_2d_f16(&h.tmap_res, p.aux0 + p.aux0_coff, p.Cout_g, p.M_total, p.aux0_cstride, 64 * mb));
  int num_sms = 0;
  PP_TRY(pp_num_sms(&num_sms));
  pp_last_conv_plan() = PPConvPlan{'g', mb, 256 / mb, 0, 1, 1, STAGES, STAGES};
  return pp_conv_launch(mb == 2 ? conv_gemm_kernel<2> : conv_gemm_kernel<1>, h, min(h.m_tiles * h.n_tiles, num_sms),
                        NUM_THREADS, SMEM_BYTES, stream);
}

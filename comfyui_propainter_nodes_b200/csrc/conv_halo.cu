// Halo-tile wgmma convolution for sm_90a: stride-1 convolutions whose A operand is fed by TMA.
//
// The implicit-GEMM kernel (conv_igemm.cu) fetches every input element once per filter tap (9x for a 3x3) with
// cp.async and streams the weight tile once per 128 output pixels; on the 3x3 / 1x5 / 5x1 layers with <= 256
// output channels that makes it L2->SM fill and instruction-issue bound.  Here one CTA tile is 16 rows x (8*MT)
// columns of output pixels (MT = 1 or 2 sub-tiles of 128 pixels):
//   * per 64-channel chunk, ONE 4-D TMA box load (cp.async.bulk.tensor, SWIZZLE_128B, out-of-image coordinates
//     zero-filled = the conv's zero padding) lands the input patch [(16+(kh-1)dh) x (8MT+(kw-1)dw)] pixels x 128 B
//     in shared memory; the A operand of filter tap (ky,kx) of sub-tile s is a *shifted view* of that patch:
//     wgmma descriptor start = patch + ((ky*dh)*BW + kx*dw + 8s)*128 B, stride between 8-pixel row groups
//     (SBO) = BW*128 B.  The 128B swizzle is a function of the absolute shared-memory address, so views that are
//     not 1024-byte aligned are consistent with what TMA wrote.
//   * the weight tile of (chunk, tap) [BN x 64] is streamed once per tile with cp.async.bulk and feeds both
//     sub-tiles, so weights move once per 256 output pixels.
// L2->SM bytes per output pixel drop ~3x on a 3x3 Cin=256 Cout=128 layer and no thread issues per-element loads.
//
// Warp roles (384 threads, one persistent CTA per SM): warpgroups 0-1 consumers (wgmma into register accumulators,
// then the fused epilogue of conv_epilogue.cuh -> global), warp 8 patch producer (TMA), warp 9 weight producer (bulk
// copy).  MT == 1: warpgroup w owns pixel rows 64w..64w+63 of the sub-tile; MT == 2: warpgroup w owns sub-tile w.
//
// Epilogue.  All three kernels share one main loop (halo_mainloop).  conv_halo_kernel runs the epilogue on the wgmma
// fragments where the layer's output can be TMA-stored (fp16, 16-byte aligned; halo_tma_configure): the tile's bias
// columns are copied to shared memory once, act1 is a compile-time case, the residual / GRU h / GRU z operands are
// TMA-loaded into shared memory while the tile's last wgmmas run, results go as fp16 into a swizzled staging tile
// (ppconv::frag_epilogue, shared with conv_gemm.cu) that one thread per warpgroup TMA-stores, and the stores drain under
// the next tile's main loop.  Every other layer, and the other two kernels, copy the accumulators through an fp32 staging
// tile 32 columns at a time into conv_epilogue16 (drain_acc), which loads its operands and stores per thread.  The
// shared-memory plan (halo_smem) is the same for both, with an epilogue region of the epilogue's size.
//
// conv_halo_tf32_kernel is the split-tf32 form (PPConvParams::split, see conv_igemm.cuh): the byte geometry is the same
// (a 128-byte swizzled K-chunk row holds 32 fp32 channels, each chunk is 4 wgmmas m64nNk8 with the same 32-byte
// descriptor step), so the tap views, rings and producers are shared; only the MMA instruction and the epilogue differ.
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include <memory>

#include "conv_epilogue.cuh"
#include "conv_igemm.cuh"
#include "dcn_sample.cuh"

namespace {

constexpr int NUM_THREADS = 384;   // warpgroup 2: warps 8-9 producers, 10-11 idle (setmaxnreg works per warpgroup)
constexpr int NUM_EPI_THREADS = 256;   // the two consumer warpgroups
constexpr int WARP_A = 8, WARP_B = 9;
constexpr int MAX_SA = 4, MAX_SB = 8;
// stages of the layers on the drain epilogue; the rest of the plan comes on top (halo_smem)
constexpr int SMEM_BUDGET = 186 * 1024;
constexpr int SMEM_MAX = 227 * 1024;   // dynamic shared memory of one CTA on sm_90
constexpr int SMEM_ALIGN_SLACK = 1024;   // dyn_smem_1024 moves the base up to a 1024-byte boundary
constexpr int BAR_BLOCK_BYTES = 1024;    // the barriers; keeps the epilogue region behind it 1024-byte aligned
constexpr int DRAIN_EPI_BYTES = 2 * ppconv::STG_BYTES;   // the drain epilogue's fp32 staging tile per consumer warpgroup

struct HaloLayer {
  PPConvParams c;
  CUtensorMap tmap[PP_MAX_SEGS];
  int MT;            // sub-tiles (128 pixels each) per CTA tile
  int BW, BH;        // patch size in pixels
  int tiles_x, tiles_y, n_tiles;
  int a_stage_bytes, b_stage_bytes, SA, SB;
  int tps;           // filter taps per weight stage: narrow N tiles pack several taps' [BN x 64] tiles into one stage, so
                     // the MMA issuer waits / commits once per group instead of once per tap (it is issue-bound there)
  int chunks;        // Cin / 64
  int flat;          // 1x1 convs: tiles are runs of 128*MT consecutive pixels of the flattened [N*H*W] pixel list
  int n_img;         // images the tile index decomposes over (1 in flat mode)
  int sub_bytes;     // A-view offset between the sub-tiles: 8 pixels (spatial) or 128 pixels (flat)
  int debug;         // bit 0: skip the epilogue math/stores (PP_CONV_NOEPI=1, mainloop-only timing experiments)
};

// A launch of conv_halo_kernel / conv_halo_tf32_kernel: the layer, and the tensor maps of the fp16 kernel's TMA-store
// epilogue (conv_prog_kernel's layers are HaloLayers: they keep the drain epilogue).
struct HaloParams : HaloLayer {
  int tma_out;       // 1: fragment epilogue + TMA stores (halo_tma_configure); 0: the fp32 staging drain of drain_acc
  CUtensorMap tm_out;    // out + out_coff (GRU_ZR: the z half), boxes of halo_panel_width(BN) channels x one
                         // warpgroup's pixels
  CUtensorMap tm_out2;   // GRU_ZR: out2 + out2_coff (r * h)
  CUtensorMap tm_aux0;   // the residual (STD) or h (GRU), loaded into the staging tile
  CUtensorMap tm_aux1;   // GRU_H: z, loaded one panel at a time into the z buffer
};

struct TileCoord {
  int n_idx, tx, ty, img, g;
};
__device__ __forceinline__ TileCoord decode_tile(const HaloLayer& h, int tile) {
  TileCoord t;
  t.n_idx = tile % h.n_tiles;
  int r = tile / h.n_tiles;
  t.tx = r % h.tiles_x; r /= h.tiles_x;
  t.ty = r % h.tiles_y; r /= h.tiles_y;
  t.img = r % h.n_img;
  t.g = r / h.n_img;
  return t;
}

__host__ __device__ inline int halo_total_tiles(const HaloLayer& h) {
  return h.n_tiles * h.tiles_x * h.tiles_y * h.n_img * h.c.groups;   // < 2^31, checked by halo_configure
}

// position in a shared-memory ring of stages
struct Ring {
  int s;
  uint32_t ph;
};

// Shared-memory carve-up of the halo kernels, from the 1024-byte aligned base:
//   SA patch stages | SB weight stages | barrier block | epilogue region of epi_bytes
// The region holds the drain's fp32 staging tiles (DRAIN_EPI_BYTES) or conv_halo_kernel's TMA epilogue
// (halo_tma_region_bytes).  The launchers call it with base == nullptr and read only `bytes`.
struct HaloSmem {
  uint8_t* a;                  // patch stages (TMA, 128B swizzle: 1024-byte aligned)
  uint8_t* b;                  // weight stages
  int SA, SB, a_stage_bytes, b_stage_bytes;
  uint64_t *a_full, *a_empty, *b_full, *b_empty;
  uint64_t* spare;             // one more barrier (conv_prog_kernel: layer_go)
  uint8_t* epi;                // the epilogue region
  int bytes;                   // dynamic shared memory, including the slack that aligns the base
};

__host__ __device__ inline HaloSmem halo_smem(uint8_t* base, int SA, int a_stage_bytes, int SB, int b_stage_bytes,
                                              int epi_bytes) {
  const int b_off = SA * a_stage_bytes, bar_off = b_off + SB * b_stage_bytes, epi_off = bar_off + BAR_BLOCK_BYTES;
  HaloSmem m;
  m.SA = SA; m.SB = SB; m.a_stage_bytes = a_stage_bytes; m.b_stage_bytes = b_stage_bytes;
  m.a = base;
  m.b = base + b_off;
  m.a_full = reinterpret_cast<uint64_t*>(base + bar_off);
  m.a_empty = m.a_full + MAX_SA;
  m.b_full = m.a_empty + MAX_SA;
  m.b_empty = m.b_full + MAX_SB;
  m.spare = m.b_empty + MAX_SB;
  m.epi = base + epi_off;
  m.bytes = SMEM_ALIGN_SLACK + epi_off + epi_bytes;
  return m;
}

// Most filter taps whose [BN x 64] weight tiles share one 16 KB weight stage (HaloLayer::tps never exceeds it).
__host__ __device__ constexpr int halo_max_tps(int bn) { return 128 / bn > 1 ? 128 / bn : 1; }

// One filter tap: 4 k-steps of 16 channels for each m64 block, then the descriptors move on to the next tap.
// TF32: the split-tf32 form (4 k-steps of 8 fp32 channels, the same 32-byte descriptor step).
template <int BN, int MB, bool TF32>
__device__ __forceinline__ void halo_tap(float (&acc)[MB][BN / 2], uint64_t (&adesc)[MB], uint64_t& bdesc, uint32_t& accum,
                                         int& kx, int kw, uint32_t step_x, uint32_t step_row, uint32_t tap16) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int b = 0; b < MB; ++b) {
      if constexpr (TF32) ppx::wgmma_tf32<BN>(acc[b], adesc[b] + 2 * k, bdesc + 2 * k, (accum | k) != 0 ? 1u : 0u);
      else ppx::wgmma_f16<BN>(acc[b], adesc[b] + 2 * k, bdesc + 2 * k, (accum | k) != 0 ? 1u : 0u);
    }
  accum = 1u;
  bdesc += tap16;
  const uint32_t step = ++kx == kw ? step_row : step_x;
  if (kx == kw) kx = 0;
#pragma unroll
  for (int b = 0; b < MB; ++b) adesc[b] += step;
}

// The wgmmas of one weight stage (tn <= NT filter taps) as one commit group.  The tap count is dispatched to a
// compile-time constant, so the group is straight-line code.  A runtime-length tap loop puts the group's wgmmas on
// several control paths; ptxas then injects warpgroup.arrive at the joins (C7519 / C7520) and makes every wgmma wait
// for the previous one.
template <int BN, int MB, int NT, bool TF32>
__device__ __forceinline__ void halo_tap_group(int tn, float (&acc)[MB][BN / 2], uint64_t (&adesc)[MB], uint64_t bdesc,
                                               uint32_t& accum, int& kx, int kw, uint32_t step_x, uint32_t step_row,
                                               uint32_t tap16) {
  using namespace ppx;
  if constexpr (NT > 1) {
    if (tn < NT) {
      halo_tap_group<BN, MB, NT - 1, TF32>(tn, acc, adesc, bdesc, accum, kx, kw, step_x, step_row, tap16);
      return;
    }
  }
  wgmma_fence();
#pragma unroll
  for (int tt = 0; tt < NT; ++tt) halo_tap<BN, MB, TF32>(acc, adesc, bdesc, accum, kx, kw, step_x, step_row, tap16);
  wgmma_commit();
}

// The main loop of one tile, run by each of the two consumer warpgroups: into register accumulators acc (MB = h.MT m64
// blocks of BN columns).  A stage is handed back to its producer once the wgmma group that read it has completed (one
// group per weight stage, one group in flight).  NT: see halo_tap_group.  TF32: the split-tf32 form.  `before_wait`
// runs once the tile's last commit group is issued, before the wait for it (the TMA epilogue issues its operand loads
// there).
template <int BN, int MB, int NT, bool TF32, class BeforeWait>
__device__ __forceinline__ void halo_mainloop(const HaloLayer& h, const HaloSmem& m, Ring& ra, Ring& rb, int wg,
                                              float (&acc)[MB][BN / 2], BeforeWait&& before_wait) {
  using namespace ppx;
  const PPConvParams& p = h.c;
  const int taps = p.kh * p.kw;
  const uint32_t sbo = h.flat ? 1024u : (uint32_t)h.BW * 128;
  const uint32_t step_x = (uint32_t)p.dw * 8;                                 // next tap in the row (16-byte units)
  const uint32_t step_row = (uint32_t)(p.dh * h.BW - (p.kw - 1) * p.dw) * 8;  // last tap of a row -> next row
  const uint32_t tap16 = (uint32_t)p.BN * 8;                                  // next tap's weight tile in the stage
  const int kw = p.kw;
  uint32_t aoff[MB];
#pragma unroll
  for (int b = 0; b < MB; ++b) aoff[b] = MB == 2 ? wg * h.sub_bytes + b * 8 * sbo : wg * 8 * sbo;
  uint32_t accum = 0;
  int pend_a = -1, pend_b = -1;
  for (int c = 0; c < h.chunks; ++c) {
    mbar_wait(&m.a_full[ra.s], ra.ph);
    uint64_t adesc[MB];
#pragma unroll
    for (int b = 0; b < MB; ++b) adesc[b] = gmma_desc_sw128_kmajor(smem_u32(m.a + ra.s * m.a_stage_bytes) + aoff[b], sbo);
    int kx = 0;
    for (int tap0 = 0; tap0 < taps; tap0 += h.tps) {
      mbar_wait(&m.b_full[rb.s], rb.ph);
      const uint64_t bdesc = gmma_desc_sw128_kmajor(smem_u32(m.b + rb.s * m.b_stage_bytes));
      halo_tap_group<BN, MB, NT, TF32>(min(h.tps, taps - tap0), acc, adesc, bdesc, accum, kx, kw, step_x, step_row, tap16);
      wgmma_wait<1>();
      if (pend_b >= 0) mbar_arrive(&m.b_empty[pend_b]);
      if (pend_a >= 0) mbar_arrive(&m.a_empty[pend_a]);
      pend_b = rb.s;
      pend_a = tap0 + h.tps >= taps ? ra.s : -1;
      if (++rb.s == m.SB) { rb.s = 0; rb.ph ^= 1; }
    }
    if (++ra.s == m.SA) { ra.s = 0; ra.ph ^= 1; }
  }
  before_wait();
  wgmma_wait<0>();
#pragma unroll
  for (int b = 0; b < MB; ++b) wgmma_fence_acc(acc[b]);
  if (pend_b >= 0) mbar_arrive(&m.b_empty[pend_b]);
  if (pend_a >= 0) mbar_arrive(&m.a_empty[pend_a]);
}

// One tile of one consumer warpgroup on the drain epilogue: the main loop, then the epilogue of this warpgroup's pixel
// rows through the fp32 staging tile `stg`.  TF32: the split-tf32 form.  PROG (conv_prog_kernel): the layer has the
// plain epilogue (PP_EPI_STD), so the GRU epilogues are not compiled in.
template <int BN, int MB, int NT, bool TF32 = false, bool PROG = false>
__device__ __forceinline__ void halo_tile(const HaloLayer& h, int tile, const HaloSmem& m, Ring& ra, Ring& rb, float* stg,
                                          int wg, int t128) {
  const PPConvParams& p = h.c;
  const TileCoord t = decode_tile(h, tile);
  const int n0 = t.n_idx * p.BN;
  const int bnt = min(p.BN, p.Cout_g_pad - n0);   // columns >= bnt of the last N tile read stale weights: never stored
  float acc[MB][BN / 2];
  halo_mainloop<BN, MB, NT, TF32>(h, m, ra, rb, wg, acc, [] {});

  // ---- epilogue
  const bool skip = (h.debug & 1) != 0;
#pragma unroll
  for (int b = 0; b < MB; ++b) {
    const int sub = MB == 2 ? wg : 0, rbase = MB == 2 ? 64 * b : 64 * wg;
    ppconv::drain_acc<BN>(acc[b], stg, t128, 4 + wg, [&](const float* src, int r64, int cc) {
      const int r = rbase + r64;   // row of the 128-pixel sub-tile: 16 rows x 8 columns (spatial) or 128 pixels (flat)
      bool mvalid;
      long long mrow;
      if (h.flat) {
        mrow = ((long long)t.tx * h.MT + sub) * 128 + r;
        mvalid = mrow < p.M_total;
      } else {
        const int oy = t.ty * 16 + (r >> 3), ox = t.tx * (8 * h.MT) + 8 * sub + (r & 7);
        mvalid = oy < p.OH && ox < p.OW;
        mrow = ((long long)t.img * p.OH + oy) * p.OW + ox;
      }
      if (!mvalid || skip || cc >= bnt || n0 + cc >= p.Cout_g) return;
      ppconv::epilogue_from_stage<TF32, PROG ? PP_EPI_STD : -1>(p, src, mrow, t.g, n0 + cc);
    });
  }
}

// ---- conv_halo_kernel's TMA epilogue (HaloParams::tma_out)
// Its epilogue region (HaloSmem::epi):
//   fp16 staging tile | the tile's bias columns | GRU_H: one z panel per warpgroup
// The staging tile holds, per consumer warpgroup, BN / pw panels of [64 MT pixels][pw channels] (ppconv::frag_epilogue
// with PW = pw and a panel stride of one warpgroup's rows).  A warpgroup's pixels are its 8 x 16
// (MT = 2) or 8 x 8 (MT = 1) block of the tile, or its run of consecutive pixels in flat mode, in box order, so row r of
// a panel is accumulator row r of the warpgroup.
__host__ __device__ constexpr int halo_panel_width(int bn) { return bn % 64 == 0 ? 64 : bn % 32 == 0 ? 32 : 16; }
__host__ __device__ constexpr int halo_out_stage_bytes(int mt, int bn) { return 2 * 64 * mt * bn * 2; }
__host__ __device__ constexpr int halo_out_bias_bytes(int bn) { return (2 * bn * 4 + 1023) / 1024 * 1024; }
__host__ __device__ constexpr int halo_out_z_bytes(int mt, int bn) { return 2 * 64 * mt * halo_panel_width(bn) * 2; }
__host__ __device__ constexpr int halo_tma_region_bytes(int mt, int bn, bool gru_h) {
  return halo_out_stage_bytes(mt, bn) + halo_out_bias_bytes(bn) + (gru_h ? halo_out_z_bytes(mt, bn) : 0);
}
// the epilogue region of a conv_halo_kernel / conv_halo_tf32_kernel launch
__host__ __device__ inline int halo_epi_bytes(const HaloParams& h) {
  return h.tma_out ? halo_tma_region_bytes(h.MT, h.c.BN, h.c.epi == PP_EPI_GRU_H) : DRAIN_EPI_BYTES;
}
// barriers of the operand loads, one per consumer warpgroup, behind HaloSmem::spare
__device__ __forceinline__ uint64_t* halo_out_bar(const HaloSmem& m, int wg) { return m.spare + 1 + wg; }

// One tile of one consumer warpgroup on the TMA path: the main loop; the operand loads of the epilogue (residual / h
// into the staging tile, GRU_H's first z panel) issued once the last commit group is out, so they overlap its wgmmas;
// the fragment epilogue into the staging tile; this warpgroup's TMA stores, which drain under the next tile's main
// loop.  The staging tile is waited for (cp.async.bulk.wait_group.read) only before it is written again.  `xph`: the
// parity of this warpgroup's operand-load barrier.
template <int BN, int MB, int NT>
__device__ __forceinline__ void halo_tile_tma(const HaloParams& h, int tile, const HaloSmem& m, Ring& ra, Ring& rb,
                                              uint32_t& xph, int wg, int t128) {
  using namespace ppx;
  const PPConvParams& p = h.c;
  constexpr int PW = halo_panel_width(BN);
  constexpr int PANEL = 64 * MB * PW * 2;
  const TileCoord t = decode_tile(h, tile);
  const int n0 = t.n_idx * BN;
  const int epi = p.epi;
  const int half_c = p.Cout_g >> 1;
  const bool r_tile = epi == PP_EPI_GRU_ZR && n0 >= half_c;   // GRU_ZR: BN divides half_c (halo_tma_configure)
  const bool has_aux = epi == PP_EPI_STD ? p.aux0 != nullptr : (epi == PP_EPI_GRU_H || r_tile);
  const int npanel = (min(BN, p.Cout_g - n0) + PW - 1) / PW;   // panels with channels to store; TMA clips the last one
  uint8_t* so = m.epi + wg * (64 * MB * BN * 2);
  float* bs = reinterpret_cast<float*>(m.epi + halo_out_stage_bytes(MB, BN)) + wg * BN;
  uint8_t* zb = m.epi + halo_out_stage_bytes(MB, BN) + halo_out_bias_bytes(BN) + wg * PANEL;
  uint64_t* xbar = halo_out_bar(m, wg);
  // this warpgroup's box: pixel coordinates (flat: first pixel) and image
  int x0, y0, img;
  if (h.flat) {
    x0 = MB == 2 ? (t.tx * 2 + wg) * 128 : t.tx * 128 + 64 * wg; y0 = 0; img = 0;
  } else {
    x0 = t.tx * (8 * MB) + (MB == 2 ? 8 * wg : 0); y0 = t.ty * 16 + (MB == 2 ? 0 : 8 * wg); img = t.img;
  }
  const int aux_c = r_tile ? n0 - half_c : n0;
  const bool issuer = t128 == 0;
  const bool skip = (h.debug & 1) != 0;
  float acc[MB][BN / 2];
  halo_mainloop<BN, MB, NT, false>(h, m, ra, rb, wg, acc, [&] {
    if (issuer && has_aux && !skip) {
      tma_store_wait_read<0>();   // the previous tile's stores have read the staging tile
      const int nz = epi == PP_EPI_GRU_H ? 1 : 0;
      mbar_arrive_expect_tx(xbar, (uint32_t)((npanel + nz) * PANEL));
      for (int pn = 0; pn < npanel; ++pn)
        tma_load_4d(smem_u32(so + pn * PANEL), &h.tm_aux0, aux_c + pn * PW, x0, y0, img, xbar);
      if (nz) tma_load_4d(smem_u32(zb), &h.tm_aux1, n0, x0, y0, img, xbar);
    }
  });
  if (skip) return;

  // the tile's bias columns; the previous tile's readers of this copy have passed its last named barrier
  ppconv::stage_bias<BN>(p, bs, t.g * p.Cout_g, n0, t128);
  const int bar_id = 4 + wg;
  if (issuer && !has_aux) tma_store_wait_read<0>();
  named_bar(bar_id, 128);
  if (has_aux) {
    mbar_wait(xbar, xph);
    xph ^= 1;
  }
  using ppconv::IntC;
  auto epilogue = [&](auto kind, auto act1, bool aux, int P) {
    ppconv::frag_epilogue<MB, BN, PW, PANEL, decltype(kind)::value, decltype(act1)::value>(p, acc, so, zb, bs, aux, r_tile,
                                                                                           P, t128);
  };
  if (epi == PP_EPI_STD) {
    switch (p.act1) {
      case PP_ACT_RELU: epilogue(IntC<PP_EPI_STD>{}, IntC<PP_ACT_RELU>{}, has_aux, 0); break;
      case PP_ACT_LRELU: epilogue(IntC<PP_EPI_STD>{}, IntC<PP_ACT_LRELU>{}, has_aux, 0); break;
      default: epilogue(IntC<PP_EPI_STD>{}, IntC<PP_ACT_NONE>{}, has_aux, 0); break;
    }
  } else if (epi == PP_EPI_GRU_ZR) {
    epilogue(IntC<PP_EPI_GRU_ZR>{}, IntC<PP_ACT_NONE>{}, r_tile, 0);
  } else {
    // one z panel at a time: before the next one is loaded, every thread has read the current one
#pragma unroll 1
    for (int pn = 0; pn < npanel; ++pn) {
      if (pn > 0) {
        named_bar(bar_id, 128);
        if (issuer) {
          mbar_arrive_expect_tx(xbar, (uint32_t)PANEL);
          tma_load_4d(smem_u32(zb), &h.tm_aux1, n0 + pn * PW, x0, y0, img, xbar);
        }
        mbar_wait(xbar, xph);
        xph ^= 1;
      }
      epilogue(IntC<PP_EPI_GRU_H>{}, IntC<PP_ACT_NONE>{}, true, pn);
    }
  }
  fence_proxy_async();           // generic-proxy smem writes -> visible to the TMA stores
  named_bar(bar_id, 128);
  if (issuer) {
    const CUtensorMap* tm = r_tile ? &h.tm_out2 : &h.tm_out;
    const int c0 = r_tile ? n0 - half_c : t.g * p.out_gstep + n0;
    for (int pn = 0; pn < npanel; ++pn) tma_store_4d(tm, smem_u32(so + pn * PANEL), c0 + pn * PW, x0, y0, img);
    tma_store_commit();
  }
}

// f(IntC<BN>, IntC<MT>) for the layer's runtime tile shape (MT == 2 layers have BN <= 128)
template <class F>
__device__ __forceinline__ void with_tile_shape(int mt, int bn, F&& f) {
  if (mt == 2) ppconv::with_tile_width<128>(bn, [&](auto n) { f(n, ppconv::IntC<2>{}); });
  else ppconv::with_tile_width<256>(bn, [&](auto n) { f(n, ppconv::IntC<1>{}); });
}

// Thread 0: the barriers of both rings (full: the producer's arrival + transaction bytes, empty: every consumer thread).
__device__ __forceinline__ void halo_smem_init_barriers(const HaloSmem& m) {
  using namespace ppx;
  for (int s = 0; s < m.SA; ++s) { mbar_init(&m.a_full[s], 1); mbar_init(&m.a_empty[s], NUM_EPI_THREADS); }
  for (int s = 0; s < m.SB; ++s) { mbar_init(&m.b_full[s], 1); mbar_init(&m.b_empty[s], NUM_EPI_THREADS); }
  mbar_fence_init();
}

// Input patch producer (TMA, one elected thread): one box load per 64-channel chunk of each of this CTA's tiles of one
// layer.  `r` runs on across the layers of a program.
__device__ __forceinline__ void halo_produce_patches(const HaloLayer& h, const HaloSmem& m, Ring& r) {
  using namespace ppx;
  const PPConvParams& p = h.c;
  const int total_tiles = halo_total_tiles(h);
  const uint32_t bytes = (uint32_t)(h.BW * h.BH * 128);
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const TileCoord t = decode_tile(h, tile);
    const int x0 = h.flat ? t.tx * (128 * h.MT) : t.tx * (8 * h.MT) - p.pw, y0 = h.flat ? 0 : t.ty * 16 - p.ph;
    for (int c = 0; c < h.chunks; ++c) {
      const int ci = c * 64;
      const int q = pp_seg_of(p, ci);
      const int ch0 = t.g * p.seg[q].gstep + (ci - p.seg[q].cbegin);
      mbar_wait(&m.a_empty[r.s], r.ph ^ 1);
      mbar_arrive_expect_tx(&m.a_full[r.s], bytes);
      tma_load_4d(smem_u32(m.a + r.s * m.a_stage_bytes), &h.tmap[q], ch0, x0, y0, t.img, &m.a_full[r.s]);
      if (++r.s == m.SA) { r.s = 0; r.ph ^= 1; }
    }
  }
}

// Weight tile producer (bulk copy, one elected thread): per chunk, the [BN x 64] tiles of the filter taps in groups of
// h.tps per stage.  `r` runs on across the layers of a program.
__device__ __forceinline__ void halo_produce_weights(const HaloLayer& h, const HaloSmem& m, Ring& r) {
  using namespace ppx;
  const PPConvParams& p = h.c;
  const int total_tiles = halo_total_tiles(h);
  const int taps = p.kh * p.kw;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const TileCoord t = decode_tile(h, tile);
    const int n0 = t.n_idx * p.BN;
    const uint32_t bytes = (uint32_t)(min(p.BN, p.Cout_g_pad - n0) * 128);
    const __half* wbase = p.wpacked + ((long long)t.g * p.num_kc * p.Cout_g_pad + n0) * 64;
    for (int c = 0; c < h.chunks; ++c) {
      for (int tap0 = 0; tap0 < taps; tap0 += h.tps) {
        const int tn = min(h.tps, taps - tap0);
        mbar_wait(&m.b_empty[r.s], r.ph ^ 1);
        mbar_arrive_expect_tx(&m.b_full[r.s], bytes * (uint32_t)tn);
        for (int t = 0; t < tn; ++t) {
          const int kc = (tap0 + t) * h.chunks + c;
          bulk_g2s(smem_u32(m.b + r.s * m.b_stage_bytes + t * p.BN * 128), wbase + (long long)kc * p.Cout_g_pad * 64, bytes,
                   &m.b_full[r.s]);
        }
        if (++r.s == m.SB) { r.s = 0; r.ph ^= 1; }
      }
    }
  }
}

template <bool TF32>
__device__ __forceinline__ void halo_body(const HaloParams& h) {
  using namespace ppx;
  const HaloSmem m = halo_smem(dyn_smem_1024(), h.SA, h.a_stage_bytes, h.SB, h.b_stage_bytes, halo_epi_bytes(h));
  const int tid = threadIdx.x, warp = tid >> 5;
  if (tid == 0) {
    if constexpr (!TF32) {
      mbar_init(halo_out_bar(m, 0), 1);
      mbar_init(halo_out_bar(m, 1), 1);
    }
    halo_smem_init_barriers(m);
  }
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  // 168 registers per thread at launch; the producer warpgroup gives its registers to the accumulator holders (an
  // increase can only use what this CTA released: 2 x 128 x (232 - 168) == 128 x (168 - 40))
  if (warp < 8) setmaxnreg_inc<232>();
  else setmaxnreg_dec<40>();
  if (warp < 8) {
    // ------------------------------------------------------------------ consumers: wgmma + epilogue
    const int wg = tid >> 7, t128 = tid & 127;
    float* stg = reinterpret_cast<float*>(m.epi + wg * ppconv::STG_BYTES);
    Ring ra = {0, 0}, rb = {0, 0};
    const int total_tiles = halo_total_tiles(h);
    if constexpr (!TF32) {
      if (h.tma_out) {
        uint32_t xph = 0;
        with_tile_shape(h.MT, h.c.BN, [&](auto bn, auto mb) {
          constexpr int BN = decltype(bn)::value;
          for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x)
            halo_tile_tma<BN, decltype(mb)::value, halo_max_tps(BN)>(h, tile, m, ra, rb, xph, wg, t128);
        });
        if (t128 == 0) tma_store_wait<0>();   // this warpgroup's last stores are complete
        return;
      }
    }
    with_tile_shape(h.MT, h.c.BN, [&](auto bn, auto mb) {
      constexpr int BN = decltype(bn)::value;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x)
        halo_tile<BN, decltype(mb)::value, halo_max_tps(BN), TF32>(h, tile, m, ra, rb, stg, wg, t128);
    });
  } else if (warp == WARP_A) {
    if (elect_one()) {
      Ring r = {0, 0};
      halo_produce_patches(h, m, r);
    }
  } else if (warp == WARP_B) {
    if (elect_one()) {
      Ring r = {0, 0};
      halo_produce_weights(h, m, r);
    }
  }
}

__global__ void __launch_bounds__(NUM_THREADS, 1) conv_halo_kernel(const __grid_constant__ HaloParams h) {
  halo_body<false>(h);
}

__global__ void __launch_bounds__(NUM_THREADS, 1) conv_halo_tf32_kernel(const __grid_constant__ HaloParams h) {
  halo_body<true>(h);
}

// ---------------------------------------------------------------------------------------------------------------------
// Multi-layer program: up to PROG_MAX_LAYERS dependent layers (stride-1 convolutions of the kind above, and modulated
// deformable sampling) executed by ONE launch of one CTA per SM, with a grid-wide barrier between consecutive layers.
// The recurrent propagation steps of flow completion are 8 dependent layers over 3,600-7,200 pixels: as separate
// launches each pays launch + prologue + pipeline fill/drain (~15-30 us, mostly fixed); here the fixed cost per layer
// is one barrier (an atomic counter in global memory) and one TMA round trip, the weight producer runs ahead across the
// barrier, and mbarriers / tensor maps are set up once.
//
// Ordering between layers: the consumer threads (the only writers of global memory) make their generic-proxy stores
// visible to the async proxy (fence.proxy.async.global), meet on a named barrier, and one thread publishes the CTA's
// arrival (threadfence + atomicAdd).  The TMA producer and the epilogue warps of the next layer spin on the counter
// (ld.acquire.gpu) before they touch that layer's inputs; the producer adds the consumer-side proxy fence before
// issuing TMA loads.  All CTAs (one per SM) are co-resident (1 CTA per SM by shared memory), so the spin cannot deadlock.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int PROG_MAX_LAYERS = 10;
enum { PROG_CONV = 0, PROG_DCN = 1 };

// The N tile widths of program layers (all with MT == 1), the ones the plan of halo_configure (one_wave) picks for the
// propagation steps of flow completion: two clips (D = 2, 7,200 pixels at 640x360) take 64 for the 128-channel layers and
// 224 for the 432-channel offset head (2 N tiles: one wave), one clip (D = 1) takes 32 and 64.  Each width instantiates
// the whole main loop and epilogue in the consumer warpgroups' 232 registers, so the list is kept this short: all eight
// widths up to 128 made the kernel spill and ptxas serialize its wgmmas, and 112 next to 224 spills too.
constexpr int PROG_WIDTHS[] = {32, 64, 224};

template <class F>
__device__ __forceinline__ void with_prog_width(int bn, F&& f) {
  static_assert(sizeof(PROG_WIDTHS) == 3 * sizeof(int), "with_prog_width: one case per PROG_WIDTHS entry");
  switch (bn) {
    case PROG_WIDTHS[0]: f(ppconv::IntC<PROG_WIDTHS[0]>{}); break;
    case PROG_WIDTHS[1]: f(ppconv::IntC<PROG_WIDTHS[1]>{}); break;
    case PROG_WIDTHS[2]: f(ppconv::IntC<PROG_WIDTHS[2]>{}); break;
    default: __trap();
  }
}

struct ProgParams {
  int n_layers;
  int SA, SB, a_stage_bytes, b_stage_bytes;   // one shared-memory carve-up for every layer
  unsigned int* counter;                      // arrivals since the counter was zeroed
  unsigned int base;                          // arrivals issued before this launch
  unsigned long long* ts;                     // debug (PP_PROG_TS=1): globaltimer of CTA 0 at [layer start, layer end]
  int kind[PROG_MAX_LAYERS];
  PPDcnArgs dcn[PROG_MAX_LAYERS];
  HaloLayer layer[PROG_MAX_LAYERS];
};

__device__ __forceinline__ void prog_wait(const unsigned int* counter, unsigned int target) {
  unsigned int v, spins = 0;
  uint64_t t0 = 0;
  for (;;) {
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
    if ((int)(v - target) >= 0) return;
    __nanosleep(64);                      // one poller per CTA, backed off: the arrivals' atomics are not starved
    if ((++spins & 0xFFFu) == 0) {       // a lost arrival must not hang the GPU: trap after ~2 s
      uint64_t now;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      if (t0 == 0) t0 = now;
      else if (now - t0 > 2000000000ull) __trap();
    }
  }
}

__global__ void __launch_bounds__(NUM_THREADS, 1) conv_prog_kernel(const __grid_constant__ ProgParams P) {
  using namespace ppx;
  const HaloSmem m = halo_smem(dyn_smem_1024(), P.SA, P.a_stage_bytes, P.SB, P.b_stage_bytes, DRAIN_EPI_BYTES);
  uint64_t* layer_go = m.spare;   // the CTA's one poller (TMA producer thread) -> consumers: layer li may start

  const int tid = threadIdx.x, warp = tid >> 5;
  const unsigned int G = gridDim.x;
  if (tid == 0) {
    mbar_init(layer_go, 1);
    halo_smem_init_barriers(m);
  }
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp < 8) setmaxnreg_inc<232>();
  else setmaxnreg_dec<40>();
  if (warp < 8) {
    // ------------------------------------------------------------------ consumers: wgmma + epilogue (+ the sampling layers)
    const int wg = tid >> 7, t128 = tid & 127;
    float* stg = reinterpret_cast<float*>(m.epi + wg * ppconv::STG_BYTES);
    Ring ra = {0, 0}, rb = {0, 0};
    for (int li = 0; li < P.n_layers; ++li) {
      // inputs of this layer (residuals, sampling sources) were written by the previous one: the producer thread polls
      // the grid counter for the whole CTA and releases the epilogue warps through a shared-memory barrier
      mbar_wait(layer_go, (uint32_t)li & 1u);
      if (P.ts != nullptr && blockIdx.x == 0 && tid == 0) {
        unsigned long long now;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
        P.ts[2 * li] = now;
      }
      if (P.kind[li] == PROG_DCN) {
        const PPDcnArgs& a = P.dcn[li];
        const unsigned per_img = (unsigned)(a.H * a.W * 144);
        const unsigned total = per_img * (unsigned)a.N;
        const unsigned stride = G * NUM_EPI_THREADS;
        // the sampling is bound by L1 wavefronts (one per uncoalesced 16/32-byte gather), not by latency: a two-phase
        // batched form (all offsets first, then all gathers) measured slower (78 vs 52 us per layer)
        for (unsigned idx = blockIdx.x * NUM_EPI_THREADS + tid; idx < total; idx += 4 * stride) {
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const unsigned i2 = idx + u * stride;
            if (i2 < total) {
              const unsigned n = i2 / per_img;
              if (a.C == 128) dcn_sample_item<8, true>(a, i2 - n * per_img, (int)n);
              else dcn_sample_item<16, true>(a, i2 - n * per_img, (int)n);
            }
          }
        }
      } else {
        const HaloLayer& h = P.layer[li];
        const int total_tiles = halo_total_tiles(h);
        // program layers are configured with MT == 1 and BN in PROG_WIDTHS (halo_configure, one_wave)
        with_prog_width(h.c.BN, [&](auto bn) {
          constexpr int BN = decltype(bn)::value;
          for (int tile = blockIdx.x; tile < total_tiles; tile += G)
            halo_tile<BN, 1, halo_max_tps(BN), false, true>(h, tile, m, ra, rb, stg, wg, t128);
        });
      }
      // publish this CTA's part of the layer: stores -> async proxy, CTA-wide meet of the writers, one arrival
      fence_proxy_async_global();
      asm volatile("bar.sync 1, %0;" ::"n"(NUM_EPI_THREADS) : "memory");
      if (tid == 0) {
        __threadfence();
        atomicAdd(P.counter, 1u);
        if (P.ts != nullptr && blockIdx.x == 0) {
          unsigned long long now;
          asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
          P.ts[2 * li + 1] = now;
        }
      }
    }
  } else if (warp == WARP_A) {
    // ------------------------------------------------------------------ input patch producer (TMA)
    if (elect_one()) {
      Ring r = {0, 0};
      for (int li = 0; li < P.n_layers; ++li) {
        if (li > 0) {     // the CTA's only poller: every CTA finished layer li-1
          prog_wait(P.counter, P.base + (unsigned int)li * G);
          fence_proxy_async_global();
        }
        mbar_arrive(layer_go);
        if (P.kind[li] == PROG_CONV) halo_produce_patches(P.layer[li], m, r);
      }
    }
  } else if (warp == WARP_B) {
    // ------------------------------------------------------------------ weight tile producer: never waits for a layer
    if (elect_one()) {
      Ring r = {0, 0};
      for (int li = 0; li < P.n_layers; ++li)
        if (P.kind[li] == PROG_CONV) halo_produce_weights(P.layer[li], m, r);
    }
  }
}

}  // namespace

// 0 = not eligible (caller falls back to the cp.async implicit-GEMM kernel), 1 = eligible.
int pp_conv_halo_eligible(const PPConvParams& p) {
  if (p.sh != 1 || p.sw != 1 || p.pad_replicate) return 0;
  const bool flat = p.kh * p.kw == 1;
  if (flat) {
    // 1x1 conv / linear layer: tiles are runs of consecutive pixels; a ragged channel tail is zero-filled by TMA
    if (p.ph != 0 || p.pw != 0 || p.groups != 1) return 0;
  } else if (p.Cin % 64 != 0) {
    return 0;   // packed K order is (tap, ci): 64-channel chunks must not straddle taps
  }
  if (!pp_conv_segs_chunked(p, flat)) return 0;
  if ((p.kw - 1) * p.dw + 16 > 256 || (p.kh - 1) * p.dh + 16 > 256) return 0;
  if ((long long)p.N * p.OH * p.OW < 128) return 0;
  return pp_tmap_supported() ? 1 : 0;
}

namespace {

// The dynamic shared memory limits of the three halo kernels (conv_halo_kernel's TMA epilogue uses all an SM has),
// raised once before the first launch.
int halo_set_smem_limit() {
  static bool done = false;
  if (!done) {
    PP_CUDA_CHECK(cudaFuncSetAttribute(conv_halo_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_MAX));
    PP_CUDA_CHECK(cudaFuncSetAttribute(conv_halo_tf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
    PP_CUDA_CHECK(cudaFuncSetAttribute(conv_prog_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
    done = true;
  }
  return PP_OK;
}

// Pipeline depth for stages of a_bytes / b_bytes in `budget` bytes: the deepest patch ring (3 or 2 stages) that leaves
// room for at least 3 weight stages, and as many weight stages as fit (at most MAX_SB).  false: nothing fits.
bool halo_stages(int budget, int a_bytes, int b_bytes, int& sa, int& sb) {
  for (sa = 3; sa >= 2; --sa) {
    sb = (budget - sa * a_bytes) / b_bytes;
    if (sb >= 3) {
      if (sb > MAX_SB) sb = MAX_SB;
      return true;
    }
  }
  return false;
}

// h.SA / h.SB for stages in `budget` bytes (halo_stages, then a 4th patch stage where that leaves the weight ring full).
bool halo_layer_stages(int budget, HaloLayer& h) {
  int sa = 0, sb = 0;
  if (!halo_stages(budget, h.a_stage_bytes, h.b_stage_bytes, sa, sb)) return false;
  if (sa == 3 && sb == MAX_SB && (budget - 4 * h.a_stage_bytes) / h.b_stage_bytes >= MAX_SB) sa = 4;
  h.SA = sa; h.SB = sb;
  return true;
}

// conv_halo_kernel's TMA epilogue for a configured fp16 layer: its tensor maps, and the stages that fit next to the
// staging tile.  false: the layer keeps the drain epilogue (plain fp32 output, an activation without a compiled-in
// case, 16-byte misaligned outputs or operands, a channel count that is not a multiple of 8, grouped outputs that are
// not packed per group, GRU_ZR tiles that straddle the z | r boundary, or stages that do not fit).
bool halo_tma_configure(HaloParams& h) {
  const PPConvParams& p = h.c;
  const int bn = p.BN, pw = halo_panel_width(bn), rows = 64 * h.MT;
  if (p.split || p.out_fp32) return false;
  if (p.epi == PP_EPI_STD && p.act1 != PP_ACT_NONE && p.act1 != PP_ACT_RELU && p.act1 != PP_ACT_LRELU) return false;
  if (p.epi != PP_EPI_STD && p.groups != 1) return false;
  if (p.epi == PP_EPI_STD && p.aux0 != nullptr && p.groups != 1) return false;
  if (p.groups > 1 && (p.out_gstep != p.Cout_g || p.Cout_g % pw != 0)) return false;
  if (p.epi == PP_EPI_GRU_ZR && (p.Cout_g % 2 != 0 || (p.Cout_g / 2) % bn != 0)) return false;
  if (!aligned16(p.out, p.out_cstride, p.out_coff) || (p.groups > 1 && p.out_gstep % 8 != 0)) return false;
  // TMA stores clip the channel dimension at 16-byte granularity (measured on H100: a 126-channel map wrote channels
  // 126 and 127), so a channel count that ends inside a 16-byte unit would overwrite its neighbours
  if (p.Cout_g % 8 != 0) return false;
  if (p.aux0 != nullptr && !aligned16(p.aux0, p.aux0_cstride, p.aux0_coff)) return false;
  if (p.epi == PP_EPI_GRU_H && !aligned16(p.aux1, p.aux1_cstride, p.aux1_coff)) return false;
  if (p.epi == PP_EPI_GRU_ZR && !aligned16(p.out2, p.out2_cstride, p.out2_coff)) return false;
  // the stages get what the rest of the plan leaves of SMEM_MAX
  const int region = halo_tma_region_bytes(h.MT, bn, p.epi == PP_EPI_GRU_H);
  HaloLayer staged = h;
  if (!halo_layer_stages(SMEM_MAX - halo_smem(nullptr, 0, 0, 0, 0, region).bytes, staged)) return false;
  h.SA = staged.SA; h.SB = staged.SB;
  // maps: (channels, x, y, image) boxes of pw x 8 x rows / 8, or (channels, pixel) boxes of pw x rows in flat mode
  auto map = [&](CUtensorMap* m, const __half* base, int cols, int cstride) {
    return h.flat ? pp_tmap_pixels_f16(m, base, cols, cstride, p.M_total, 1, 1, pw, rows, 1)
                  : pp_tmap_pixels_f16(m, base, cols, cstride, p.OW, p.OH, p.N, pw, 8, rows / 8);
  };
  const __half* out = static_cast<const __half*>(p.out) + p.out_coff;
  const int half_c = p.Cout_g / 2;
  if (p.epi == PP_EPI_GRU_ZR) {
    if (map(&h.tm_out, out, half_c, p.out_cstride) != PP_OK) return false;
    if (map(&h.tm_out2, p.out2 + p.out2_coff, half_c, p.out2_cstride) != PP_OK) return false;
    if (map(&h.tm_aux0, p.aux0 + p.aux0_coff, half_c, p.aux0_cstride) != PP_OK) return false;
  } else {
    if (map(&h.tm_out, out, (p.groups - 1) * p.out_gstep + p.Cout_g, p.out_cstride) != PP_OK) return false;
    if (p.aux0 != nullptr && map(&h.tm_aux0, p.aux0 + p.aux0_coff, p.Cout_g, p.aux0_cstride) != PP_OK) return false;
    if (p.epi == PP_EPI_GRU_H && map(&h.tm_aux1, p.aux1 + p.aux1_coff, p.Cout_g, p.aux1_cstride) != PP_OK) return false;
  }
  h.tma_out = 1;
  return true;
}

// Tile shape, pipeline depth and tensor maps of one layer.  one_wave: the layer is one of a multi-layer program whose
// layers are separated by grid-wide barriers -- prefer the least work per CTA (a second, partial wave doubles the
// layer's latency) over fewer weight re-reads, among the tile widths the program kernel instantiates.
int halo_configure(const PPConvParams& pin, HaloLayer& h, bool one_wave) {
  h.c = pin;
  PPConvParams& p = h.c;
  int num_sms = 0;
  PP_TRY(pp_num_sms(&num_sms));
  const bool flat = p.kh * p.kw == 1;
  // N tile: <= 128 columns (MT x BN accumulators of a consumer warpgroup stay within 128 registers per thread)
  const int n_tiles0 = pp_ceil_div(p.Cout_g_pad, 128);
  int bn = pp_ceil_div(pp_ceil_div(p.Cout_g_pad, n_tiles0), 16) * 16;
  const int tiles_y = flat ? 1 : pp_ceil_div(p.OH, 16);
  auto tiles_x = [&](int mt) { return flat ? (int)pp_ceil_div64(p.M_total, 128 * mt) : pp_ceil_div(p.OW, 8 * mt); };
  const int n_img = flat ? 1 : p.N;
  auto count = [&](int mt, int bn_) {
    return (long long)pp_ceil_div(p.Cout_g_pad, bn_) * tiles_x(mt) * tiles_y * n_img * p.groups;
  };
  int mt = count(2, bn) < num_sms ? 1 : 2;
  while (count(mt, bn) < num_sms && bn >= 64 && bn % 32 == 0) bn /= 2;   // small launches: more, narrower tiles
  if (one_wave) {
    // 128-pixel tiles of a width the program kernel instantiates (PROG_WIDTHS).  The layer takes as long as the CTA with
    // the most work, waves x BN columns: the width that makes that smallest, among equals the one with fewer waves.
    // At 640x360 with two clips this puts every layer of a propagation step in one wave of <= 132 tiles.
    mt = 1;
    long long best_cols = -1, best_waves = 0;
    for (const int b : PROG_WIDTHS) {
      const long long waves = (count(1, b) + num_sms - 1) / num_sms;
      if (best_cols < 0 || waves * b < best_cols || (waves * b == best_cols && waves < best_waves)) {
        best_cols = waves * b;
        best_waves = waves;
        bn = b;
      }
    }
  }
  p.BN = bn;
  h.MT = mt;
  h.flat = flat ? 1 : 0;
  h.n_img = n_img;
  h.BW = flat ? 128 * mt : 8 * mt + (p.kw - 1) * p.dw;
  h.BH = flat ? 1 : 16 + (p.kh - 1) * p.dh;
  h.sub_bytes = flat ? 128 * 128 : 8 * 128;
  h.tiles_x = tiles_x(mt);
  h.tiles_y = tiles_y;
  h.n_tiles = pp_ceil_div(p.Cout_g_pad, bn);
  h.chunks = pp_ceil_div(p.Cin, 64);
  h.a_stage_bytes = pp_ceil_div(h.BW * h.BH * 128, 1024) * 1024;
  // narrow N tiles: several filter taps per weight stage (<= 16 KB), see HaloLayer::tps
  h.tps = min(halo_max_tps(bn), p.kh * p.kw);
  h.b_stage_bytes = h.tps * bn * 128;
  PP_REQUIRE(halo_layer_stages(SMEM_BUDGET, h), "conv_halo: patch %dx%d does not fit shared memory", h.BW, h.BH);
  h.debug = pp_conv_noepi();
  const long long total_tiles = count(mt, bn);
  PP_REQUIRE(total_tiles < (1LL << 31), "conv_halo: too many tiles");
  return pp_conv_input_tmaps(p, h.BW, h.BH, flat, h.tmap);
}

}  // namespace

int pp_launch_conv_halo(const PPConvParams& pin, cudaStream_t stream) {
  HaloParams h;
  memset(&h, 0, sizeof(h));
  PP_TRY(halo_configure(pin, h, false));
  PP_TRY(halo_set_smem_limit());
  int num_sms = 0;
  PP_TRY(pp_num_sms(&num_sms));
  halo_tma_configure(h);   // sets h.tma_out, or the layer keeps the drain epilogue
  pp_last_conv_plan() = PPConvPlan{'h', h.MT, h.c.BN, h.tps, h.flat, h.tma_out, h.SA, h.SB};
  const int smem = halo_smem(nullptr, h.SA, h.a_stage_bytes, h.SB, h.b_stage_bytes, halo_epi_bytes(h)).bytes;
  return pp_conv_launch(h.c.split ? conv_halo_tf32_kernel : conv_halo_kernel, h, min(halo_total_tiles(h), num_sms),
                        NUM_THREADS, smem, stream);
}

// ---- multi-layer programs ------------------------------------------------------------------------------------------
namespace {
thread_local PPProgRecorder* g_recorder = nullptr;
}

struct PPProgRecorder {
  ProgParams prog;
  double flops = 0.0;
  int n_conv = 0;
};

bool pp_prog_recording() { return g_recorder != nullptr; }

int pp_prog_begin() {
  PP_REQUIRE(g_recorder == nullptr, "conv program: already recording");
  g_recorder = new PPProgRecorder();
  memset(&g_recorder->prog, 0, sizeof(ProgParams));
  return PP_OK;
}

void pp_prog_abort() {
  delete g_recorder;
  g_recorder = nullptr;
}

int pp_prog_record_conv(const PPConvParams& p) {
  PPProgRecorder* r = g_recorder;
  PP_REQUIRE(r != nullptr, "conv program: not recording");
  PP_REQUIRE(r->prog.n_layers < PROG_MAX_LAYERS, "conv program: more than %d layers", PROG_MAX_LAYERS);
  PP_REQUIRE(pp_conv_halo_eligible(p), "conv program: layer is not a stride-1 TMA halo-kernel convolution");
  PP_REQUIRE(!p.split, "conv program: split-tf32 layers are not supported");
  PP_REQUIRE(p.epi == PP_EPI_STD, "conv program: only the plain epilogue (bias, activations, residual) is compiled in");
  const int li = r->prog.n_layers;
  PP_TRY(halo_configure(p, r->prog.layer[li], true));
  const HaloLayer& h = r->prog.layer[li];
  PP_REQUIRE(h.MT == 1 && (h.c.BN == PROG_WIDTHS[0] || h.c.BN == PROG_WIDTHS[1] || h.c.BN == PROG_WIDTHS[2]),
             "conv program: layer tile %d x %d columns is not instantiated", h.MT, h.c.BN);
  r->prog.kind[li] = PROG_CONV;
  r->prog.n_layers++;
  r->n_conv++;
  return PP_OK;
}

int pp_prog_record_dcn(const PPDcnArgs& a) {
  PPProgRecorder* r = g_recorder;
  PP_REQUIRE(r != nullptr, "conv program: not recording");
  PP_REQUIRE(r->prog.n_layers < PROG_MAX_LAYERS, "conv program: more than %d layers", PROG_MAX_LAYERS);
  const int li = r->prog.n_layers;
  r->prog.kind[li] = PROG_DCN;
  r->prog.dcn[li] = a;
  r->prog.n_layers++;
  return PP_OK;
}

// Launches the recorded layers as ONE kernel (grid = one CTA per SM); `counter` is a zero-initialised device word shared
// by all programs of a stream, `*arrivals` the host-side count of arrivals issued so far on it.
int pp_prog_end(unsigned int* counter, unsigned int* arrivals, cudaStream_t stream) {
  PPProgRecorder* r = g_recorder;
  PP_REQUIRE(r != nullptr, "conv program: not recording");
  g_recorder = nullptr;
  std::unique_ptr<PPProgRecorder> guard(r);
  ProgParams& P = r->prog;
  if (P.n_layers == 0) return PP_OK;
  PP_TRY(halo_set_smem_limit());
  int num_sms = 0;
  PP_TRY(pp_num_sms(&num_sms));
  int a_max = 1024, b_max = 2048;
  for (int i = 0; i < P.n_layers; ++i)
    if (P.kind[i] == PROG_CONV) {
      if (P.layer[i].a_stage_bytes > a_max) a_max = P.layer[i].a_stage_bytes;
      if (P.layer[i].b_stage_bytes > b_max) b_max = P.layer[i].b_stage_bytes;
    }
  int sa = 0, sb = 0;
  PP_REQUIRE(halo_stages(SMEM_BUDGET, a_max, b_max, sa, sb), "conv program: stages do not fit shared memory (A %d B, B %d B)",
             a_max, b_max);
  P.SA = sa; P.SB = sb; P.a_stage_bytes = a_max; P.b_stage_bytes = b_max;
  P.counter = counter;
  P.base = *arrivals;
  static int ts_mode = -1, ts_printed = 0;
  static unsigned long long* ts_dev = nullptr;
  if (ts_mode < 0) {
    const char* e = getenv("PP_PROG_TS");
    ts_mode = (e != nullptr && atoi(e) != 0) ? atoi(e) : 0;
    if (ts_mode) PP_CUDA_CHECK(cudaMalloc(&ts_dev, 2 * PROG_MAX_LAYERS * sizeof(unsigned long long)));
  }
  P.ts = (ts_mode && ts_printed < ts_mode) ? ts_dev : nullptr;
  const int grid = num_sms;
  *arrivals += (unsigned int)(P.n_layers * grid);
  PP_TRY(pp_conv_launch(conv_prog_kernel, P, grid, NUM_THREADS, halo_smem(nullptr, sa, a_max, sb, b_max, DRAIN_EPI_BYTES).bytes, stream));
  if (P.ts != nullptr) {      // debug: per-layer wall time of CTA 0 (serialises the stream)
    unsigned long long h[2 * PROG_MAX_LAYERS];
    PP_CUDA_CHECK(cudaStreamSynchronize(stream));
    PP_CUDA_CHECK(cudaMemcpy(h, ts_dev, sizeof(h), cudaMemcpyDeviceToHost));
    ++ts_printed;
    fprintf(stderr, "[prog %d] %d layers:", ts_printed, P.n_layers);
    for (int i = 0; i < P.n_layers; ++i) {
      const HaloLayer& L = P.layer[i];
      if (P.kind[i] == PROG_CONV)
        fprintf(stderr, " | conv K=%d N=%d bn=%d mt=%d tiles=%d: %.1f us (gap %.1f)", L.c.K_total, L.c.Cout_g, L.c.BN, L.MT,
                halo_total_tiles(L), (h[2 * i + 1] - h[2 * i]) / 1e3, i ? (h[2 * i] - h[2 * i - 1]) / 1e3 : 0.0);
      else
        fprintf(stderr, " | dcn: %.1f us (gap %.1f)", (h[2 * i + 1] - h[2 * i]) / 1e3, i ? (h[2 * i] - h[2 * i - 1]) / 1e3 : 0.0);
    }
    fprintf(stderr, " | total %.1f us\n", (h[2 * P.n_layers - 1] - h[0]) / 1e3);
  }
  return PP_OK;
}

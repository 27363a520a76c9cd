// Epilogue shared by the wgmma conv kernels: 16 consecutive output channels of one output pixel
// (accumulators already in registers) -> bias / activation / residual / GRU gate fusions -> global memory.
#pragma once
#include "conv_igemm.cuh"
#include "wgmma_ops.cuh"

namespace ppconv {

// ACC (the split-tf32 epilogue): fp32-accurate tanh (pp_common.cuh) instead of the fast-math tanh.approx, whose error is
// below the fp16 storage rounding but far above fp32's
// Works on any run of N values: 16 consecutive channels in conv_epilogue16, a fragment's 4 values in frag_epilogue.
template <int ACT, bool ACC = false, int N>
__device__ __forceinline__ void act16_t(float (&v)[N], float slope) {
#pragma unroll
  for (int i = 0; i < N; ++i) {
    if (ACT == PP_ACT_RELU) v[i] = fmaxf(v[i], 0.f);
    else if (ACT == PP_ACT_LRELU) v[i] = v[i] > 0.f ? v[i] : v[i] * slope;
    else if (ACT == PP_ACT_SIGMOID) v[i] = ppx::sigmoidf_(v[i]);
    else if (ACT == PP_ACT_TANH) v[i] = ACC ? ppx::tanh_acc(v[i]) : tanhf(v[i]);
    else if (ACT == PP_ACT_GELU) v[i] = ppx::gelu_erf(v[i]);
  }
}
// one (uniform) branch per N values instead of one per value
template <bool ACC = false, int N>
__device__ __forceinline__ void act16(float (&v)[N], int act, float slope) {
  switch (act) {
    case PP_ACT_RELU: act16_t<PP_ACT_RELU, ACC>(v, slope); break;
    case PP_ACT_LRELU: act16_t<PP_ACT_LRELU, ACC>(v, slope); break;
    case PP_ACT_SIGMOID: act16_t<PP_ACT_SIGMOID, ACC>(v, slope); break;
    case PP_ACT_TANH: act16_t<PP_ACT_TANH, ACC>(v, slope); break;
    case PP_ACT_GELU: act16_t<PP_ACT_GELU, ACC>(v, slope); break;
    default: break;
  }
}

// 16 consecutive fp16 values <-> registers.  `vec` (uniform per launch, checked on the host) says that full
// runs are 16-byte aligned, so they move as 2 x 16-byte accesses; partial runs take the scalar tail.
__device__ __forceinline__ void load16(const __half* src, int nvalid, bool vec, float (&r)[16]) {
  if (vec && nvalid == 16) {
    const uint4 a = reinterpret_cast<const uint4*>(src)[0], b = reinterpret_cast<const uint4*>(src)[1];
    const __half2* ha = reinterpret_cast<const __half2*>(&a);
    const __half2* hb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 fa = __half22float2(ha[i]), fb = __half22float2(hb[i]);
      r[2 * i] = fa.x; r[2 * i + 1] = fa.y; r[8 + 2 * i] = fb.x; r[8 + 2 * i + 1] = fb.y;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 16; ++i) r[i] = i < nvalid ? __half2float(src[i]) : 0.f;
  }
}
__device__ __forceinline__ void store16(__half* dst, int nvalid, bool vec, const float (&v)[16]) {
  if (vec && nvalid == 16) {
    __align__(16) __half2 h[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    reinterpret_cast<uint4*>(dst)[0] = reinterpret_cast<uint4*>(h)[0];
    reinterpret_cast<uint4*>(dst)[1] = reinterpret_cast<uint4*>(h)[1];
  } else {
#pragma unroll
    for (int i = 0; i < 16; ++i)
      if (i < nvalid) dst[i] = __float2half_rn(v[i]);
  }
}

// `raw`: 16 fp32 accumulators (tile columns ng0-n0 .. +15) of output pixel `mrow` (flattened N*OH*OW index),
// group g, first channel ng0 (within the group; ng0 < Cout_g).  `epi`/`vec` are launch-uniform.
// frag_epilogue (below) repeats this operation order per value for every epilogue kind; keep the two in step, a layer's
// results do not depend on which kernel or epilogue path ran it.
__device__ __forceinline__ void conv_epilogue16(const PPConvParams& p, const uint32_t (&raw)[16], long long mrow, int g,
                                                int ng0, int epi, bool vec) {
    const int nvalid = min(16, p.Cout_g - ng0);
    float v[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = __uint_as_float(raw[i]);
    if (p.bias != nullptr) {
      const float* bp = p.bias + g * p.Cout_g + ng0;
      if (vec && nvalid == 16) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float4 b4 = __ldg(reinterpret_cast<const float4*>(bp) + i);
          v[4 * i] += b4.x; v[4 * i + 1] += b4.y; v[4 * i + 2] += b4.z; v[4 * i + 3] += b4.w;
        }
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i)
          if (i < nvalid) v[i] += __ldg(bp + i);
      }
    }
    if (epi == PP_EPI_STD) {
      act16(v, p.act1, p.slope);
      if (p.scale != 1.f) {
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] *= p.scale;
      }
      if (p.aux0 != nullptr) {
        float r[16];
        load16(p.aux0 + mrow * p.aux0_cstride + p.aux0_coff + ng0, nvalid, vec, r);
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] += r[i];
      }
      act16(v, p.act2, p.slope);
      const long long o = mrow * p.out_cstride + p.out_coff + (long long)g * p.out_gstep + ng0;
      if (p.out_fp32) {
        float* dst = reinterpret_cast<float*>(p.out) + o;
        if (vec && nvalid == 16) {
#pragma unroll
          for (int i = 0; i < 4; ++i)
            reinterpret_cast<float4*>(dst)[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
        } else {
#pragma unroll
          for (int i = 0; i < 16; ++i)
            if (i < nvalid) dst[i] = v[i];
        }
      } else {
        store16(reinterpret_cast<__half*>(p.out) + o, nvalid, vec, v);
      }
    } else if (epi == PP_EPI_GRU_ZR) {
      const int half_c = p.Cout_g >> 1;
      act16_t<PP_ACT_SIGMOID>(v, 0.f);
      if (ng0 < half_c) {
        store16(reinterpret_cast<__half*>(p.out) + mrow * p.out_cstride + p.out_coff + ng0, nvalid, vec, v);
      } else {
        const int c = ng0 - half_c;
        float h[16];
        load16(p.aux0 + mrow * p.aux0_cstride + p.aux0_coff + c, nvalid, vec, h);
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] *= h[i];
        store16(p.out2 + mrow * p.out2_cstride + p.out2_coff + c, nvalid, vec, v);
      }
    } else {  // PP_EPI_GRU_H
      float h[16], z[16];
      load16(p.aux0 + mrow * p.aux0_cstride + p.aux0_coff + ng0, nvalid, vec, h);
      load16(p.aux1 + mrow * p.aux1_cstride + p.aux1_coff + ng0, nvalid, vec, z);
      act16_t<PP_ACT_TANH>(v, 0.f);
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = (1.f - z[i]) * h[i] + z[i] * v[i];
      store16(reinterpret_cast<__half*>(p.out) + mrow * p.out_cstride + p.out_coff + ng0, nvalid, vec, v);
    }
}

// ---- fragment epilogue of the TMA-store kernels (conv_gemm_kernel, conv_halo_kernel's TMA path)
// A consumer warpgroup writes its rows of the tile as fp16 into a staging tile in shared memory, panels of PW channels
// (64 / 32 / 16: 128B / 64B / 32B swizzle), each swizzled like the TMA box that stores it; panel P starts at P * PANEL.

// Thread t128 copies the tile's bias columns 2 t128 and 2 t128 + 1 (bias channels goff + n0 + c, zero past Cout_g) to
// `bs`: one coalesced load per thread instead of a dependent global load per fragment column.  goff: g * Cout_g.
template <int BN>
__device__ __forceinline__ void stage_bias(const PPConvParams& p, float* bs, int goff, int n0, int t128) {
  const int c0 = 2 * t128, n = goff + n0 + c0;
  float2 bv = make_float2(0.f, 0.f);
  if (p.bias != nullptr && c0 < BN) {
    if (n0 + c0 < p.Cout_g) bv.x = __ldg(p.bias + n);
    if (n0 + c0 + 1 < p.Cout_g) bv.y = __ldg(p.bias + n + 1);
  }
  if (c0 < BN) *reinterpret_cast<float2*>(bs + c0) = bv;
}

// Byte offset of (row r, channel c % PW) within a panel: rows of PW * 2 bytes, the box swizzle XORs the 16-byte unit
// index with the row's address bits 7.. (panels start 1024-byte aligned, so panel-relative bits are absolute ones).
template <int PW>
__device__ __forceinline__ int frag_stg_off(int r, int c) {
  return r * PW * 2 + ((((c & (PW - 1)) >> 3) ^ ((r * PW * 2 >> 7) & (PW / 8 - 1))) << 4) + (c & 7) * 2;
}

// The fragment epilogue of one warpgroup into its staging tile `so`, in conv_epilogue16's operation order per value.
// bs: the tile's bias columns (stage_bias).  STD: act1 is ACT1 (p.act1, dispatched once per tile, so the loop over the
// fragments has no indirect branch), act2 is applied when set, and the residual (has_aux) is read from the staging tile
// (TMA-loaded there) and overwritten in place.  GRU_ZR: sigmoid; r tiles multiply by h (in the staging tile).  GRU_H:
// tanh, then (1 - z) h + z q with h in the staging tile and z in the warpgroup's z panel `zb`, which holds one panel at a
// time: panel P of the tile reads it.  Every column of the tile (of panel P for GRU_H) is written, columns past Cout_g
// are never stored, so the loop is straight-line code whose shared-memory accesses the compiler can batch.
template <int MB, int BN, int PW, int PANEL, int EPI, int ACT1>
__device__ __forceinline__ void frag_epilogue(const PPConvParams& p, const float (&acc)[MB][BN / 2], uint8_t* so,
                                              const uint8_t* zb, const float* bs, bool has_aux, bool r_tile, int P,
                                              int t128) {
  const bool has_bias = p.bias != nullptr;
  const float scale = p.scale, slope = p.slope;
  const int act2 = p.act2;
  // fragment of m64nNk16: register 4j + i of thread t holds row 16 * (t / 32) + (t % 32) / 4 + 8 * (i / 2), column
  // 8j + 2 * (t % 4) + i % 2
  const int fr = 16 * (t128 >> 5) + ((t128 & 31) >> 2), fc = 2 * (t128 & 3);
#pragma unroll
  for (int b = 0; b < MB; ++b) {
    const int r = 64 * b + fr;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = 8 * j + fc;
      if (EPI == PP_EPI_GRU_H && col / PW != P) continue;
      // rows r and r + 8 differ above the swizzle's row bits
      const int off = (col / PW) * PANEL + frag_stg_off<PW>(r, col);
      __half2* lo = reinterpret_cast<__half2*>(so + off);
      __half2* hi = reinterpret_cast<__half2*>(so + off + 8 * PW * 2);
      const float2 bias = *reinterpret_cast<const float2*>(bs + col);
      float v[4] = {acc[b][4 * j], acc[b][4 * j + 1], acc[b][4 * j + 2], acc[b][4 * j + 3]};
      float a[4] = {0.f, 0.f, 0.f, 0.f};
      if (has_aux) {
        const float2 a0 = __half22float2(*lo), a1 = __half22float2(*hi);
        a[0] = a0.x; a[1] = a0.y; a[2] = a1.x; a[3] = a1.y;
      }
      if (has_bias) {
        v[0] += bias.x; v[1] += bias.y; v[2] += bias.x; v[3] += bias.y;
      }
      if constexpr (EPI == PP_EPI_STD) {
        act16_t<ACT1>(v, slope);
        if (scale != 1.f) {
#pragma unroll
          for (int i = 0; i < 4; ++i) v[i] *= scale;
        }
        if (has_aux) {
#pragma unroll
          for (int i = 0; i < 4; ++i) v[i] += a[i];
        }
        if (act2 != PP_ACT_NONE) act16(v, act2, slope);
      } else if constexpr (EPI == PP_EPI_GRU_ZR) {
        act16_t<PP_ACT_SIGMOID>(v, 0.f);
        if (r_tile) {
#pragma unroll
          for (int i = 0; i < 4; ++i) v[i] *= a[i];
        }
      } else {
        const int zoff = frag_stg_off<PW>(r, col);
        const float2 z0 = __half22float2(*reinterpret_cast<const __half2*>(zb + zoff));
        const float2 z1 = __half22float2(*reinterpret_cast<const __half2*>(zb + zoff + 8 * PW * 2));
        const float z[4] = {z0.x, z0.y, z1.x, z1.y};
        act16_t<PP_ACT_TANH>(v, 0.f);
#pragma unroll
        for (int i = 0; i < 4; ++i) v[i] = (1.f - z[i]) * a[i] + z[i] * v[i];
      }
      *lo = __floats2half2_rn(v[0], v[1]);
      *hi = __floats2half2_rn(v[2], v[3]);
    }
  }
}

// ---- split-tf32 form (PPConvParams::split): fp32 [hi | lo] operands, see conv_igemm.cuh
// 16 consecutive channels x = hi + lo of a split tensor (hi at src, lo `lo` floats further)
__device__ __forceinline__ void load16_split(const float* src, int lo, int nvalid, bool vec, float (&r)[16]) {
  if (vec && nvalid == 16) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float4 h = reinterpret_cast<const float4*>(src)[i], l = reinterpret_cast<const float4*>(src + lo)[i];
      r[4 * i] = h.x + l.x; r[4 * i + 1] = h.y + l.y; r[4 * i + 2] = h.z + l.z; r[4 * i + 3] = h.w + l.w;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 16; ++i) r[i] = i < nvalid ? src[i] + src[lo + i] : 0.f;
  }
}
__device__ __forceinline__ void store16_split(float* dst, int lo, int nvalid, bool vec, const float (&v)[16]) {
  float h[16], l[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) { h[i] = ppx::tf32_rna(v[i]); l[i] = v[i] - h[i]; }
  if (vec && nvalid == 16) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      reinterpret_cast<float4*>(dst)[i] = make_float4(h[4 * i], h[4 * i + 1], h[4 * i + 2], h[4 * i + 3]);
      reinterpret_cast<float4*>(dst + lo)[i] = make_float4(l[4 * i], l[4 * i + 1], l[4 * i + 2], l[4 * i + 3]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 16; ++i)
      if (i < nvalid) { dst[i] = h[i]; dst[lo + i] = l[i]; }
  }
}

// conv_epilogue16 of the split-tf32 form: the same three epilogue kinds; auxiliary operands are read as hi + lo, results
// are written as hi / lo pairs (or plain fp32 with out_fp32).
__device__ __forceinline__ void conv_epilogue16_split(const PPConvParams& p, const float (&acc)[16], long long mrow, int g,
                                                      int ng0, bool vec) {
  const int nvalid = min(16, p.Cout_g - ng0);
  float v[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = acc[i];
  if (p.bias != nullptr) {
    const float* bp = p.bias + g * p.Cout_g + ng0;
#pragma unroll
    for (int i = 0; i < 16; ++i)
      if (i < nvalid) v[i] += __ldg(bp + i);
  }
  const float* aux0 = reinterpret_cast<const float*>(p.aux0);
  const float* aux1 = reinterpret_cast<const float*>(p.aux1);
  float* out = reinterpret_cast<float*>(p.out);
  if (p.epi == PP_EPI_STD) {
    act16<true>(v, p.act1, p.slope);
    if (p.scale != 1.f) {
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] *= p.scale;
    }
    if (aux0 != nullptr) {
      float r[16];
      load16_split(aux0 + mrow * p.aux0_cstride + p.aux0_coff + ng0, p.aux0_lo, nvalid, vec, r);
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] += r[i];
    }
    act16<true>(v, p.act2, p.slope);
    float* dst = out + mrow * p.out_cstride + p.out_coff + (long long)g * p.out_gstep + ng0;
    if (p.out_fp32) {
      if (vec && nvalid == 16) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
          reinterpret_cast<float4*>(dst)[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i)
          if (i < nvalid) dst[i] = v[i];
      }
    } else {
      store16_split(dst, p.out_lo, nvalid, vec, v);
    }
  } else if (p.epi == PP_EPI_GRU_ZR) {
    const int half_c = p.Cout_g >> 1;
    act16_t<PP_ACT_SIGMOID, true>(v, 0.f);
    if (ng0 < half_c) {
      store16_split(out + mrow * p.out_cstride + p.out_coff + ng0, p.out_lo, nvalid, vec, v);
    } else {
      const int c = ng0 - half_c;
      float h[16];
      load16_split(aux0 + mrow * p.aux0_cstride + p.aux0_coff + c, p.aux0_lo, nvalid, vec, h);
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] *= h[i];
      store16_split(reinterpret_cast<float*>(p.out2) + mrow * p.out2_cstride + p.out2_coff + c, p.out2_lo, nvalid, vec, v);
    }
  } else {  // PP_EPI_GRU_H
    float h[16], z[16];
    load16_split(aux0 + mrow * p.aux0_cstride + p.aux0_coff + ng0, p.aux0_lo, nvalid, vec, h);
    load16_split(aux1 + mrow * p.aux1_cstride + p.aux1_coff + ng0, p.aux1_lo, nvalid, vec, z);
    act16_t<PP_ACT_TANH, true>(v, 0.f);
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = (1.f - z[i]) * h[i] + z[i] * v[i];
    store16_split(out + mrow * p.out_cstride + p.out_coff + ng0, p.out_lo, nvalid, vec, v);
  }
}

// ---- accumulator hand-off for the wgmma kernels
// A warpgroup's m64 x N accumulator is spread over its 128 threads in the wgmma fragment layout (pp_common.cuh); the
// epilogue wants 16 consecutive channels of one pixel per thread.  Per 32-column chunk the warpgroup writes its
// fragments into a [64][STG_LD] fp32 staging tile, meets on a named barrier, and thread t takes row t / 2, columns
// 16 * (t % 2) .. +15 of the chunk.
constexpr int STG_LD = 40;                  // floats per row: the float2 writes of a half-warp hit 32 distinct banks
constexpr int STG_BYTES = 64 * STG_LD * 4;  // per warpgroup

// `emit(src, r, c)`: 16 fp32 values at `src` are columns c .. c+15 of row r (0..63) of the accumulator.  The chunk loop
// is a runtime loop (one inlined copy of the epilogue); only the register -> staging copy is unrolled per chunk.
template <int N, class Emit>
__device__ __forceinline__ void drain_acc(const float (&acc)[N / 2], float* stg, int t128, int bar_id, Emit&& emit) {
  const int wrow = 16 * (t128 >> 5) + ((t128 & 31) >> 2), wcol = 2 * (t128 & 3);
#pragma unroll 1
  for (int c0 = 0; c0 < N; c0 += 32) {
#pragma unroll
    for (int cc = 0; cc < N; cc += 32) {
      if (cc == c0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (cc + 8 * j < N) {
            const int i = (cc / 8 + j) * 4;
            *reinterpret_cast<float2*>(stg + wrow * STG_LD + 8 * j + wcol) = make_float2(acc[i], acc[i + 1]);
            *reinterpret_cast<float2*>(stg + (wrow + 8) * STG_LD + 8 * j + wcol) = make_float2(acc[i + 2], acc[i + 3]);
          }
        }
      }
    }
    ppx::named_bar(bar_id, 128);
    const int c = c0 + 16 * (t128 & 1);
    if (c < N) emit(stg + (t128 >> 1) * STG_LD + 16 * (t128 & 1), t128 >> 1, c);
    ppx::named_bar(bar_id, 128);
  }
}

// conv_epilogue16 (SPLIT: conv_epilogue16_split) on 16 staged accumulators.  EPI >= 0: the layer's epilogue kind, known
// at compile time (only that branch of conv_epilogue16 is generated); -1: p.epi at run time.
template <bool SPLIT = false, int EPI = -1>
__device__ __forceinline__ void epilogue_from_stage(const PPConvParams& p, const float* src, long long mrow, int g, int ng0) {
  if constexpr (SPLIT) {
    float acc[16];
#pragma unroll
    for (int i = 0; i < 16; i += 4) {
      const float4 v = *reinterpret_cast<const float4*>(src + i);
      acc[i] = v.x; acc[i + 1] = v.y; acc[i + 2] = v.z; acc[i + 3] = v.w;
    }
    conv_epilogue16_split(p, acc, mrow, g, ng0, p.vec_ok != 0);
  } else {
    uint32_t raw[16];
#pragma unroll
    for (int i = 0; i < 16; i += 4) {
      const float4 v = *reinterpret_cast<const float4*>(src + i);
      raw[i] = __float_as_uint(v.x); raw[i + 1] = __float_as_uint(v.y);
      raw[i + 2] = __float_as_uint(v.z); raw[i + 3] = __float_as_uint(v.w);
    }
    conv_epilogue16(p, raw, mrow, g, ng0, EPI >= 0 ? EPI : p.epi, p.vec_ok != 0);
  }
}

// f(IntC<BN>{}) for the runtime tile width bn (a multiple of 16, at most MAX_N)
template <int V>
struct IntC { static constexpr int value = V; };
template <int MAX_N, class F>
__device__ __forceinline__ void with_tile_width(int bn, F&& f) {
  switch (bn) {
    case 16: f(IntC<16>{}); break;
    case 32: f(IntC<32>{}); break;
    case 48: f(IntC<48>{}); break;
    case 64: f(IntC<64>{}); break;
    case 80: f(IntC<80>{}); break;
    case 96: f(IntC<96>{}); break;
    case 112: f(IntC<112>{}); break;
    case 128: f(IntC<128>{}); break;
    default:
      if constexpr (MAX_N > 128) {
        switch (bn) {
          case 144: f(IntC<144>{}); break;
          case 160: f(IntC<160>{}); break;
          case 176: f(IntC<176>{}); break;
          case 192: f(IntC<192>{}); break;
          case 208: f(IntC<208>{}); break;
          case 224: f(IntC<224>{}); break;
          case 240: f(IntC<240>{}); break;
          case 256: f(IntC<256>{}); break;
          default: __trap();
        }
      } else {
        __trap();
      }
  }
}

}  // namespace ppconv

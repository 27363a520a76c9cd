// Implicit-GEMM convolution / linear layer on Hopper tensor cores (wgmma, sm_90a).
//
//   out[m][n] = epilogue( sum_k A[m][k] * Wt[n][k] + bias[n] )
//   m = (image, oy, ox) flattened, n = output channel, k = (ky, kx, ci)
//
// Activations are NHWC fp16 with channel strides that are multiples of 8 (16 B), so every 16-byte
// im2col vector lies inside one filter tap.  A conv input may be the channel-concatenation of up to
// PP_MAX_SEGS tensors (segments): the torch.cat calls of the reference become address arithmetic here.
//
// Split-tf32 form (PPConvParams::split = 1, the fp32 RAFT path): every activation tensor is fp32 and stores each
// channel as a pair hi = tf32(x), lo = x - hi, the hi values of the C channels of a pixel followed by the lo values
// ([pix][hi C | lo C], hi + lo == x exactly).  A conv reads the segments (hi, lo, hi) against a weight image whose K rows
// are [W_hi; W_hi; W_lo], so one tf32 GEMM computes hi*W_hi + lo*W_hi + hi*W_lo ~ x*W to ~2^-21 (3xTF32).  The
// producers only move bytes: segment fields, Cin and the weight image are given in 2-byte units (a 128-byte K-chunk row
// holds 32 fp32 values instead of 64 fp16), and only the MMA instruction and the epilogue differ.
#pragma once
#include <cuda.h>

#include "pp_common.cuh"

enum PPAct : int { PP_ACT_NONE = 0, PP_ACT_RELU = 1, PP_ACT_LRELU = 2, PP_ACT_SIGMOID = 3, PP_ACT_TANH = 4,
                   PP_ACT_GELU = 5 };

enum PPEpi : int {
  PP_EPI_STD = 0,      // v = act2( act1(acc + bias) * scale + residual )
  PP_EPI_GRU_ZR = 1,   // n < half: z = sigmoid(v) -> out ; n >= half: r = sigmoid(v), out2 = r * h
  PP_EPI_GRU_H = 2,    // q = tanh(v); out = (1 - z) * h + z * q   (h = aux0, z = aux1)
};

struct PPConvSeg {
  const __half* ptr;
  int cstride;   // elements between consecutive pixels
  int coff;      // first channel of this segment inside the pixel
  int gstep;     // added to coff per group index
  int cbegin;    // first conv-input channel (per group) covered by this segment
  int cend;      // one past the last conv-input channel covered (multiple of 8)
  int cvalid;    // 0, or the number of channels that really exist in memory (< cend - cbegin): the rest read as
                 // zero (TMA out-of-bounds fill; halo kernel only) -- lets a 32-channel tensor feed 64-wide K chunks
};

constexpr int PP_MAX_SEGS = 6;   // gru.q of the split-tf32 path: (r*h, x) x (hi, lo, hi)

struct PPConvParams {
  PPConvSeg seg[PP_MAX_SEGS];
  int nseg;
  int N, H, W, OH, OW;
  int Cin;                // per-group input channels as seen by the kernel (multiple of 8)
  int kh, kw, sh, sw, ph, pw, dh, dw;
  int pad_replicate;      // 0: zeros outside, 1: clamp coordinates (replicate padding)
  int K_total;            // kh*kw*Cin
  int num_kc;             // ceil(K_total / 64)
  int M_total;            // N*OH*OW
  const __half* wpacked;  // [groups][num_kc][Cout_g_pad] rows of 64 fp16, 128B-swizzled tile image
  const float* bias;      // [groups*Cout_g] or nullptr
  int Cout_g, Cout_g_pad, BN, groups;
  int stages;
  int vec_ok;             // set by the launcher: every epilogue pointer/stride allows 16-byte accesses on full runs
  // epilogue
  int epi, act1, act2;
  float slope, scale;
  void* out; int out_cstride, out_coff, out_gstep, out_fp32;
  const __half* aux0; int aux0_cstride, aux0_coff;   // residual (STD) or h (GRU)
  const __half* aux1; int aux1_cstride, aux1_coff;   // z (GRU_H)
  __half* out2; int out2_cstride, out2_coff;          // r*h destination (GRU_ZR)
  // split-tf32 form (see above): 1 = tf32 MMAs; out / aux0 / aux1 / out2 are fp32 [hi | lo] tensors whose lo value of a
  // channel lies *_lo floats after its hi value (strides and offsets in floats).  out_fp32 = 1 writes plain fp32 instead.
  int split;
  int out_lo, aux0_lo, aux1_lo, out2_lo;
};

int pp_launch_conv(const PPConvParams& p, cudaStream_t stream);
// The tile plan of a conv launch, as the launchers chose it (read back by pp_op_conv_last_plan, so that tests can show
// which kernel branch a case ran).
struct PPConvPlan {
  char kind;     // 'g' flat GEMM kernel, 'h' TMA halo-tile kernel, 'i' cp.async implicit GEMM, 'p' recorded into a
                 // multi-layer program, '?' none yet
  int m;         // halo: MT (128-pixel sub-tiles per CTA tile); gemm: MB (m64 blocks per consumer warpgroup); else 0
  int bn;        // N tile width
  int tps;       // halo: filter taps per weight stage; else 0
  int flat;      // halo: 1x1 flat mode (gemm: always 1)
  int tma_out;   // fragment epilogue + TMA stores (gemm: always 1)
  int sa, sb;    // stages of the A (patch / im2col) and B (weight) rings; igemm / gemm: one ring, sb = sa
};
// the plan of the last pp_launch_conv of this thread; the launchers fill it in
PPConvPlan& pp_last_conv_plan();
// which kernel the last pp_launch_conv of this thread went to (PPConvPlan::kind; profiling labels)
inline char pp_last_conv_kind() { return pp_last_conv_plan().kind; }
// conv_halo.cu: TMA halo-tile kernel for stride-1 convolutions (dispatched from pp_launch_conv when eligible).
// `p` must already carry num_kc / vec_ok.
int pp_conv_halo_eligible(const PPConvParams& p);
int pp_launch_conv_halo(const PPConvParams& p, cudaStream_t stream);
// conv_gemm.cu: wide-tile GEMM kernel for 1x1 convolutions and linear layers with the plain fp16 epilogue (dispatched
// from pp_launch_conv ahead of the halo kernel when eligible).  `p` must already carry num_kc / M_total / vec_ok.
int pp_conv_gemm_eligible(const PPConvParams& p);
int pp_launch_conv_gemm(const PPConvParams& p, cudaStream_t stream);

// ---- host plumbing of the conv kernels (conv_igemm.cu, next to pp_launch_conv)
// SM count of the current device, queried once.
int pp_num_sms(int* n);
// cuTensorMapEncodeTiled is available: the halo and GEMM kernels load their operands with TMA.
bool pp_tmap_supported();
// TMA tensor maps (fp16, 128B swizzle) of the input segments, boxes of 64 channels x bw x bh pixels; flat: the N*H*W
// pixels as one dimension.  And a 2-D [rows][cols] map with row stride `ld` and 64 x box_rows boxes.
int pp_conv_input_tmaps(const PPConvParams& p, int bw, int bh, bool flat, CUtensorMap* maps);
int pp_tmap_2d_f16(CUtensorMap* map, const __half* base, int cols, long long rows, int ld, int box_rows);
// A 4-D [n][h][w][cols] map of a pixel tensor with `cstride` elements per pixel (flat: w pixels, h = n = 1), boxes of
// box_c channels (64, 32 or 16: 128B, 64B or 32B swizzle) x box_w x box_h pixels.
int pp_tmap_pixels_f16(CUtensorMap* map, const __half* base, int cols, int cstride, long long w, int h, int n, int box_c,
                       int box_w, int box_h);
// 1 when PP_CONV_NOEPI=1 is set: the halo and GEMM kernels skip the epilogue math and stores (main-loop-only timing)
int pp_conv_noepi();

// The TMA kernels load 64-channel K chunks from one segment each, so no chunk may straddle two segments: every segment
// starts on a chunk boundary, and only the last segment of a flat (1x1) layer may end inside one (TMA zero-fills the
// ragged channel tail).
inline bool pp_conv_segs_chunked(const PPConvParams& p, bool flat) {
  for (int i = 0; i < p.nseg; ++i) {
    if (p.seg[i].cbegin % 64 != 0) return false;
    if (p.seg[i].cend % 64 != 0 && !(flat && i == p.nseg - 1)) return false;
  }
  return true;
}

// An fp16 pixel tensor (base pointer, elements per pixel, first channel) whose every pixel's channel run starts 16-byte
// aligned, as TMA loads and stores of its rows need.
inline bool aligned16(const void* ptr, int cstride, int coff) {
  return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && cstride % 8 == 0 && coff % 8 == 0;
}

// The segment that holds conv-input channel `ci`.
__device__ __forceinline__ int pp_seg_of(const PPConvParams& p, int ci) {
  int q = 0;
#pragma unroll
  for (int t = 1; t < PP_MAX_SEGS; ++t)
    if (t < p.nseg && ci >= p.seg[t].cbegin) q = t;
  return q;
}

// A persistent conv kernel launch (1-D grid) with programmatic dependent launch: the kernel's griddepcontrol.wait
// orders its reads after the previous kernel in the stream.
template <class Params>
int pp_conv_launch(void (*kernel)(Params), const Params& params, int grid, int threads, size_t smem_bytes,
                   cudaStream_t stream) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  PP_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, params));
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

// Multi-layer programs (conv_halo.cu): between pp_prog_begin() and pp_prog_end() every eligible convolution handed to
// pp_launch_conv and every pp_k_dcn_sample call of this thread is RECORDED instead of launched; pp_prog_end launches
// the recorded, mutually dependent layers as ONE persistent kernel with grid-wide barriers between them.
struct PPDcnArgs;
struct PPProgRecorder;
bool pp_prog_recording();
int pp_prog_begin();
void pp_prog_abort();
int pp_prog_record_conv(const PPConvParams& p);
int pp_prog_record_dcn(const PPDcnArgs& a);
int pp_prog_end(unsigned int* counter, unsigned int* arrivals, cudaStream_t stream);

// Sparse-transformer support kernels: LayerNorm, pooled tokens, window flags, fold (overlap-add),
// max-pool of masks, host-composite replacement.  The windowed attention itself is in attention.cu.
#include "kernels.cuh"

namespace {

constexpr int TPB = 256;
inline int nblocks(long long n, int per = TPB) { return (int)((n + per - 1) / per); }

// ------------------------------------------------------------------------------------------------
// LayerNorm over C=512 (nn.LayerNorm, eps 1e-5; sparse_transformer.py:425-431).  One warp per token.
// Rows are re-mapped from the [t][gh][gw] token grid into the zero-padded [t][nh][nw] grid the window
// attention works on (padding tokens stay zero *before* the Q/K/V linears, sparse_transformer.py:212-221).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) layernorm512(const __half* __restrict__ x, const float* __restrict__ gamma,
                                                    const float* __restrict__ beta, __half* __restrict__ out, long long rows,
                                                    int gh, int gw, int nh, int nw) {
  // one warp per row, rows strided by the number of warps in the grid; lane l always owns channels 16l..16l+15, so
  // its gamma / beta values are loaded once into registers instead of once per row (they were 80 % of the L1 traffic)
  const int lane = threadIdx.x & 31;
  const long long warp0 = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  float g[16], bt[16];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 gg = __ldg(reinterpret_cast<const float4*>(gamma) + lane * 4 + i);
    const float4 bb = __ldg(reinterpret_cast<const float4*>(beta) + lane * 4 + i);
    g[4 * i] = gg.x; g[4 * i + 1] = gg.y; g[4 * i + 2] = gg.z; g[4 * i + 3] = gg.w;
    bt[4 * i] = bb.x; bt[4 * i + 1] = bb.y; bt[4 * i + 2] = bb.z; bt[4 * i + 3] = bb.w;
  }
  for (long long row = warp0; row < rows; row += nwarps) {
    const uint4* xp = reinterpret_cast<const uint4*>(x + row * 512) + lane * 2;
    uint4 raw[2] = {xp[0], xp[1]};
    float v[16];
    const __half2* h = reinterpret_cast<const __half2*>(raw);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float2 f = __half22float2(h[i]);
      v[2 * i] = f.x; v[2 * i + 1] = f.y;
      s += f.x + f.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s * (1.f / 512.f);
    // two-pass variance over the values already in registers: E[x^2] - mean^2 cancels catastrophically once
    // |mean| / std reaches ~30 (fp32 sums of x^2 lose the variance in their rounding)
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float a = v[2 * i] - mean, b = v[2 * i + 1] - mean;
      q += a * a + b * b;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q * (1.f / 512.f) + 1e-5f);
    __align__(16) __half2 o2[8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
      o2[i] = __floats2half2_rn((v[2 * i] - mean) * rstd * g[2 * i] + bt[2 * i],
                                (v[2 * i + 1] - mean) * rstd * g[2 * i + 1] + bt[2 * i + 1]);
    long long orow = row;
    if (nh != gh || nw != gw) {
      const int xx = row % gw;
      const long long t = row / gw;
      const int yy = t % gh;
      const long long f = t / gh;
      orow = (f * nh + yy) * nw + xx;
    }
    uint4* op = reinterpret_cast<uint4*>(out + orow * 512) + lane * 2;
    op[0] = reinterpret_cast<uint4*>(o2)[0];
    op[1] = reinterpret_cast<uint4*>(o2)[1];
  }
}

// ------------------------------------------------------------------------------------------------
// Learned depthwise 4x4 stride-4 pooling of the (padded, normalised) tokens (pool_layer,
// sparse_transformer.py:176-180, 294-297).  x [t][nh][nw][C] -> out [t][ph][pw][C]; w [16 taps][C] fp32.
__global__ void __launch_bounds__(256) pool_tokens(const __half* __restrict__ x, const float* __restrict__ w,
                                                   const float* __restrict__ b, __half* __restrict__ out, int nh, int nw,
                                                   int ph, int pw, int C) {
  // one thread per (pooled token, 8-channel vector); w is [16 taps][C] (transposed when registered, engine.py)
  const int C8 = C >> 3;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (unsigned)(ph * pw * C8)) return;
  const int c8 = idx % (unsigned)C8;
  const int r = idx / (unsigned)C8;
  const int px = r % pw, py = r / pw, f = blockIdx.y;
  float acc[8];
  {
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(b + c8 * 8)), b1 = __ldg(reinterpret_cast<const float4*>(b + c8 * 8) + 1);
    acc[0] = b0.x; acc[1] = b0.y; acc[2] = b0.z; acc[3] = b0.w; acc[4] = b1.x; acc[5] = b1.y; acc[6] = b1.z; acc[7] = b1.w;
  }
  const __half* xb = x + (((long long)f * nh + 4 * py) * nw + 4 * px) * C + c8 * 8;
#pragma unroll
  for (int ky = 0; ky < 4; ++ky)
#pragma unroll
    for (int kx = 0; kx < 4; ++kx) {
      const uint4 q = *reinterpret_cast<const uint4*>(xb + (long long)(ky * nw + kx) * C);
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(w + (ky * 4 + kx) * C + c8 * 8));
      const float4 w1 = __ldg(reinterpret_cast<const float4*>(w + (ky * 4 + kx) * C + c8 * 8) + 1);
      const __half2* hq = reinterpret_cast<const __half2*>(&q);
      const float2 v0 = __half22float2(hq[0]), v1 = __half22float2(hq[1]), v2 = __half22float2(hq[2]), v3 = __half22float2(hq[3]);
      acc[0] += w0.x * v0.x; acc[1] += w0.y * v0.y; acc[2] += w0.z * v1.x; acc[3] += w0.w * v1.y;
      acc[4] += w1.x * v2.x; acc[5] += w1.y * v2.y; acc[6] += w1.z * v3.x; acc[7] += w1.w * v3.y;
    }
  __align__(16) __half2 o[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) o[e] = __floats2half2_rn(acc[2 * e], acc[2 * e + 1]);
  *reinterpret_cast<uint4*>(out + (((long long)f * ph + py) * pw + px) * C + c8 * 8) = *reinterpret_cast<uint4*>(o);
}

// Window dispatch flags (propainter.py:417-428 max_pool(7,3,3) of the 1/4-res local masks, then
// sparse_transformer.py:322-326 max over each 5x9 window and sum over local frames):
// flag[w] = 1 if any local-frame mask pixel falls in the receptive field of any token of window w.
// mask4: [T][h4][w4] fp16 values at element stride cs (channel co); sliding window `widx` covers frames
// win_f0[widx] .. +win_lt[widx].  One block per (5x9 token window, sliding window); flags[widx][win].
__global__ void window_flags(const __half* __restrict__ mask4, int cs, int co, const int* __restrict__ win_f0,
                             const int* __restrict__ win_lt, int h4, int w4, int gh, int gw, int nww,
                             int* __restrict__ flags) {
  const int win = blockIdx.x, widx = blockIdx.y;
  const int wy = win / nww, wx = win % nww;
  const int lt = win_lt[widx];
  const __half* mbase = mask4 + (long long)win_f0[widx] * h4 * w4 * cs;
  int any = 0;
  const int per_frame = 5 * 9 * 49;
  for (int i = threadIdx.x; i < lt * per_frame; i += blockDim.x) {
    const int f = i / per_frame;
    int r = i - f * per_frame;
    const int tok = r / 49, tap = r - tok * 49;
    const int ty = wy * 5 + tok / 9, tx = wx * 9 + tok % 9;
    if (ty >= gh || tx >= gw) continue;  // zero padding of the mask grid
    const int y = ty * 3 - 3 + tap / 7, x = tx * 3 - 3 + tap % 7;
    if (y < 0 || y >= h4 || x < 0 || x >= w4) continue;
    if (__half2float(mbase[(((long long)f * h4 + y) * w4 + x) * cs + co]) > 0.f) any = 1;
  }
  any = __syncthreads_or(any);
  if (threadIdx.x == 0) flags[widx * gridDim.x + win] = any;
}

// ------------------------------------------------------------------------------------------------
// Overlap-add of 7x7 stride-3 pad-3 patches (F.fold) in gather form, optionally divided by the overlap
// count (FusionFeedForward, sparse_transformer.py:92-121) and passed through GELU (the reference applies
// GELU after unfold; unfold only copies, and GELU(0)=0 keeps the zero padding, so GELU-then-unfold is
// identical).  x: [t*gh*gw][cs], column (ky*7+kx)*C + c  (weights are permuted to this order when packed).
// out: [t][H][W][C].  One thread per (pixel, 8-channel vector).
// ------------------------------------------------------------------------------------------------
__global__ void fold7x7s3(const __half* __restrict__ x, int cs, __half* __restrict__ out, int t, int H, int W, int C,
                          int gh, int gw, int normalise, int gelu) {
  const int C8 = C / 8;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;   // grid = (x chunks, rows, frames): 32-bit index math
  if (idx >= (unsigned)(W * C8)) return;
  const int c8 = idx % (unsigned)C8, px = idx / (unsigned)C8;
  const int py = blockIdx.y, f = blockIdx.z;
  (void)t;
  // a pixel is covered by at most 3x3 patches (7x7 patches, stride 3): all nine 16-byte loads are issued up front
  // (predicated), then accumulated in the original order (descending token row / column)
  const int ty1 = min((py + 3) / 3, gh - 1), tx1 = min((px + 3) / 3, gw - 1);
  uint4 q[9];
  bool ok[9];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int ty = ty1 - a, ky = py + 3 - 3 * ty;
    const bool vy = ty >= 0 && ky <= 6;
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const int tx = tx1 - b, kx = px + 3 - 3 * tx;
      const bool v = vy && tx >= 0 && kx <= 6;
      ok[a * 3 + b] = v;
      q[a * 3 + b] = make_uint4(0, 0, 0, 0);
      if (v)
        q[a * 3 + b] = *reinterpret_cast<const uint4*>(x + (((long long)f * gh + ty) * gw + tx) * cs +
                                                       (ky * 7 + kx) * C + c8 * 8);
    }
  }
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  int cnt = 0;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    if (!ok[t]) continue;
    const __half2* hq = reinterpret_cast<const __half2*>(&q[t]);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 v = __half22float2(hq[e]);
      acc[2 * e] += v.x;
      acc[2 * e + 1] += v.y;
    }
    ++cnt;
  }
  const float inv = (normalise && cnt > 0) ? 1.f / (float)cnt : 1.f;
  __align__(16) __half2 o[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float a = acc[2 * e] * inv, b = acc[2 * e + 1] * inv;
    if (gelu) { a = ppx::gelu_erf(a); b = ppx::gelu_erf(b); }
    o[e] = __floats2half2_rn(a, b);
  }
  *reinterpret_cast<uint4*>(out + ((((long long)f * H + py) * W + px) * C) + c8 * 8) = *reinterpret_cast<uint4*>(o);
}

// ------------------------------------------------------------------------------------------------
// Device replacement of the host composite (propainter_inference.py:283-307) with identical integer
// semantics: img = trunc((pred+1)/2*255); sel = img*m + orig*(1-m) in uint8; first visit stores, later
// visits store trunc(0.5*prev + 0.5*sel).  `visited[frame]` is updated by the host between launches.
// ------------------------------------------------------------------------------------------------
__global__ void composite(const __half* __restrict__ pred, int pred_cs, const float* __restrict__ masks,
                          const uint8_t* __restrict__ orig, uint8_t* __restrict__ comp,
                          const int* __restrict__ frame_ids, const int* __restrict__ first_visit, int lt,
                          long long HW, int half_math) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)lt * HW) return;
  const int i = idx / HW;
  const long long p = idx - (long long)i * HW;
  const int fr = frame_ids[i];
  const int m = (int)(uint8_t)masks[(long long)fr * HW + p];
  const __half* pr = pred + idx * pred_cs;
  const uint8_t* og = orig + ((long long)fr * HW + p) * 3;
  uint8_t* cp = comp + ((long long)fr * HW + p) * 3;
  const int first = first_visit[i];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    // fp16="disable": the reference holds float32 here.  fp16="enable": (pred + 1) / 2 is evaluated in half on the
    // device and the numpy "* 255" stays half too -- two extra roundings that move ~6 % of the bytes by one
    float v;
    if (half_math) {
      const __half a = __float2half_rn(__half2float(pr[c]) + 1.f);   // half add, round to nearest even
      v = __half2float(__float2half_rn(__half2float(a) * 0.5f * 255.f));   // /2 is exact in half
    } else {
      v = (__half2float(pr[c]) + 1.f) / 2.f * 255.f;
    }
    const uint8_t pu = (uint8_t)(int)v;  // astype(np.uint8): truncation (values are within [0,255])
    const uint8_t sel = (uint8_t)(pu * m + og[c] * (1 - m));
    cp[c] = first ? sel : (uint8_t)(int)((float)cp[c] * 0.5f + (float)sel * 0.5f);
  }
}

}  // namespace

int pp_k_layernorm(const __half* x, const float* gamma, const float* beta, __half* out, long long rows, int gh, int gw,
                   int nh, int nw, cudaStream_t st) {
  if (rows == 0) return PP_OK;
  {
    const long long want = (rows + 7) / 8;                 // 8 rows (warps) per block
    const int grid = (int)(want < 148 * 32 ? want : 148 * 32);   // a few rows per warp: gamma/beta loads amortised
    layernorm512<<<grid, 256, 0, st>>>(x, gamma, beta, out, rows, gh, gw, nh, nw);
  }
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_pool_tokens(const __half* x, const float* w, const float* b, __half* out, int t, int nh, int nw, int ph,
                     int pw, int C, cudaStream_t st) {
  if ((long long)t * ph * pw * C == 0) return PP_OK;
  PP_REQUIRE(C % 8 == 0 && t <= 65535, "pool_tokens: C=%d t=%d", C, t);
  pool_tokens<<<dim3(pp_ceil_div(ph * pw * (C / 8), 256), t), 256, 0, st>>>(x, w, b, out, nh, nw, ph, pw, C);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_window_flags(const __half* mask4, int cs, int co, const int* win_f0, const int* win_lt, int n_windows, int h4,
                      int w4, int gh, int gw, int nwh, int nww, int* flags, cudaStream_t st) {
  window_flags<<<dim3(nwh * nww, n_windows), 256, 0, st>>>(mask4, cs, co, win_f0, win_lt, h4, w4, gh, gw, nww, flags);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_fold(const __half* x, int cs, __half* out, int t, int H, int W, int C, int gh, int gw, int normalise,
              int gelu, cudaStream_t st) {
  PP_REQUIRE(C % 8 == 0 && cs % 8 == 0, "fold: C=%d cs=%d must be multiples of 8", C, cs);
  if ((long long)t * H * W == 0) return PP_OK;
  PP_REQUIRE(H <= 65535 && t <= 65535, "fold: %d rows / %d frames exceed the grid limits", H, t);
  fold7x7s3<<<dim3(pp_ceil_div(W * (C / 8), 256), H, t), 256, 0, st>>>(x, cs, out, t, H, W, C, gh, gw, normalise, gelu);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_composite(const __half* pred, int pred_cs, const float* masks, const uint8_t* orig, uint8_t* comp,
                   const int* frame_ids, const int* first_visit, int lt, int H, int W, int half_math, cudaStream_t st) {
  const long long HW = (long long)H * W;
  composite<<<nblocks(HW * lt), TPB, 0, st>>>(pred, pred_cs, masks, orig, comp, frame_ids, first_visit, lt, HW,
                                              half_math);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

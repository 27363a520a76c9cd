// Device-side pre/post-processing with the reference's integer semantics (SURVEY.md section 8f.1; reference
// utils/image_utils.py:106-290) for both nodes, bit-identical to the host path, PIL's 8-bit bicubic resize included.
#include <math.h>

#include <vector>

#include "kernels.cuh"

namespace {

constexpr int TPB = 256;
inline int nblocks(long long n, int per = TPB) { return (int)((n + per - 1) / per); }

// 8-bit value -> frame value in [-1,1]: float32 u8 / 255, * 2, - 1, each rounded to nearest like the host's
// _stack_to_tensor(...) * 2 - 1 (image_utils.py:95-103); explicit roundings, so --use_fast_math cannot change them
__device__ __forceinline__ float u8_to_pm1(uint8_t q) {
  return __fsub_rn(__fmul_rn(__fdiv_rn((float)q, 255.f), 2.f), 1.f);
}

// IMAGE [T,H,W,3] float 0..1 -> uint8 by *255, clip, truncate (image_utils.py:112) and
// frames [T,3,H,W] = u8/255*2-1 (image_utils.py:186-190)
__global__ void quantize_frames(const float* __restrict__ img, uint8_t* __restrict__ u8, float* __restrict__ frames,
                                long long HW, long long total) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;  // over T*H*W pixels
  if (idx >= total) return;
  const long long t = idx / HW, p = idx - t * HW;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = fminf(fmaxf(__fmul_rn(img[idx * 3 + c], 255.f), 0.f), 255.f);
    const uint8_t q = (uint8_t)(int)v;
    u8[idx * 3 + c] = q;
    frames[(t * 3 + c) * HW + p] = u8_to_pm1(q);
  }
}

// MASK [Tm,H,W] float -> 8-bit ((m*255).clamp(0,255).byte(), image_utils.py:128-134), then N iterations of the
// cross-shaped binary dilation of scipy.ndimage.binary_dilation (== dilation by the L1 ball of radius N, zero
// border), or the > 0.1 threshold when N == 0 (image_utils.py:152-170).  Output float {0,1}, broadcast to T frames.
__global__ void mask_u8(const float* __restrict__ m, uint8_t* __restrict__ nz, long long total) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const float v = fminf(fmaxf(__fmul_rn(m[idx], 255.f), 0.f), 255.f);
  nz[idx] = ((uint8_t)(int)v) != 0 ? 1 : 0;
}

__global__ void dilate_diamond(const uint8_t* __restrict__ nz, float* __restrict__ out, int Tm, int T, int H, int W,
                               int radius) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)T * H * W) return;
  const int x = idx % W;
  long long r = idx / W;
  const int y = r % H;
  const int t = r / H;
  const uint8_t* src = nz + (long long)(Tm == 1 ? 0 : t) * H * W;
  int any = 0;
  for (int dy = -radius; dy <= radius && !any; ++dy) {
    const int yy = y + dy;
    if (yy < 0 || yy >= H) continue;
    const int span = radius - (dy < 0 ? -dy : dy);
    const int x0 = max(0, x - span), x1 = min(W - 1, x + span);
    for (int xx = x0; xx <= x1; ++xx)
      if (src[(long long)yy * W + xx]) { any = 1; break; }
  }
  out[idx] = any ? 1.f : 0.f;
}

// ------------------------------------------------------------------------------------------------
// PIL's bicubic resize of 8-bit images (reference utils/image_utils.py:98-103 -> Image.resize(size), Pillow's
// ImagingResample, 8 bits per channel), bit for bit: a horizontal then a vertical pass, each a convolution with
// per-output-pixel coefficient windows precomputed in double precision (cubic a = -0.5, support 2 * max(scale, 1),
// normalised), quantised to 22-bit fixed point with round-half-away, accumulated in int32 from 1 << 21 and clipped to
// 0..255 after >> 22.  The intermediate image of the first pass is uint8, as in Pillow.
// ------------------------------------------------------------------------------------------------
__global__ void resize_axis_u8(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, long long outer, int in_size,
                               int out_size, long long inner, const int* __restrict__ kk, const int* __restrict__ bounds,
                               int ksize) {
  // tensor viewed as [outer][in_size][inner] -> [outer][out_size][inner]
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= outer * out_size * inner) return;
  const long long i = idx % inner;
  const long long r = idx / inner;
  const int xx = (int)(r % out_size);
  const long long o = r / out_size;
  const int xmin = bounds[2 * xx], xmax = bounds[2 * xx + 1];
  const int* k = kk + (long long)xx * ksize;
  const uint8_t* s = src + (o * in_size + xmin) * inner + i;
  int ss = 1 << 21;
  for (int x = 0; x < xmax; ++x) ss += (int)s[(long long)x * inner] * k[x];
  const int v = ss >> 22;
  dst[idx] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

__global__ void quantize_u8(const float* __restrict__ img, uint8_t* __restrict__ u8, long long n) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = fminf(fmaxf(__fmul_rn(img[i], 255.f), 0.f), 255.f);
  u8[i] = (uint8_t)(int)v;
}

// uint8 [T,H,W,3] -> frames [T,3,H,W] = u8/255*2-1 (image_utils.py:186-190)
__global__ void u8_to_frames(const uint8_t* __restrict__ u8, float* __restrict__ frames, long long HW, long long total) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const long long t = idx / HW, p = idx - t * HW;
#pragma unroll
  for (int c = 0; c < 3; ++c)
    frames[(t * 3 + c) * HW + p] = u8_to_pm1(u8[idx * 3 + c]);
}

// Outpainting canvas (extrapolation + _tensorise, image_utils.py:115-139): the rw x rh frames src [T,rh,rw,3] placed at
// (x0, y0) on a zero pw x ph canvas -> orig [T,ph,pw,3], frames [T,3,ph,pw] = u8/255*2-1, and the band masks [T,1,ph,pw]
// in {0,1}: masks_dilated is 1 outside the window, flow_masks also on the window's outer iw columns / ih rows.
__global__ void outpaint_canvas(const uint8_t* __restrict__ src, uint8_t* __restrict__ orig, float* __restrict__ frames,
                                float* __restrict__ flow_masks, float* __restrict__ masks_dilated, int rw, int rh, int pw,
                                int ph, int x0, int y0, int iw, int ih, long long total) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;  // over T*ph*pw pixels
  if (idx >= total) return;
  const long long HW = (long long)ph * pw, t = idx / HW, p = idx - t * HW;
  const int sy = (int)(p / pw) - y0, sx = (int)(p % pw) - x0;
  const bool in = sx >= 0 && sx < rw && sy >= 0 && sy < rh;
  const bool inner = sx >= iw && sx < rw - iw && sy >= ih && sy < rh - ih;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const uint8_t q = in ? src[((t * rh + sy) * rw + sx) * 3 + c] : 0;
    orig[idx * 3 + c] = q;
    frames[(t * 3 + c) * HW + p] = u8_to_pm1(q);
  }
  flow_masks[idx] = inner ? 0.f : 1.f;
  masks_dilated[idx] = in ? 0.f : 1.f;
}

// uint8 [T,H,W,3] -> float32 / 255 (handle_output, image_utils.py:281-283)
__global__ void u8_to_unit_float(const uint8_t* __restrict__ src, float* __restrict__ dst, long long n) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) dst[i] = __fdiv_rn((float)src[i], 255.f);
}

}  // namespace

int pp_k_quantize_frames(const float* img, uint8_t* u8, float* frames, int T, int H, int W, cudaStream_t st) {
  const long long HW = (long long)H * W, total = HW * T;
  quantize_frames<<<nblocks(total), TPB, 0, st>>>(img, u8, frames, HW, total);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_prepare_masks(const float* mask, int Tm, int T, int H, int W, int iters_flow, int iters_dil, uint8_t* scratch,
                       float* flow_masks, float* masks_dilated, cudaStream_t st) {
  PP_REQUIRE(Tm == 1 || Tm == T, "prepare_masks: mask length %d must be 1 or %d", Tm, T);
  const long long n = (long long)Tm * H * W;
  mask_u8<<<nblocks(n), TPB, 0, st>>>(mask, scratch, n);
  dilate_diamond<<<nblocks((long long)T * H * W), TPB, 0, st>>>(scratch, flow_masks, Tm, T, H, W, iters_flow);
  dilate_diamond<<<nblocks((long long)T * H * W), TPB, 0, st>>>(scratch, masks_dilated, Tm, T, H, W, iters_dil);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

namespace {

// Pillow's precompute_coeffs + normalize_coeffs_8bpc for the bicubic filter over the whole axis (box = full image)
void bicubic_coeffs(int in_size, int out_size, std::vector<int>& kk, std::vector<int>& bounds, int& ksize) {
  auto filt = [](double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
  };
  double scale = (double)in_size / out_size, filterscale = scale;
  if (filterscale < 1.0) filterscale = 1.0;
  const double support = 2.0 * filterscale;
  ksize = (int)ceil(support) * 2 + 1;
  kk.assign((size_t)out_size * ksize, 0);
  bounds.assign((size_t)out_size * 2, 0);
  std::vector<double> w(ksize);
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = 0.0 + (xx + 0.5) * scale, ss = 1.0 / filterscale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      w[x] = filt((x + xmin - center + 0.5) * ss);
      ww += w[x];
    }
    for (int x = 0; x < xmax; ++x) {
      const double v = ww != 0.0 ? w[x] / ww : w[x];
      kk[(size_t)xx * ksize + x] = v < 0 ? (int)(-0.5 + v * (double)(1 << 22)) : (int)(0.5 + v * (double)(1 << 22));
    }
    bounds[2 * xx] = xmin;
    bounds[2 * xx + 1] = xmax;
  }
}

}  // namespace

// src [T][H][W][C] uint8 -> dst [T][OH][OW][C]; tmp holds T*H*OW*C bytes, coef 2*(max(OW,OH)*(ksize+2)) ints (device).
int pp_k_resize_bicubic_u8(const uint8_t* src, uint8_t* dst, uint8_t* tmp, int* coef, size_t coef_ints, int T, int H, int W,
                           int C, int OH, int OW, cudaStream_t st) {
  const uint8_t* cur = src;
  int curW = W;
  size_t used = 0;
  auto pass = [&](const uint8_t* in, uint8_t* out, long long outer, int in_size, int out_size, long long inner) -> int {
    std::vector<int> kk, bounds;
    int ksize = 0;
    bicubic_coeffs(in_size, out_size, kk, bounds, ksize);
    PP_REQUIRE(used + kk.size() + bounds.size() <= coef_ints, "resize: coefficient scratch too small");
    int* dk = coef + used;
    int* db = dk + kk.size();
    used += kk.size() + bounds.size();
    PP_CUDA_CHECK(cudaMemcpyAsync(dk, kk.data(), kk.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    PP_CUDA_CHECK(cudaMemcpyAsync(db, bounds.data(), bounds.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    PP_CUDA_CHECK(cudaStreamSynchronize(st));    // the host vectors go out of scope (pageable async copies are staged, but be explicit)
    const long long n = outer * out_size * inner;
    resize_axis_u8<<<nblocks(n), TPB, 0, st>>>(in, out, outer, in_size, out_size, inner, dk, db, ksize);
    PP_CUDA_CHECK(cudaGetLastError());
    return PP_OK;
  };
  if (OW != W) {   // horizontal pass first, like Pillow
    uint8_t* out = (OH != H) ? tmp : dst;
    PP_TRY(pass(cur, out, (long long)T * H, W, OW, C));
    cur = out;
    curW = OW;
  }
  if (OH != H) PP_TRY(pass(cur, dst, T, H, OH, (long long)curW * C));
  if (OW == W && OH == H) PP_CUDA_CHECK(cudaMemcpyAsync(dst, src, (size_t)T * H * W * C, cudaMemcpyDeviceToDevice, st));
  return PP_OK;
}

int pp_k_quantize_u8(const float* img, uint8_t* u8, long long n, cudaStream_t st) {
  quantize_u8<<<nblocks(n), TPB, 0, st>>>(img, u8, n);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_u8_to_frames(const uint8_t* u8, float* frames, int T, int H, int W, cudaStream_t st) {
  const long long HW = (long long)H * W, total = HW * T;
  u8_to_frames<<<nblocks(total), TPB, 0, st>>>(u8, frames, HW, total);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

// dilations straight from an 8-bit mask image (non-zero = set), e.g. the resized mask
int pp_k_dilate_masks_u8(const uint8_t* mask_u8, int Tm, int T, int H, int W, int iters_flow, int iters_dil,
                         float* flow_masks, float* masks_dilated, cudaStream_t st) {
  PP_REQUIRE(Tm == 1 || Tm == T, "prepare_masks: mask length %d must be 1 or %d", Tm, T);
  dilate_diamond<<<nblocks((long long)T * H * W), TPB, 0, st>>>(mask_u8, flow_masks, Tm, T, H, W, iters_flow);
  dilate_diamond<<<nblocks((long long)T * H * W), TPB, 0, st>>>(mask_u8, masks_dilated, Tm, T, H, W, iters_dil);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

// window [T,rh,rw,3] uint8 (0 < rw <= pw, 0 < rh <= ph) centred on the pw x ph canvas like extrapolation
// (image_utils.py:120-130): offsets int((pw - rw) / 2), int((ph - rh) / 2); the flow mask's 4-px inset only on the axes
// whose band is wider than 10 px
int pp_k_outpaint_canvas(const uint8_t* window, int T, int rw, int rh, int pw, int ph, uint8_t* orig, float* frames,
                         float* flow_masks, float* masks_dilated, cudaStream_t st) {
  const int x0 = (pw - rw) / 2, y0 = (ph - rh) / 2;
  const int iw = x0 > 10 ? 4 : 0, ih = y0 > 10 ? 4 : 0;
  const long long total = (long long)T * ph * pw;
  outpaint_canvas<<<nblocks(total), TPB, 0, st>>>(window, orig, frames, flow_masks, masks_dilated, rw, rh, pw, ph, x0, y0,
                                                  iw, ih, total);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_u8_to_unit_float(const uint8_t* src, float* dst, long long n, cudaStream_t st) {
  u8_to_unit_float<<<nblocks(n), TPB, 0, st>>>(src, dst, n);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

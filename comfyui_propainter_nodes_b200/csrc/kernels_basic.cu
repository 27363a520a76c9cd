// Layout conversion and small elementwise kernels (HBM-bound, coalesced / vectorised).
#include "kernels.cuh"

namespace {

constexpr int TPB = 256;
inline int nblocks(long long n, int per = TPB) { return (int)((n + per - 1) / per); }

// NCHW fp32 -> NHWC fp16 into a channel slice [co, co+C) of a pixel of dst_cs elements; channels
// [co+C, co+zero_to) are zero-filled (padding channels must be finite for the tensor-core path).
__global__ void nchw_f32_to_nhwc_f16(const float* __restrict__ src, __half* __restrict__ dst, int C, long long HW,
                                     long long npix, int dst_cs, int dst_co, int zero_to) {
  long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const long long n = p / HW, hw = p - n * HW;
  __half* d = dst + p * dst_cs + dst_co;
  const float* s = src + n * C * HW + hw;
  for (int c = 0; c < C; ++c) d[c] = __float2half_rn(s[c * HW]);
  for (int c = C; c < zero_to; ++c) d[c] = __float2half_rn(0.f);
}

// Bilinear x2 upsample, align_corners=True (reference deconv: F.interpolate(scale_factor=2, 'bilinear', True)).
// One thread per (2x2 block of output pixels, 8-channel vector).  With scale (H-1)/(2H-1) < 1/2 the outputs of block
// (r, c) interpolate between input rows (r-1, r) / (r, r+1) and columns (c-1, c) / (c, c+1): interior blocks load and
// convert the 3x3 neighbourhood once (9 loads for 4 outputs); blocks where the floor() of a source coordinate is not
// the canonical one (image borders, float rounding) take the generic 4-loads-per-output path.  Per output the
// arithmetic is w00*a + w01*b + w10*c + w11*d in fp32 with one rounding on both paths.
// grid = (x chunks, block rows, images): all index math is 32-bit.
__device__ __forceinline__ void up8(const uint4& q, float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&q);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 t = __half22float2(h[e]);
    f[2 * e] = t.x; f[2 * e + 1] = t.y;
  }
}
__device__ __forceinline__ void up_store(__half* dp, const float (&a)[8], const float (&b)[8], const float (&c)[8],
                                         const float (&d)[8], float ly, float lx) {
  const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
  __align__(16) __half2 o[4];
#pragma unroll
  for (int e = 0; e < 4; ++e)
    o[e] = __floats2half2_rn(w00 * a[2 * e] + w01 * b[2 * e] + w10 * c[2 * e] + w11 * d[2 * e],
                             w00 * a[2 * e + 1] + w01 * b[2 * e + 1] + w10 * c[2 * e + 1] + w11 * d[2 * e + 1]);
  *reinterpret_cast<uint4*>(dp) = *reinterpret_cast<uint4*>(o);
}
__global__ void __launch_bounds__(256) upsample2x_ac(const __half* __restrict__ src, int src_cs, int src_co,
                                                     __half* __restrict__ dst, int dst_cs, int dst_co, int H, int W, int C8) {
  const int OW = 2 * W, OH = 2 * H;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (unsigned)(W * C8)) return;
  const int c8 = idx % (unsigned)C8, c = idx / (unsigned)C8;   // block column
  const int r = blockIdx.y, n = blockIdx.z;                    // block row, image
  const float sy = OH > 1 ? (float)(H - 1) / (float)(OH - 1) : 0.f;
  const float sx = OW > 1 ? (float)(W - 1) / (float)(OW - 1) : 0.f;
  const float fy0 = sy * (float)(2 * r), fy1 = sy * (float)(2 * r + 1);
  const float fx0 = sx * (float)(2 * c), fx1 = sx * (float)(2 * c + 1);
  const int ay0 = (int)fy0, ay1 = (int)fy1, ax0 = (int)fx0, ax1 = (int)fx1;
  const __half* base = src + (long long)n * H * W * src_cs + src_co + c8 * 8;
  __half* dbase = dst + (long long)n * OH * OW * dst_cs + dst_co + c8 * 8;
  if (ay0 == r - 1 && ay1 == r && r + 1 < H && ax0 == c - 1 && ax1 == c && c + 1 < W && r > 0 && c > 0) {
    float v[3][3][8];
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int i = 0; i < 3; ++i)
        up8(*reinterpret_cast<const uint4*>(base + (long long)((r - 1 + j) * W + (c - 1 + i)) * src_cs), v[j][i]);
    const float ly0 = fy0 - (float)ay0, ly1 = fy1 - (float)ay1, lx0 = fx0 - (float)ax0, lx1 = fx1 - (float)ax1;
    __half* d0 = dbase + ((long long)(2 * r) * OW + 2 * c) * dst_cs;
    up_store(d0, v[0][0], v[0][1], v[1][0], v[1][1], ly0, lx0);
    up_store(d0 + dst_cs, v[0][1], v[0][2], v[1][1], v[1][2], ly0, lx1);
    up_store(d0 + (long long)OW * dst_cs, v[1][0], v[1][1], v[2][0], v[2][1], ly1, lx0);
    up_store(d0 + (long long)(OW + 1) * dst_cs, v[1][1], v[1][2], v[2][1], v[2][2], ly1, lx1);
    return;
  }
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const float fy = dy ? fy1 : fy0, fx = dx ? fx1 : fx0;
      const int y0 = dy ? ay1 : ay0, x0 = dx ? ax1 : ax0;
      const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
      float a[8], b[8], cc[8], d[8];
      up8(*reinterpret_cast<const uint4*>(base + (long long)(y0 * W + x0) * src_cs), a);
      up8(*reinterpret_cast<const uint4*>(base + (long long)(y0 * W + x1) * src_cs), b);
      up8(*reinterpret_cast<const uint4*>(base + (long long)(y1 * W + x0) * src_cs), cc);
      up8(*reinterpret_cast<const uint4*>(base + (long long)(y1 * W + x1) * src_cs), d);
      up_store(dbase + ((long long)(2 * r + dy) * OW + 2 * c + dx) * dst_cs, a, b, cc, d, fy - (float)y0, fx - (float)x0);
    }
}

// The split-tf32 form (fp32 flow completion): x = hi + lo in, tf32(y) | y - tf32(y) out.  One thread per (output pixel,
// 4-channel vector); ATen's CPU bilinear order h0 * (w0 * a + w1 * b) + h1 * (w0 * c + w1 * d) with source index
// (H-1)/(2H-1) * o, lambda = src - floor(src), every product and sum rounded on its own.
__device__ __forceinline__ float4 ld_split4(const float* p, int C) {
  const float4 h = *reinterpret_cast<const float4*>(p), l = *reinterpret_cast<const float4*>(p + C);
  return make_float4(__fadd_rn(h.x, l.x), __fadd_rn(h.y, l.y), __fadd_rn(h.z, l.z), __fadd_rn(h.w, l.w));
}
__device__ __forceinline__ float lerp_rn(float a, float b, float w0, float w1) {
  return __fadd_rn(__fmul_rn(w0, a), __fmul_rn(w1, b));
}
__global__ void __launch_bounds__(256) upsample2x_split(const float* __restrict__ src, float* __restrict__ dst, int H,
                                                        int W, int C) {
  const int OW = 2 * W, OH = 2 * H, C4 = C / 4;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (unsigned)(OW * C4)) return;
  const int c4 = idx % (unsigned)C4, ox = idx / (unsigned)C4;
  const int oy = blockIdx.y, n = blockIdx.z;
  const float sy = (float)(H - 1) / (float)(OH - 1), sx = (float)(W - 1) / (float)(OW - 1);
  const float fy = __fmul_rn(sy, (float)oy), fx = __fmul_rn(sx, (float)ox);
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
  const float h1 = fminf(fmaxf(__fsub_rn(fy, (float)y0), 0.f), 1.f), w1 = fminf(fmaxf(__fsub_rn(fx, (float)x0), 0.f), 1.f);
  const float h0 = __fsub_rn(1.f, h1), w0 = __fsub_rn(1.f, w1);
  const float* base = src + (long long)n * H * W * 2 * C + 4 * c4;
  const float4 a = ld_split4(base + (long long)(y0 * W + x0) * 2 * C, C);
  const float4 b = ld_split4(base + (long long)(y0 * W + x1) * 2 * C, C);
  const float4 c = ld_split4(base + (long long)(y1 * W + x0) * 2 * C, C);
  const float4 d = ld_split4(base + (long long)(y1 * W + x1) * 2 * C, C);
  const float r[4] = {
      lerp_rn(lerp_rn(a.x, b.x, w0, w1), lerp_rn(c.x, d.x, w0, w1), h0, h1),
      lerp_rn(lerp_rn(a.y, b.y, w0, w1), lerp_rn(c.y, d.y, w0, w1), h0, h1),
      lerp_rn(lerp_rn(a.z, b.z, w0, w1), lerp_rn(c.z, d.z, w0, w1), h0, h1),
      lerp_rn(lerp_rn(a.w, b.w, w0, w1), lerp_rn(c.w, d.w, w0, w1), h0, h1)};
  float hi[4], lo[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) { hi[e] = ppx::tf32_rna(r[e]); lo[e] = __fsub_rn(r[e], hi[e]); }
  float* dp = dst + ((long long)n * OH * OW + (long long)oy * OW + ox) * 2 * C + 4 * c4;
  *reinterpret_cast<float4*>(dp) = make_float4(hi[0], hi[1], hi[2], hi[3]);
  *reinterpret_cast<float4*>(dp + C) = make_float4(lo[0], lo[1], lo[2], lo[3]);
}

// dst block j <- src block idx[j]; blocks are `block16` 16-byte units (frame-sized gathers for window batching)
__global__ void gather_blocks(uint4* __restrict__ dst, const uint4* __restrict__ src, const int* __restrict__ idx,
                              long long n, long long block16) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n * block16) return;
  const long long j = i / block16, u = i - j * block16;
  dst[i] = src[(long long)idx[j] * block16 + u];
}

// dst block dst_idx[j] <- src block src_idx[j] (scatter of per-window results into window-major slots)
__global__ void copy_blocks(uint4* __restrict__ dst, const int* __restrict__ dst_idx, const uint4* __restrict__ src,
                            const int* __restrict__ src_idx, long long n, long long block16) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n * block16) return;
  const long long j = i / block16, u = i - j * block16;
  dst[(long long)dst_idx[j] * block16 + u] = src[(long long)src_idx[j] * block16 + u];
}

}  // namespace

int pp_k_nchw_to_act(const float* src, __half* dst, int N, int C, int H, int W, int cs, cudaStream_t st, int dst_co,
                     int zero_fill_to) {
  const long long npix = (long long)N * H * W;
  if (npix == 0) return PP_OK;
  nchw_f32_to_nhwc_f16<<<nblocks(npix), TPB, 0, st>>>(src, dst, C, (long long)H * W, npix, cs, dst_co,
                                                       zero_fill_to < 0 ? cs - dst_co : zero_fill_to);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_upsample2x(const __half* src, int src_cs, int src_co, __half* dst, int dst_cs, int dst_co, int N, int H,
                    int W, int C, cudaStream_t st) {
  PP_REQUIRE(C % 8 == 0 && src_cs % 8 == 0 && dst_cs % 8 == 0 && src_co % 8 == 0 && dst_co % 8 == 0,
             "upsample2x: channels must be multiples of 8");
  if ((long long)N * H * W == 0) return PP_OK;
  PP_REQUIRE(H <= 65535 && N <= 65535, "upsample2x: %d rows / %d images exceed the grid limits", H, N);
  const dim3 grid(pp_ceil_div(W * (C / 8), 256), H, N);
  upsample2x_ac<<<grid, 256, 0, st>>>(src, src_cs, src_co, dst, dst_cs, dst_co, H, W, C / 8);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_upsample2x(const float* src, float* dst, int N, int H, int W, int C, cudaStream_t st) {
  PP_REQUIRE(C % 4 == 0 && H >= 1 && W >= 1, "upsample2x (split): C=%d must be a multiple of 4", C);
  if ((long long)N * H * W == 0) return PP_OK;
  PP_REQUIRE(2 * H <= 65535 && N <= 65535, "upsample2x: %d rows / %d images exceed the grid limits", 2 * H, N);
  const dim3 grid(pp_ceil_div(2 * W * (C / 4), 256), 2 * H, N);
  upsample2x_split<<<grid, 256, 0, st>>>(src, dst, H, W, C);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_gather_blocks(void* dst, const void* src, const int* idx_dev, long long n, long long block_bytes,
                       cudaStream_t st) {
  PP_REQUIRE(block_bytes % 16 == 0, "gather_blocks: block size must be a multiple of 16 bytes");
  if (n == 0) return PP_OK;
  const long long b16 = block_bytes / 16;
  gather_blocks<<<nblocks(n * b16), TPB, 0, st>>>(static_cast<uint4*>(dst), static_cast<const uint4*>(src), idx_dev, n,
                                                   b16);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_copy_blocks(void* dst, const int* dst_idx_dev, const void* src, const int* src_idx_dev, long long n,
                     long long block_bytes, cudaStream_t st) {
  PP_REQUIRE(block_bytes % 16 == 0, "copy_blocks: block size must be a multiple of 16 bytes");
  if (n == 0) return PP_OK;
  const long long b16 = block_bytes / 16;
  copy_blocks<<<nblocks(n * b16), TPB, 0, st>>>(static_cast<uint4*>(dst), dst_idx_dev, static_cast<const uint4*>(src),
                                                 src_idx_dev, n, b16);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

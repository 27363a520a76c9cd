// RAFT-specific HBM-bound kernels: instance norm, correlation pyramid pooling + 9x9x4 lookup,
// GRU state plumbing, convex upsampling.  Reference call sites are cited per kernel.
// The *_f32 forms serve the fp32 RAFT path: activations are split-tf32 pair tensors [pix][hi C | lo C] (conv_igemm.cuh)
// read as hi + lo, the correlation pyramid is plain fp32.
#include "kernels.cuh"

namespace {

constexpr int TPB = 256;

inline int nblocks(long long n, int per = TPB) { return (int)((n + per - 1) / per); }

// ------------------------------------------------------------------------------------------------
// InstanceNorm2d(affine=False) statistics: per (image, channel) sum and sum of squares.
// grid (chunks, N); block = 256 threads; thread t owns channel pair (t % (C/2)) and strides pixels.
// (reference: RAFT/extractor.py fnet norm layers, F.instance_norm eps=1e-5, biased variance)
// ------------------------------------------------------------------------------------------------
// Deterministic: no floating-point atomics.  A block reduces its pixel lanes in lane order, writes its partial sums to
// `partial[n][block][2C]`, and the block that arrives last (integer counter) adds the partials in block order -- the
// result does not depend on scheduling, so RAFT (and everything after it) is bit-reproducible run to run and between
// the single-GPU and the sharded multi-GPU execution.
// F32: x is a split pair tensor (float, [pix][hi C | lo C]), else fp16 [pix][C].
// The fp16 form takes the variance as E[x^2] - mean^2, which cancels for channels whose mean is large against their
// spread but stays below the fp16 storage rounding up to mean / std ~ 30.  The F32 form runs twice: the first launch
// leaves the sums of x, the second (`centred`) sums d = x - m1 and d^2 about that first mean m1 and leaves
// [mean | variance] = [m1 + E[d] | E[d^2] - E[d]^2] (the corrected two-pass algorithm: no cancellation, and the
// mean is not limited by the rounding of a sum of HW values).
template <bool F32>
__global__ void instnorm_stats(const void* __restrict__ xv, int HW, int C, float* __restrict__ sums,
                               float* __restrict__ partial, unsigned int* __restrict__ counters, int pix_per_block,
                               int centred) {
  extern __shared__ float sm[];  // [lanes][2C]
  __shared__ bool last;
  const int n = blockIdx.y;
  const int C2 = C >> 1;
  const int lanes = blockDim.x / C2;  // pixel lanes per block
  const int cp = threadIdx.x % C2;
  const int pl = threadIdx.x / C2;
  const int p0 = blockIdx.x * pix_per_block;
  const int p1 = min(HW, p0 + pix_per_block);
  if (pl < lanes) {
    float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
    float m0 = 0.f, m1 = 0.f;
    if (F32 && centred) {
      const float inv = 1.f / (float)HW;
      m0 = sums[(long long)n * 2 * C + 2 * cp] * inv;
      m1 = sums[(long long)n * 2 * C + 2 * cp + 1] * inv;
    }
    const __half2* base = reinterpret_cast<const __half2*>(reinterpret_cast<const __half*>(xv) + ((long long)n * HW) * C) + cp;
    const float* fbase = reinterpret_cast<const float*>(xv) + ((long long)n * HW) * 2 * C + 2 * cp;
    for (int p = p0 + pl; p < p1; p += lanes) {
      float2 v;
      if constexpr (F32) {
        const float2 h = *reinterpret_cast<const float2*>(fbase + (long long)p * 2 * C);
        const float2 l = *reinterpret_cast<const float2*>(fbase + (long long)p * 2 * C + C);
        v = make_float2(h.x + l.x - m0, h.y + l.y - m1);
      } else {
        v = __half22float2(base[(long long)p * C2]);
      }
      s0 += v.x; s1 += v.y;
      if (!F32 || centred) { q0 += v.x * v.x; q1 += v.y * v.y; }   // F32: the first pass needs the sums of x only
    }
    float* row = sm + pl * 2 * C;
    row[2 * cp] = s0; row[2 * cp + 1] = s1; row[C + 2 * cp] = q0; row[C + 2 * cp + 1] = q1;
  }
  __syncthreads();
  float* mine = partial + ((long long)n * gridDim.x + blockIdx.x) * 2 * C;
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
    float acc = 0.f;
    for (int l = 0; l < lanes; ++l) acc += sm[l * 2 * C + i];
    mine[i] = acc;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&counters[n], 1u) == gridDim.x - 1;
  __syncthreads();
  if (last) {
    __threadfence();
    const float* all = partial + (long long)n * gridDim.x * 2 * C;
    float* out = sums + (long long)n * 2 * C;
    if (F32 && centred) {   // every block has read m1 before it arrived: out can be overwritten
      const float inv = 1.f / (float)HW;
      for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float ds = 0.f, dq = 0.f;
        for (unsigned b = 0; b < gridDim.x; ++b) {
          ds += __ldcg(all + (long long)b * 2 * C + c);
          dq += __ldcg(all + (long long)b * 2 * C + C + c);
        }
        const float dm = ds * inv;
        out[c] = out[c] * inv + dm;
        out[C + c] = fmaxf(dq * inv - dm * dm, 0.f);
      }
    } else {
      for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
        float acc = 0.f;
        for (unsigned b = 0; b < gridDim.x; ++b) acc += __ldcg(all + (long long)b * 2 * C + i);
        out[i] = acc;
      }
    }
  }
}

// out = [relu]( (x - mean) * rstd );  if residual: out = relu(residual + out)   (ResidualBlock tail)
// F32: x, residual and out are split pair tensors (float, [pix][hi C | lo C]), else fp16 [pix][C].
__device__ __forceinline__ float2 ld_split2(const float* p, int C) {
  const float2 h = *reinterpret_cast<const float2*>(p), l = *reinterpret_cast<const float2*>(p + C);
  return make_float2(h.x + l.x, h.y + l.y);
}
__device__ __forceinline__ void st_split2(float* p, int C, float a, float b) {
  const float ha = ppx::tf32_rna(a), hb = ppx::tf32_rna(b);
  *reinterpret_cast<float2*>(p) = make_float2(ha, hb);
  *reinterpret_cast<float2*>(p + C) = make_float2(a - ha, b - hb);
}
__device__ __forceinline__ void st_split1(float* p, int C, float a) {
  const float h = ppx::tf32_rna(a);
  p[0] = h;
  p[C] = a - h;
}

template <bool F32>
__global__ void __launch_bounds__(256) instnorm_apply(const void* __restrict__ xv, const float* __restrict__ sums,
                                                      const void* __restrict__ residual, void* __restrict__ out, int HW,
                                                      int C, int relu) {
  // grid = (chunks of one image's HW*C/2 channel pairs, images): 32-bit index math, statistics row uniform per block
  const int C2 = C >> 1;
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (unsigned)(HW * C2)) return;
  const int n = blockIdx.y;
  const int cp = i % (unsigned)C2;
  const long long idx = (long long)n * HW * C2 + i;
  const float inv = 1.f / (float)HW;
  const float* s = sums + (long long)n * 2 * C;
  // F32: s holds [mean | variance] (instnorm_stats, centred), else [sum x | sum x^2]
  const float m0 = F32 ? s[2 * cp] : s[2 * cp] * inv, m1 = F32 ? s[2 * cp + 1] : s[2 * cp + 1] * inv;
  const float v0 = F32 ? s[C + 2 * cp] : fmaxf(s[C + 2 * cp] * inv - m0 * m0, 0.f);
  const float v1 = F32 ? s[C + 2 * cp + 1] : fmaxf(s[C + 2 * cp + 1] * inv - m1 * m1, 0.f);
  const float r0 = F32 ? __frsqrt_rn(v0 + 1e-5f) : rsqrtf(v0 + 1e-5f);
  const float r1 = F32 ? __frsqrt_rn(v1 + 1e-5f) : rsqrtf(v1 + 1e-5f);
  // split tensors: pixel idx / C2, channel pair cp
  const long long fo = (long long)n * HW * 2 * C + (long long)(i / (unsigned)C2) * 2 * C + 2 * cp;
  const float2 x2 = F32 ? ld_split2(reinterpret_cast<const float*>(xv) + fo, C)
                        : __half22float2(reinterpret_cast<const __half2*>(xv)[idx]);
  float a = (x2.x - m0) * r0, b = (x2.y - m1) * r1;
  if (relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
  if (residual != nullptr) {
    const float2 rv = F32 ? ld_split2(reinterpret_cast<const float*>(residual) + fo, C)
                          : __half22float2(reinterpret_cast<const __half2*>(residual)[idx]);
    a = fmaxf(a + rv.x, 0.f);
    b = fmaxf(b + rv.y, 0.f);
  }
  if constexpr (F32) st_split2(reinterpret_cast<float*>(out) + fo, C, a, b);
  else reinterpret_cast<__half2*>(out)[idx] = __floats2half2_rn(a, b);
}

// ------------------------------------------------------------------------------------------------
// Pack a row-major [G][R][K] fp16 matrix into the swizzled B-operand tile image consumed by the
// wgmma GEMM ([G][K/64][R_pad] rows of 128 B, 16-byte chunk index XOR (row & 7)); rows >= R are zero.
// Used for the all-pairs correlation, where fmap2 plays the role of the weights (RAFT/corr.py:52-60).
// ------------------------------------------------------------------------------------------------
__global__ void pack_b_operand(const __half* __restrict__ src, __half* __restrict__ dst, int R, int R_pad, int K,
                               long long total) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;  // one 16-byte chunk each
  if (idx >= total) return;
  const int chunks_per_row = K / 8;
  const int ch = idx % chunks_per_row;
  long long t = idx / chunks_per_row;
  const int r = t % R_pad;
  const int g = t / R_pad;
  uint4 v = make_uint4(0, 0, 0, 0);
  if (r < R) v = *reinterpret_cast<const uint4*>(src + ((long long)g * R + r) * K + ch * 8);
  const int kc = ch >> 3, c = ch & 7;
  const int num_kc = K / 64;
  __half* d = dst + (((long long)g * num_kc + kc) * R_pad + r) * 64 + ((c ^ (r & 7)) << 3);
  *reinterpret_cast<uint4*>(d) = v;
}

// 2x2 average pooling of every [h][w] correlation map (F.avg_pool2d(corr, 2, stride=2), corr.py:25-27).
// One block per query map (32-bit index math); each thread produces output pairs from two 8-byte row reads.
// T = __half (fp16 pyramid) or float (fp32 pyramid)
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ void from_f(float v, __half* d) { *d = __float2half_rn(v); }
__device__ __forceinline__ void from_f(float v, float* d) { *d = v; }

template <class T>
__global__ void __launch_bounds__(128) corr_pool(const T* __restrict__ src, T* __restrict__ dst, int h, int w) {
  const int oh = h >> 1, ow = w >> 1;
  const long long q = blockIdx.x;
  const T* s = src + q * (long long)(h * w);
  T* d = dst + q * (long long)(oh * ow);
  for (int i = threadIdx.x; i < oh * ow; i += blockDim.x) {
    const int oy = i / ow, ox = i - oy * ow;
    const T* r = s + 2 * oy * w + 2 * ox;
    const float a = to_f(r[0]) + to_f(r[1]) + to_f(r[w]) + to_f(r[w + 1]);
    from_f(0.25f * a, d + i);
  }
}

// ------------------------------------------------------------------------------------------------
// Correlation lookup (CorrBlock.__call__, corr.py:29-50; bilinear_sampler, RAFT/utils/utils.py:66-80).
// Output channel c = l*81 + i*9 + j samples level l at (x/2^l + (i-4), y/2^l + (j-4)), bilinear,
// zeros outside, align_corners=True.
// ------------------------------------------------------------------------------------------------
template <class T>
struct CorrLevels {
  const T* p[4];
};
__device__ __forceinline__ float2 ld_pair(const __half* m) { return __half22float2(*reinterpret_cast<const __half2*>(m)); }
__device__ __forceinline__ float2 ld_pair(const float* m) { return *reinterpret_cast<const float2*>(m); }

// One warp per query pixel.  For a given (pixel, level) all 81 outputs share the same bilinear fractions
// (the window offsets are integers), so the warp stages the tap window of each level in shared memory once
// (zero outside the map) and every lane then blends 4 staged taps per output:
//   out[l*81 + i*9 + j] = bilerp(T_l[j..j+1][i..i+1])      (i moves x, j moves y -- the meshgrid quirk)
// Taps are fetched as aligned fp16 pairs (12 columns starting at the even column <= x0-4; map widths are even at
// every level for the sizes ProPainter produces, odd widths take the scalar path), which halves the load
// instructions; the output loop runs level by level with the level's fractions in registers.
// Global traffic per pixel = the algorithmic 8 B coords + 4x100 taps + 324 outputs; stores are contiguous.
// E = __half: fp16 pyramid, fp16 output [nq][out_cs].  E = float: fp32 pyramid, split output [nq][hi out_cs | lo out_cs].
constexpr int LOOKUP_WARPS = 8;
constexpr int TAP_COLS = 12;   // staged columns per tap row
constexpr int TAP_STRIDE = 10 * TAP_COLS;

template <class E>
__global__ void __launch_bounds__(LOOKUP_WARPS * 32) corr_lookup(CorrLevels<E> lv, const float* __restrict__ coords,
                                                                 E* __restrict__ out, int out_cs, long long nq,
                                                                 int h8, int w8) {
  constexpr bool F32 = sizeof(E) == 4;
  __shared__ float taps[LOOKUP_WARPS][4][TAP_STRIDE];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long q = (long long)blockIdx.x * LOOKUP_WARPS + warp;
  if (q >= nq) return;
  const float cx = coords[q * 2], cy = coords[q * 2 + 1];
  float fa[4], fb[4];   // bilinear fractions and even-column phase of every level: registers of every lane
  int ph[4];
#pragma unroll
  for (int l = 0; l < 4; ++l) {
    const float inv = 1.f / (float)(1 << l);
    const int h = h8 >> l, w = w8 >> l;
    const float x = cx * inv, y = cy * inv;
    const float fx = floorf(x), fy = floorf(y);
    const int x0 = (int)fx - 4, y0 = (int)fy - 4;
    const int xa = x0 & ~1;                       // even column <= x0 (also for negative x0)
    fa[l] = x - fx; fb[l] = y - fy; ph[l] = x0 - xa;
    const E* m = lv.p[l] + q * (long long)(h * w);
    float* T = taps[warp][l];
    if ((w & 1) == 0) {
#pragma unroll
      for (int t2 = lane; t2 < 60; t2 += 32) {    // 10 rows x 6 aligned pairs
        const int ty = t2 / 6, tp = t2 - ty * 6;
        const int yy = y0 + ty, xx = xa + 2 * tp;
        float2 v = make_float2(0.f, 0.f);
        if ((unsigned)yy < (unsigned)h && (unsigned)xx < (unsigned)w)
          v = ld_pair(m + yy * w + xx);
        T[ty * TAP_COLS + 2 * tp] = v.x;
        T[ty * TAP_COLS + 2 * tp + 1] = v.y;
      }
    } else {
      for (int t = lane; t < TAP_STRIDE; t += 32) {
        const int ty = t / TAP_COLS, tx = t - ty * TAP_COLS;
        const int yy = y0 + ty, xx = xa + tx;
        float v = 0.f;
        if ((unsigned)yy < (unsigned)h && (unsigned)xx < (unsigned)w) v = to_f(m[yy * w + xx]);
        T[t] = v;
      }
    }
  }
  __syncwarp();
  E* o = out + q * out_cs * (F32 ? 2 : 1);
#pragma unroll
  for (int l = 0; l < 4; ++l) {
    const float a = fa[l], b = fb[l];
    const float* T = taps[warp][l] + ph[l];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int r = lane + 32 * k;                 // output i*9 + j of this level
      if (r < 81) {
        const int i = (r * 57) >> 9, j = r - 9 * i;  // r / 9, r % 9 for r < 81
        const float* t = T + j * TAP_COLS + i;
        const float top = t[0] + a * (t[1] - t[0]);
        const float bot = t[TAP_COLS] + a * (t[TAP_COLS + 1] - t[TAP_COLS]);
        const float v = top + b * (bot - top);
        if constexpr (F32) {
          const float hi = ppx::tf32_rna(v);
          o[l * 81 + r] = hi;
          o[out_cs + l * 81 + r] = v - hi;
        } else {
          o[l * 81 + r] = __float2half_rn(v);
        }
      }
    }
  }
  for (int c = 324 + lane; c < out_cs * (F32 ? 2 : 1); c += 32)   // padding channels (hi and lo)
    if (c < out_cs || c >= out_cs + 324) from_f(0.f, o + c);
}

// cnet output -> GRU state: h = tanh(c[:, :128]) into hx[:, 0:128], inp = relu(c[:, 128:]) into hx[:, 128:256]
// (raft.py:119-122)
__global__ void cnet_split(const __half* __restrict__ c, __half* __restrict__ hx, int hx_cs, long long total) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int ch = idx % 256;
  const long long p = idx / 256;
  const float v = __half2float(c[idx]);
  hx[p * hx_cs + ch] = __float2half_rn(ch < 128 ? tanhf(v) : fmaxf(v, 0.f));
}

// coords1 = coords0 (+ delta); flow = coords1 - coords0 written (fp16) to the motion-encoder input
// ([.,8], channels 2..7 zero) and to the last two channels of the GRU input (raft.py:124-140).
__global__ void raft_coords(const float* __restrict__ delta, float* __restrict__ coords1, __half* __restrict__ flow8,
                            __half* __restrict__ hx, int hx_cs, int hx_flow_co, long long total, int P, int w8,
                            int init) {
  long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (q >= total) return;
  const int p = q % P;
  const float x0 = (float)(p % w8), y0 = (float)(p / w8);
  float x, y;
  if (init) { x = x0; y = y0; }
  else { x = coords1[2 * q] + delta[2 * q]; y = coords1[2 * q + 1] + delta[2 * q + 1]; }
  coords1[2 * q] = x;
  coords1[2 * q + 1] = y;
  const __half fx = __float2half_rn(x - x0), fy = __float2half_rn(y - y0);
  __half* f = flow8 + q * 8;
  f[0] = fx; f[1] = fy;
  if (init) for (int k = 2; k < 8; ++k) f[k] = __float2half_rn(0.f);
  hx[q * hx_cs + hx_flow_co] = fx;
  hx[q * hx_cs + hx_flow_co + 1] = fy;
}

// Convex 8x upsampling (RAFT.upsample_flow, raft.py:81-92): softmax over the 9 neighbours' logits
// mask[k*64 + sy*8 + sx], weighted sum of 8*flow (3x3 unfold, zero padding).  Output NCHW fp32.
// T = __half: fp16 mask [q][576]; T = float: split mask [q][hi 576 | lo 576], with fp32-accurate exp and division
template <class T>
__global__ void convex_upsample(const float* __restrict__ coords1, const T* __restrict__ mask,
                                float* __restrict__ out, int B, int h8, int w8) {
  constexpr bool F32 = sizeof(T) == 4;
  const int H = 8 * h8, W = 8 * w8;
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)B * H * W) return;
  const int X = idx % W;
  long long t = idx / W;
  const int Y = t % H;
  const int b = t / H;
  const int x = X >> 3, sx = X & 7, y = Y >> 3, sy = Y & 7;
  const long long q = ((long long)b * h8 + y) * w8 + x;
  const T* mk = mask + q * 576 * (F32 ? 2 : 1) + sy * 8 + sx;
  float lg[9], mx = -1e30f;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    lg[k] = F32 ? to_f(mk[k * 64]) + to_f(mk[576 + k * 64]) : to_f(mk[k * 64]);
    mx = fmaxf(mx, lg[k]);
  }
  float den = 0.f, ux = 0.f, uy = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const float e = F32 ? ppx::exp_acc(lg[k] - mx) : __expf(lg[k] - mx);
    den += e;
    const int ny = y + k / 3 - 1, nx = x + k % 3 - 1;
    if (ny >= 0 && ny < h8 && nx >= 0 && nx < w8) {
      const long long nq = ((long long)b * h8 + ny) * w8 + nx;
      ux += e * 8.f * (coords1[2 * nq] - (float)nx);
      uy += e * 8.f * (coords1[2 * nq + 1] - (float)ny);
    }
  }
  const long long HWl = (long long)H * W;
  out[((long long)b * 2) * HWl + (long long)Y * W + X] = F32 ? __fdiv_rn(ux, den) : ux / den;
  out[((long long)b * 2 + 1) * HWl + (long long)Y * W + X] = F32 ? __fdiv_rn(uy, den) : uy / den;
}

// ---- fp32 path only --------------------------------------------------------------------------------------------------
// frames [N][C][H][W] fp32 -> split pair tensor [N*H*W][hi cs | lo cs] (channels C..cs-1 zero)
__global__ void nchw_to_split(const float* __restrict__ src, float* __restrict__ dst, int C, int HW, int cs, long long total) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;   // (pixel, channel < cs)
  if (idx >= total) return;
  const int c = (int)(idx % cs);
  const long long pix = idx / cs;
  const long long n = pix / HW;
  const float v = c < C ? src[(n * C + c) * HW + (pix - n * HW)] : 0.f;
  st_split1(dst + pix * 2 * cs + c, cs, v);
}

// Pack a split pair tensor [G][R][hi K | lo K] into the split B-operand image of the correlation GEMM: per row the 3K
// values [hi; hi; lo] (against the A segments (hi, lo, hi)) in [G][3K/32][R_pad] rows of 32 floats, 16-byte unit index
// XOR (row & 7); rows >= R are zero.
__global__ void pack_b_operand_split(const float* __restrict__ src, float* __restrict__ dst, int R, int R_pad, int K,
                                     long long total) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;   // one 16-byte unit (4 floats) each
  if (idx >= total) return;
  const int units = 3 * K / 4;
  const int u = (int)(idx % units);
  const long long t = idx / units;
  const int r = (int)(t % R_pad);
  const long long g = t / R_pad;
  const int k0 = 4 * u, sec = k0 / K, c = k0 - sec * K;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (r < R) v = *reinterpret_cast<const float4*>(src + (g * R + r) * 2 * K + (sec == 2 ? K : 0) + c);
  const int kc = k0 >> 5, uc = (k0 & 31) >> 2;
  *reinterpret_cast<float4*>(dst + ((g * (3 * K / 32) + kc) * R_pad + r) * 32 + ((uc ^ (r & 7)) << 2)) = v;
}

// cnet_split on split tensors: c [p][hi 256 | lo 256] -> hx [p][hi hx_C | lo hx_C] channels 0..255
__global__ void cnet_split_f32(const float* __restrict__ c, float* __restrict__ hx, int hx_C, long long total) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int ch = idx % 256;
  const long long p = idx / 256;
  const float v = c[p * 512 + ch] + c[p * 512 + 256 + ch];
  st_split1(hx + p * 2 * hx_C + ch, hx_C, ch < 128 ? ppx::tanh_acc(v) : fmaxf(v, 0.f));
}

// raft_coords of the fp32 path: the flow goes (split) to channels hx_flow_co, +1 of the GRU state only; the motion
// encoder's 7x7 patches are taken from coords1 directly (flow_patch7x7_f32)
__global__ void raft_coords_f32(const float* __restrict__ delta, float* __restrict__ coords1, float* __restrict__ hx,
                                int hx_C, int hx_flow_co, long long total, int P, int w8, int init) {
  const long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (q >= total) return;
  const int p = q % P;
  const float x0 = (float)(p % w8), y0 = (float)(p / w8);
  float x, y;
  if (init) { x = x0; y = y0; }
  else { x = coords1[2 * q] + delta[2 * q]; y = coords1[2 * q + 1] + delta[2 * q + 1]; }
  coords1[2 * q] = x;
  coords1[2 * q + 1] = y;
  float* f = hx + q * 2 * hx_C + hx_flow_co;
  st_split1(f, hx_C, x - x0);
  st_split1(f + 1, hx_C, y - y0);
}

// flow_patch7x7 of the fp32 path: flow = coords1 - coords0 of the 49 neighbours, split output [M][hi 128 | lo 128].
// One thread per (pixel, patch value).
__global__ void flow_patch7x7_f32(const float* __restrict__ coords1, float* __restrict__ out, int h, int w, long long total) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int v = (int)(idx & 127), tap = v >> 1, ch = v & 1;
  const long long pix = idx >> 7;
  const int hw = h * w;
  const long long img = pix / hw;
  const int p = (int)(pix - img * hw), y = p / w, x = p - y * w;
  float f = 0.f;
  if (tap < 49) {
    const int yy = y + tap / 7 - 3, xx = x + tap % 7 - 3;
    if (yy >= 0 && yy < h && xx >= 0 && xx < w)
      f = coords1[(img * hw + (long long)yy * w + xx) * 2 + ch] - (float)(ch ? yy : xx);
  }
  st_split1(out + pix * 256 + v, 128, f);
}

}  // namespace

size_t pp_k_instnorm_scratch_floats(int N, int HW, int C) {
  return (size_t)N * 2 * C * (pp_ceil_div(HW, 1024) + 1) + (size_t)N + 64;
}

// sums: scratch of pp_k_instnorm_scratch_floats(N, HW, C) floats; the statistics [N][2][C] are its first N*2*C entries
template <class E>
int pp_k_instnorm_stats(const E* x, int N, int HW, int C, float* sums, cudaStream_t st) {
  constexpr bool F32 = sizeof(E) == 4;
  PP_REQUIRE(C % 2 == 0 && C <= 256, "instnorm: unsupported C=%d", C);
  const int pix_per_block = 1024;
  const int nblk = pp_ceil_div(HW, pix_per_block);
  float* partial = sums + (size_t)N * 2 * C;
  unsigned int* counters = reinterpret_cast<unsigned int*>(partial + (size_t)N * nblk * 2 * C);
  dim3 grid(nblk, N);
  const int lanes = 256 / (C / 2);
  for (int centred = 0; centred < (F32 ? 2 : 1); ++centred) {   // fp32: sums of x, then sums of (x - mean)^2
    PP_CUDA_CHECK(cudaMemsetAsync(counters, 0, (size_t)N * sizeof(unsigned int), st));
    instnorm_stats<F32><<<grid, 256, (size_t)lanes * 2 * C * sizeof(float), st>>>(x, HW, C, sums, partial, counters,
                                                                                  pix_per_block, centred);
    PP_CUDA_CHECK(cudaGetLastError());
  }
  return PP_OK;
}
template int pp_k_instnorm_stats(const __half*, int, int, int, float*, cudaStream_t);
template int pp_k_instnorm_stats(const float*, int, int, int, float*, cudaStream_t);

template <class E>
int pp_k_instnorm_apply(const E* x, const float* sums, const E* residual, E* out, int N, int HW, int C, int relu,
                        cudaStream_t st) {
  if ((long long)N * HW == 0) return PP_OK;
  PP_REQUIRE(N <= 65535 && (long long)HW * (C / 2) < (1LL << 31), "instnorm: %d images of %d pixels exceed the grid limits", N, HW);
  instnorm_apply<sizeof(E) == 4><<<dim3(pp_ceil_div(HW * (C / 2), 256), N), 256, 0, st>>>(x, sums, residual, out, HW, C,
                                                                                          relu);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}
template int pp_k_instnorm_apply(const __half*, const float*, const __half*, __half*, int, int, int, int, cudaStream_t);
template int pp_k_instnorm_apply(const float*, const float*, const float*, float*, int, int, int, int, cudaStream_t);

int pp_k_nchw_to_act(const float* src, float* dst, int N, int C, int H, int W, int cs, cudaStream_t st) {
  PP_REQUIRE(C <= cs && cs % 4 == 0, "nchw_to_split: C=%d cs=%d", C, cs);
  const long long total = (long long)N * H * W * cs;
  if (total == 0) return PP_OK;
  nchw_to_split<<<nblocks(total), TPB, 0, st>>>(src, dst, C, H * W, cs, total);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_pack_b_operand(const float* src, float* dst, int G, int R, int R_pad, int K, cudaStream_t st) {
  PP_REQUIRE(K % 32 == 0 && R_pad % 8 == 0, "pack_b_operand_split: K=%d must be a multiple of 32", K);
  const long long total = (long long)G * R_pad * (3 * K / 4);
  pack_b_operand_split<<<nblocks(total), TPB, 0, st>>>(src, dst, R, R_pad, K, total);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_pack_b_operand(const __half* src, __half* dst, int G, int R, int R_pad, int K, cudaStream_t st) {
  PP_REQUIRE(K % 64 == 0 && R_pad % 8 == 0, "pack_b_operand: K=%d must be a multiple of 64", K);
  const long long total = (long long)G * R_pad * (K / 8);
  pack_b_operand<<<nblocks(total), TPB, 0, st>>>(src, dst, R, R_pad, K, total);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

template <class E>
int pp_k_corr_pool(const E* src, E* dst, long long nq, int h, int w, cudaStream_t st) {
  if (nq * (h / 2) * (w / 2) == 0) return PP_OK;
  PP_REQUIRE(nq < (1LL << 31), "corr_pool: too many query maps");
  corr_pool<E><<<(unsigned)nq, 128, 0, st>>>(src, dst, h, w);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}
template int pp_k_corr_pool(const __half*, __half*, long long, int, int, cudaStream_t);
template int pp_k_corr_pool(const float*, float*, long long, int, int, cudaStream_t);

template <class E>
int pp_k_corr_lookup(const E* l0, const E* l1, const E* l2, const E* l3, const float* coords, E* out, int out_C,
                     long long nq, int h8, int w8, cudaStream_t st) {
  PP_REQUIRE(out_C >= 324 && out_C <= 352, "corr_lookup: out_C=%d not in [324,352]", out_C);
  CorrLevels<E> lv;
  lv.p[0] = l0; lv.p[1] = l1; lv.p[2] = l2; lv.p[3] = l3;
  corr_lookup<E><<<(unsigned)((nq + LOOKUP_WARPS - 1) / LOOKUP_WARPS), LOOKUP_WARPS * 32, 0, st>>>(lv, coords, out,
                                                                                                 out_C, nq, h8, w8);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}
template int pp_k_corr_lookup(const __half*, const __half*, const __half*, const __half*, const float*, __half*, int,
                              long long, int, int, cudaStream_t);
template int pp_k_corr_lookup(const float*, const float*, const float*, const float*, const float*, float*, int,
                              long long, int, int, cudaStream_t);

int pp_k_cnet_split(const __half* c, __half* hx, int hx_C, long long npix, cudaStream_t st) {
  cnet_split<<<nblocks(npix * 256), TPB, 0, st>>>(c, hx, hx_C, npix * 256);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_cnet_split(const float* c, float* hx, int hx_C, long long npix, cudaStream_t st) {
  cnet_split_f32<<<nblocks(npix * 256), TPB, 0, st>>>(c, hx, hx_C, npix * 256);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

// im2col of the 2-channel flow for BasicMotionEncoder.convf1 (7x7, pad 3; update.py:97,105): per pixel the 49 taps x (dx, dy)
// = 98 values in (ky, kx, channel) order, zero outside the map, zero-padded to 128 -> [M][128] fp16, so that the layer runs
// as a K = 128 flat GEMM on the TMA kernel instead of a K = 49 x 8 (6 of 8 channels padding) implicit GEMM.
// One thread per (pixel, 16-byte unit = 4 taps).
__global__ void flow_patch7x7(const __half* __restrict__ flow8, uint4* __restrict__ out, int h, int w, long long total_units) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= total_units) return;
  const int u = (int)(idx & 15);
  const long long pix = idx >> 4;
  const int hw = h * w;
  const long long img = pix / hw;
  const int p = (int)(pix - img * hw), y = p / w, x = p - y * w;
  __align__(16) __half2 v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int tap = u * 4 + i;
    v[i] = __floats2half2_rn(0.f, 0.f);
    if (tap < 49) {
      const int yy = y + tap / 7 - 3, xx = x + tap % 7 - 3;
      if (yy >= 0 && yy < h && xx >= 0 && xx < w)
        v[i] = *reinterpret_cast<const __half2*>(flow8 + ((img * hw + (long long)yy * w + xx) << 3));
    }
  }
  out[idx] = *reinterpret_cast<uint4*>(v);
}

int pp_k_flow_patch7x7(const __half* flow8, __half* out, int B, int h8, int w8, cudaStream_t st) {
  const long long total = (long long)B * h8 * w8 * 16;
  if (total == 0) return PP_OK;
  flow_patch7x7<<<nblocks(total), TPB, 0, st>>>(flow8, reinterpret_cast<uint4*>(out), h8, w8, total);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_flow_patch7x7(const float* coords1, float* out, int B, int h8, int w8, cudaStream_t st) {
  const long long total = (long long)B * h8 * w8 * 128;
  if (total == 0) return PP_OK;
  flow_patch7x7_f32<<<nblocks(total), TPB, 0, st>>>(coords1, out, h8, w8, total);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_raft_coords(const float* delta, float* coords1, float* hx, int hx_C, int hx_flow_co, int B, int h8, int w8,
                     cudaStream_t st) {
  const long long total = (long long)B * h8 * w8;
  raft_coords_f32<<<nblocks(total), TPB, 0, st>>>(delta, coords1, hx, hx_C, hx_flow_co, total, h8 * w8, w8,
                                                   delta == nullptr ? 1 : 0);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_raft_coords(const float* delta, float* coords1, __half* flow8, __half* hx, int hx_C, int hx_flow_co, int B,
                     int h8, int w8, cudaStream_t st) {
  const long long total = (long long)B * h8 * w8;
  raft_coords<<<nblocks(total), TPB, 0, st>>>(delta, coords1, flow8, hx, hx_C, hx_flow_co, total, h8 * w8, w8,
                                               delta == nullptr ? 1 : 0);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

template <class E>
int pp_k_convex_upsample(const float* coords1, const E* mask, float* out_nchw, int B, int h8, int w8, cudaStream_t st) {
  const long long total = (long long)B * 64 * h8 * w8;
  convex_upsample<E><<<nblocks(total), TPB, 0, st>>>(coords1, mask, out_nchw, B, h8, w8);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}
template int pp_k_convex_upsample(const float*, const __half*, float*, int, int, int, cudaStream_t);
template int pp_k_convex_upsample(const float*, const float*, float*, int, int, int, cudaStream_t);

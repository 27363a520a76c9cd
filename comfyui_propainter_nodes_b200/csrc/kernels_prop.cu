// Flow-guided propagation kernels: fused image-propagation step, flow warps, fb-consistency,
// modulated deformable sampling, flow-completion pack/combine, 1/4 downsampling.
#include <stdlib.h>

#include <type_traits>

#include "kernels.cuh"
#include "conv_igemm.cuh"
#include "dcn_sample.cuh"

namespace {

constexpr int TPB = 256;
inline int nblocks(long long n, int per = TPB) { return (int)((n + per - 1) / per); }

// Sampling position of grid_sample(align_corners=True) for pixel coordinate (x + flow): the reference
// normalises with 2*g/max(W-1,1)-1 (flow_loss_utils.py:41-43) and ATen's CUDA sampler un-normalises with
// ((g+1)/2)*(W-1).  The round trip is kept (no FMA contraction) so `nearest` picks the same texel.
__device__ __forceinline__ float sample_coord(float g, int size) {
  const float d = (float)max(size - 1, 1);
  const float nrm = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, g), d), 1.0f);
  return __fmul_rn(__fdiv_rn(__fadd_rn(nrm, 1.0f), 2.0f), (float)(size - 1));
}

struct Bilin {
  int x0, y0;
  float w00, w01, w10, w11;  // weights, already zero for out-of-range corners
};

// The weights are ATen's CPU form (w = x - floor(x), e = 1 - w; nw = s * e ...).  ATen's CUDA form ((ix_se - ix) *
// (iy_se - iy) ...) gives the same weight on every in-range corner: for floor(sx) >= 0, sx - floor(sx) is exact, so
// both round the same exact value once; they differ only for floor(sx) = -1, on the weight of column -1, which is out
// of range and zeroed here.
__device__ __forceinline__ Bilin bilin_setup(float sx, float sy, int W, int H) {
  Bilin b;
  const float fx = floorf(sx), fy = floorf(sy);
  b.x0 = (int)fx; b.y0 = (int)fy;
  const float ax = sx - fx, ay = sy - fy;
  const bool x0in = b.x0 >= 0 && b.x0 < W, x1in = b.x0 + 1 >= 0 && b.x0 + 1 < W;
  const bool y0in = b.y0 >= 0 && b.y0 < H, y1in = b.y0 + 1 >= 0 && b.y0 + 1 < H;
  b.w00 = (y0in && x0in) ? (1.f - ax) * (1.f - ay) : 0.f;
  b.w01 = (y0in && x1in) ? ax * (1.f - ay) : 0.f;
  b.w10 = (y1in && x0in) ? (1.f - ax) * ay : 0.f;
  b.w11 = (y1in && x1in) ? ax * ay : 0.f;
  return b;
}

// bilinear sample of a 2-channel fp16 flow field [H][W][2]
__device__ __forceinline__ float2 sample_flow2(const __half2* f, const Bilin& b, int W) {
  float2 r = make_float2(0.f, 0.f);
  if (b.w00 != 0.f) { const float2 v = __half22float2(f[b.y0 * W + b.x0]); r.x += b.w00 * v.x; r.y += b.w00 * v.y; }
  if (b.w01 != 0.f) { const float2 v = __half22float2(f[b.y0 * W + b.x0 + 1]); r.x += b.w01 * v.x; r.y += b.w01 * v.y; }
  if (b.w10 != 0.f) { const float2 v = __half22float2(f[(b.y0 + 1) * W + b.x0]); r.x += b.w10 * v.x; r.y += b.w10 * v.y; }
  if (b.w11 != 0.f) { const float2 v = __half22float2(f[(b.y0 + 1) * W + b.x0 + 1]); r.x += b.w11 * v.x; r.y += b.w11 * v.y; }
  return r;
}

// fbConsistencyCheck (model/propainter.py:27-36): |f_p + warp(f_c, f_p)|^2 < 0.01(|f_p|^2 + |warp|^2) + 0.5
__device__ __forceinline__ float fb_valid(float2 fp, float2 fcw) {
  const float dx = fp.x + fcw.x, dy = fp.y + fcw.y;
  const float mag = fp.x * fp.x + fp.y * fp.y + fcw.x * fcw.x + fcw.y * fcw.y;
  return (dx * dx + dy * dy) < (0.01f * mag + 0.5f) ? 1.f : 0.f;
}

// fp32 forms of sample_flow2 / fb_valid for the fp32 image propagation: every product and sum rounded on its own, in
// the order torch's CPU fp32 evaluation uses (grid_sample's nw + ne + sw + se; fbConsistencyCheck's per-tensor ops),
// so the discrete decisions downstream (fb test, 0.1 threshold) are the ones the reference takes on the CPU.  No FMA
// contraction.  (ATen's CUDA grid_sample is compiled with contraction, so it can round these sums differently.)
__device__ __forceinline__ float2 sample_flow2_rn(const float2* f, const Bilin& b, int W) {
  float2 r = make_float2(0.f, 0.f);
  auto acc = [&](float w, float2 v) { r.x = __fadd_rn(r.x, __fmul_rn(w, v.x)); r.y = __fadd_rn(r.y, __fmul_rn(w, v.y)); };
  if (b.w00 != 0.f) acc(b.w00, f[b.y0 * W + b.x0]);
  if (b.w01 != 0.f) acc(b.w01, f[b.y0 * W + b.x0 + 1]);
  if (b.w10 != 0.f) acc(b.w10, f[(b.y0 + 1) * W + b.x0]);
  if (b.w11 != 0.f) acc(b.w11, f[(b.y0 + 1) * W + b.x0 + 1]);
  return r;
}

__device__ __forceinline__ float fb_valid_rn(float2 fp, float2 fcw) {
  const float dx = __fadd_rn(fp.x, fcw.x), dy = __fadd_rn(fp.y, fcw.y);
  const float mag = __fadd_rn(__fadd_rn(__fmul_rn(fp.x, fp.x), __fmul_rn(fp.y, fp.y)),
                              __fadd_rn(__fmul_rn(fcw.x, fcw.x), __fmul_rn(fcw.y, fcw.y)));
  return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) < __fadd_rn(__fmul_rn(0.01f, mag), 0.5f) ? 1.f : 0.f;
}

// Storage of the image-propagation kernels.  A pixel is (r, g, b, mask) in one vector access: 4 x fp16 (uint2) on the
// fp16 path, float4 on the fp32 path (the node's fp16="disable"); flows are __half2 / float2.  The fp32 form also runs
// the bilinear sums and the fb test through the *_rn forms above.
struct ImgF16 {
  using Pix = uint2;
  using Flow = __half2;
  static constexpr bool exact = false;
  __device__ static float2 flow(Flow f) { return __half22float2(f); }
  __device__ static float2 rg(const Pix& t) { return __half22float2(*reinterpret_cast<const __half2*>(&t.x)); }
  __device__ static float2 bm(const Pix& t) { return __half22float2(*reinterpret_cast<const __half2*>(&t.y)); }
  __device__ static float mask_of(const Pix& t) { return __half2float(reinterpret_cast<const __half*>(&t)[3]); }
  __device__ static float mask_at(const Pix* p, int i) { return __half2float(reinterpret_cast<const __half*>(&p[i])[3]); }
  __device__ static Pix make(float r, float g, float b, float m) {
    uint2 o;
    *reinterpret_cast<__half2*>(&o.x) = __floats2half2_rn(r, g);
    *reinterpret_cast<__half2*>(&o.y) = __floats2half2_rn(b, m);
    return o;
  }
  __device__ static Flow make_flow(float x, float y) { return __floats2half2_rn(x, y); }
};

struct ImgF32 {
  using Pix = float4;
  using Flow = float2;
  static constexpr bool exact = true;
  __device__ static float2 flow(Flow f) { return f; }
  __device__ static float2 rg(const Pix& t) { return make_float2(t.x, t.y); }
  __device__ static float2 bm(const Pix& t) { return make_float2(t.z, t.w); }
  __device__ static float mask_of(const Pix& t) { return t.w; }
  __device__ static float mask_at(const Pix* p, int i) { return reinterpret_cast<const float*>(&p[i])[3]; }
  __device__ static Pix make(float r, float g, float b, float m) { return make_float4(r, g, b, m); }
  __device__ static Flow make_flow(float x, float y) { return make_float2(x, y); }
};

// storage type of a launcher's element type (__half / float)
template <class E>
using ImgOf = std::conditional_t<sizeof(E) == 4, ImgF32, ImgF16>;

template <class S>
__device__ __forceinline__ float fb_valid_of(float2 fp, const typename S::Flow* fchk, const Bilin& b, int W) {
  if constexpr (S::exact) return fb_valid_rn(fp, sample_flow2_rn(fchk, b, W));
  else return fb_valid(fp, sample_flow2(fchk, b, W));
}

// bilinear mask sum: w * m over the non-zero corners in grid_sample's order (nw, ne, sw, se)
template <class S>
__device__ __forceinline__ void mask_acc(float& mw, float w, float m) {
  if constexpr (S::exact) mw = __fadd_rn(mw, __fmul_rn(w, m));
  else mw += w * m;
}

// ------------------------------------------------------------------------------------------------
// One time step of the non-learnable image propagation (BidirectionalPropagation(3, learnable=False),
// model/propainter.py:157-196), fully fused: fb check, nearest warp of the propagated pixels, bilinear
// warp + 0.1 threshold of the propagated mask, mask algebra, blend.
// Pixel layout: 4 x fp16 = (r, g, b, mask) so one 8-byte access moves a whole pixel.
// Algorithmic traffic: cur 8 B + prop gather 8 B (+ 3 more mask taps) + out 8 B + 2 flows 4 B each.
// ------------------------------------------------------------------------------------------------
template <class S>
__global__ void imgprop_step(const typename S::Pix* __restrict__ cur, const typename S::Pix* __restrict__ prop_in,
                             typename S::Pix* __restrict__ prop_out, const typename S::Flow* __restrict__ flow_prop,
                             const typename S::Flow* __restrict__ flow_check, int H, int W) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= H * W) return;
  const int x = idx % W, y = idx / W;
  const float2 fp = S::flow(flow_prop[idx]);
  const float sx = sample_coord((float)x + fp.x, W), sy = sample_coord((float)y + fp.y, H);
  const Bilin b = bilin_setup(sx, sy, W, H);
  const float valid = fb_valid_of<S>(fp, flow_check, b, W);
  // nearest texel of the propagated frame
  const int nx = (int)nearbyintf(sx), ny = (int)nearbyintf(sy);
  float wr = 0.f, wg = 0.f, wb = 0.f;
  if (nx >= 0 && nx < W && ny >= 0 && ny < H) {
    const typename S::Pix t = prop_in[ny * W + nx];
    const float2 a = S::rg(t);
    const float2 c = S::bm(t);
    wr = a.x; wg = a.y; wb = c.x;
  }
  // bilinear sample of the propagated mask (4th channel)
  float mw = 0.f;
  if (b.w00 != 0.f) mask_acc<S>(mw, b.w00, S::mask_at(prop_in, b.y0 * W + b.x0));
  if (b.w01 != 0.f) mask_acc<S>(mw, b.w01, S::mask_at(prop_in, b.y0 * W + b.x0 + 1));
  if (b.w10 != 0.f) mask_acc<S>(mw, b.w10, S::mask_at(prop_in, (b.y0 + 1) * W + b.x0));
  if (b.w11 != 0.f) mask_acc<S>(mw, b.w11, S::mask_at(prop_in, (b.y0 + 1) * W + b.x0 + 1));
  const float mv = mw > 0.1f ? 1.f : 0.f;
  const typename S::Pix cu = cur[idx];
  const float2 c01 = S::rg(cu);
  const float2 c23 = S::bm(cu);
  const float mcur = c23.y;
  const float u = (mcur * valid * (1.f - mv)) > 0.1f ? 1.f : 0.f;
  const float mnew = (mcur * (1.f - valid * (1.f - mv))) > 0.1f ? 1.f : 0.f;
  const float r = u * wr + (1.f - u) * c01.x, g = u * wg + (1.f - u) * c01.y, bb = u * wb + (1.f - u) * c23.x;
  prop_out[idx] = S::make(r, g, bb, mnew);
}

// ------------------------------------------------------------------------------------------------
// The whole bidirectional propagation (2(T-1) serial steps) as ONE persistent kernel.
//
// A step only changes pixels whose current mask is set: for m_cur = 0 the blend weight u and the new mask are 0 and
// the output is the current pixel (model/propainter.py:186-196).  So the kernel works on the bounding box of the
// hole (union over the clip, computed on the device), with `bwd` and `fwd` pre-initialised to the packed input, and
// a grid-wide barrier between steps replaces 158 kernel launches.  Everything that does not depend on the
// previous step (current pixel, both flows, the fb-consistency test, the sampling positions) is fetched for step
// s+1 before the barrier of step s, so the serial chain per step is one barrier + one gather from L2.
// ------------------------------------------------------------------------------------------------
template <class S>
struct PropPre {        // the step-independent half of one pixel's work
  int pix;              // pixel index in the frame, -1: nothing to do
  int near;             // nearest texel index of the propagated frame or -1
  int x0, y0;
  float w00, w01, w10, w11;
  float valid;
  typename S::Pix cur;
};

template <class S>
__device__ __forceinline__ PropPre<S> prop_pre(const typename S::Pix* __restrict__ cur,
                                               const typename S::Flow* __restrict__ flow_prop,
                                               const typename S::Flow* __restrict__ flow_check, int pix, int H, int W,
                                               bool cur_is_input) {
  PropPre<S> r;
  r.pix = pix;
  r.near = -1;
  r.cur = cur_is_input ? __ldg(&cur[pix]) : __ldcg(&cur[pix]);
  const float mcur = S::mask_of(r.cur);
  r.valid = 0.f; r.x0 = r.y0 = 0; r.w00 = r.w01 = r.w10 = r.w11 = 0.f;
  if (mcur == 0.f) { r.near = -2; return r; }          // -2: pass-through pixel
  const int x = pix % W, y = pix / W;
  const float2 fp = S::flow(__ldg(&flow_prop[pix]));
  const float sx = sample_coord((float)x + fp.x, W), sy = sample_coord((float)y + fp.y, H);
  const Bilin b = bilin_setup(sx, sy, W, H);
  r.valid = fb_valid_of<S>(fp, flow_check, b, W);
  const int nx = (int)nearbyintf(sx), ny = (int)nearbyintf(sy);
  if (nx >= 0 && nx < W && ny >= 0 && ny < H) r.near = ny * W + nx;
  r.x0 = b.x0; r.y0 = b.y0; r.w00 = b.w00; r.w01 = b.w01; r.w10 = b.w10; r.w11 = b.w11;
  return r;
}

template <class S>
__device__ __forceinline__ typename S::Pix prop_post(const PropPre<S>& r, const typename S::Pix* prop_in, int W) {
  float wr = 0.f, wg = 0.f, wb = 0.f;
  if (r.near >= 0) {
    const typename S::Pix t = __ldcg(&prop_in[r.near]);
    const float2 a = S::rg(t);
    const float2 c = S::bm(t);
    wr = a.x; wg = a.y; wb = c.x;
  }
  float mw = 0.f;
  auto mk = [&](int i) { return S::mask_of(__ldcg(&prop_in[i])); };
  if (r.w00 != 0.f) mask_acc<S>(mw, r.w00, mk(r.y0 * W + r.x0));
  if (r.w01 != 0.f) mask_acc<S>(mw, r.w01, mk(r.y0 * W + r.x0 + 1));
  if (r.w10 != 0.f) mask_acc<S>(mw, r.w10, mk((r.y0 + 1) * W + r.x0));
  if (r.w11 != 0.f) mask_acc<S>(mw, r.w11, mk((r.y0 + 1) * W + r.x0 + 1));
  const float mv = mw > 0.1f ? 1.f : 0.f;
  const float2 c01 = S::rg(r.cur);
  const float2 c23 = S::bm(r.cur);
  const float mcur = c23.y;
  const float u = (mcur * r.valid * (1.f - mv)) > 0.1f ? 1.f : 0.f;
  const float mnew = (mcur * (1.f - r.valid * (1.f - mv))) > 0.1f ? 1.f : 0.f;
  return S::make(u * wr + (1.f - u) * c01.x, u * wg + (1.f - u) * c01.y, u * wb + (1.f - u) * c23.x, mnew);
}

// bbox = {x0, y0, x1, y1} (inclusive) of mask > 0 over all frames; initialised to {W, H, -1, -1}
__global__ void mask_bbox(const float* __restrict__ masks, long long total, int HW, int W, int* __restrict__ bbox) {
  int x0 = 1 << 30, y0 = 1 << 30, x1 = -1, y1 = -1;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    if (masks[i] != 0.f) {
      const int p = (int)(i % HW), x = p % W, y = p / W;
      x0 = min(x0, x); y0 = min(y0, y); x1 = max(x1, x); y1 = max(y1, y);
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    x0 = min(x0, __shfl_xor_sync(0xffffffffu, x0, o)); y0 = min(y0, __shfl_xor_sync(0xffffffffu, y0, o));
    x1 = max(x1, __shfl_xor_sync(0xffffffffu, x1, o)); y1 = max(y1, __shfl_xor_sync(0xffffffffu, y1, o));
  }
  if ((threadIdx.x & 31) == 0 && x1 >= 0) {
    atomicMin(&bbox[0], x0); atomicMin(&bbox[1], y0); atomicMax(&bbox[2], x1); atomicMax(&bbox[3], y1);
  }
}

template <class S>
__global__ void __launch_bounds__(256) imgprop_persistent(const typename S::Pix* __restrict__ in4, typename S::Pix* bwd,
                                                          typename S::Pix* fwd, const typename S::Flow* __restrict__ ff,
                                                          const typename S::Flow* __restrict__ fbk, int T, int H, int W,
                                                          const int* __restrict__ bbox, unsigned int* counter) {
  using Pix = typename S::Pix;
  using Flow = typename S::Flow;
  const int bx0 = bbox[0], by0 = bbox[1], bw = bbox[2] - bbox[0] + 1, bh = bbox[3] - bbox[1] + 1;
  if (bbox[2] < 0) return;                                  // no hole anywhere: outputs are the pre-copied inputs
  const int npix = bw * bh;
  const int nthreads = gridDim.x * blockDim.x, gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const long long HW = (long long)H * W;
  const int steps = 2 * (T - 1);
  auto bufs = [&](int s, const Pix*& cur, const Pix*& pin, Pix*& out, const Flow*& fprop, const Flow*& fchk) {
    if (s < T - 1) {          // backward pass: idx = T-2 .. 0, prop flow = forward flow, check = backward flow
      const int idx = T - 2 - s;
      cur = in4 + idx * HW; pin = bwd + (idx + 1) * HW; out = bwd + idx * HW; fprop = ff + idx * HW; fchk = fbk + idx * HW;
    } else {                  // forward pass over the backward pass's outputs: idx = 1 .. T-1
      const int idx = s - (T - 1) + 1;
      cur = bwd + idx * HW; pin = fwd + (idx - 1) * HW; out = fwd + idx * HW; fprop = fbk + (idx - 1) * HW; fchk = ff + (idx - 1) * HW;
    }
  };
  auto pixel_of = [&](int j) { return (by0 + j / bw) * W + bx0 + j % bw; };
  const Pix *cur, *pin;
  Pix* out;
  const Flow *fprop, *fchk;
  PropPre<S> pre;
  pre.pix = -1;
  if (gtid < npix) {
    bufs(0, cur, pin, out, fprop, fchk);
    pre = prop_pre<S>(cur, fprop, fchk, pixel_of(gtid), H, W, true);
  }
  for (int s = 0; s < steps; ++s) {
    bufs(s, cur, pin, out, fprop, fchk);
    const bool fwd_pass = s >= T - 1;
    // first pixel of this thread: its step-independent half was fetched before the previous barrier
    if (pre.pix >= 0) {
      if (pre.near != -2) {
        const Pix o = prop_post<S>(pre, pin, W);
        out[pre.pix] = o;
        if (s == T - 2) fwd[pre.pix] = o;                   // frame 0 of the forward pass is the backward result
      } else if (fwd_pass) {
        out[pre.pix] = pre.cur;                             // pass-through (backward pass: already the pre-copied input)
      } else if (s == T - 2) {
        fwd[pre.pix] = pre.cur;
      }
    }
    for (int j = gtid + nthreads; j < npix; j += nthreads) {   // holes larger than the grid: remaining pixels
      const PropPre<S> q = prop_pre<S>(cur, fprop, fchk, pixel_of(j), H, W, !fwd_pass);
      if (q.near != -2) {
        const Pix o = prop_post<S>(q, pin, W);
        out[q.pix] = o;
        if (s == T - 2) fwd[q.pix] = o;
      } else if (fwd_pass) {
        out[q.pix] = q.cur;
      } else if (s == T - 2) {
        fwd[q.pix] = q.cur;
      }
    }
    if (s + 1 < steps && gtid < npix) {
      const Pix *c2, *p2;
      Pix* o2;
      const Flow *f2, *k2;
      bufs(s + 1, c2, p2, o2, f2, k2);
      // in the forward pass `cur` is a backward-pass output of THIS thread (same pixel mapping), complete by now
      pre = prop_pre<S>(c2, f2, k2, pixel_of(gtid), H, W, s + 1 < T - 1);
    }
    ppx::grid_barrier(counter, (unsigned)(s + 1) * gridDim.x);
  }
}

// frames [T,3,H,W] f32 (already multiplied by (1-mask) here) + masks -> [T][H][W][4] fp16 / fp32
template <class S>
__global__ void imgprop_pack(const float* __restrict__ frames, const float* __restrict__ masks,
                             typename S::Pix* __restrict__ dst, long long HW, long long total) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const long long t = idx / HW, p = idx - t * HW;
  const float m = masks[idx];
  const float* f = frames + t * 3 * HW + p;
  const float k = 1.f - m;
  dst[idx] = S::make(f[0] * k, f[HW] * k, f[2 * HW] * k, m);
}

// updated = frames*(1-m) + prop*m ; updated mask = propagated mask   (propainter_inference.py:213-219)
template <class S>
__global__ void imgprop_finish(const typename S::Pix* __restrict__ prop, const float* __restrict__ frames,
                               const float* __restrict__ masks, float* __restrict__ uf, float* __restrict__ um,
                               long long HW, long long total) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const long long t = idx / HW, p = idx - t * HW;
  const typename S::Pix v = prop[idx];
  const float2 a = S::rg(v);
  const float2 c = S::bm(v);
  const float m = masks[idx], k = 1.f - m;
  const float* f = frames + t * 3 * HW + p;
  float* o = uf + t * 3 * HW + p;
  o[0] = f[0] * k + a.x * m;
  o[HW] = f[HW] * k + a.y * m;
  o[2 * HW] = f[2 * HW] * k + c.x * m;
  um[idx] = c.y;
}

// [n,2,H,W] f32 -> [n][H][W][2] fp16 / fp32
template <class S>
__global__ void flow_to_nhwc2(const float* __restrict__ src, typename S::Flow* __restrict__ dst, long long HW,
                              long long total) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const long long n = idx / HW, p = idx - n * HW;
  dst[idx] = S::make_flow(src[(n * 2) * HW + p], src[(n * 2 + 1) * HW + p]);
}

// ------------------------------------------------------------------------------------------------
// Flow completion input: cat(flow * (1 - mask), mask) per frame (recurrent_flow_completion.py:361-366, 320-323),
// optionally time-reversed (backward flows are flipped before the network, :375-376).  -> [T][H][W][8] fp16.
// ------------------------------------------------------------------------------------------------
__global__ void rfc_pack_input(const float* __restrict__ flows, const float* __restrict__ masks,
                               uint4* __restrict__ dst, int T, long long HW, int reverse, long long dst_tstride) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)T * HW) return;
  const long long t = idx / HW, p = idx - t * HW;
  const long long ts = reverse ? (T - 1 - t) : t;
  const float m = masks[ts * HW + p];
  const float k = 1.f - m;
  uint4 o = make_uint4(0, 0, 0, 0);
  *reinterpret_cast<__half2*>(&o.x) = __floats2half2_rn(flows[(ts * 2) * HW + p] * k, flows[(ts * 2 + 1) * HW + p] * k);
  *reinterpret_cast<__half2*>(&o.y) = __floats2half2_rn(m, 0.f);
  dst[t * dst_tstride + p] = o;
}

// The fp32 form (the node's fp16="disable"): the same four channels as a split-tf32 pixel [hi 4 | lo 4]
// (conv_igemm.cuh), the products rounded as torch's fp32 flows * (1 - masks) does.
__global__ void rfc_pack_input_f32(const float* __restrict__ flows, const float* __restrict__ masks,
                                   float4* __restrict__ dst, int T, long long HW, int reverse, long long dst_tstride) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)T * HW) return;
  const long long t = idx / HW, p = idx - t * HW;
  const long long ts = reverse ? (T - 1 - t) : t;
  const float m = masks[ts * HW + p];
  const float k = __fsub_rn(1.f, m);
  const float v[4] = {__fmul_rn(flows[(ts * 2) * HW + p], k), __fmul_rn(flows[(ts * 2 + 1) * HW + p], k), m, 0.f};
  float hi[4], lo[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) { hi[c] = ppx::tf32_rna(v[c]); lo[c] = __fsub_rn(v[c], hi[c]); }
  float4* d = dst + (t * dst_tstride + p) * 2;
  d[0] = make_float4(hi[0], hi[1], hi[2], hi[3]);
  d[1] = make_float4(lo[0], lo[1], lo[2], lo[3]);
}

// combine_flow (recurrent_flow_completion.py:389-400): out = pred*m + gt*(1-m), un-reversing time.
__global__ void rfc_combine(const __half* __restrict__ pred, int pred_cs, const float* __restrict__ gt,
                            const float* __restrict__ masks, float* __restrict__ out, int T, long long HW,
                            int reverse, long long pred_tstride) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)T * HW) return;
  const long long t = idx / HW, p = idx - t * HW;
  const long long ts = reverse ? (T - 1 - t) : t;  // network time index holding frame t
  const __half* pr = pred + (ts * pred_tstride + p) * pred_cs;
  const float m = masks[idx], k = 1.f - m;
  out[(t * 2) * HW + p] = __half2float(pr[0]) * m + gt[(t * 2) * HW + p] * k;
  out[(t * 2 + 1) * HW + p] = __half2float(pr[1]) * m + gt[(t * 2 + 1) * HW + p] * k;
}

// The fp32 form: plain fp32 pred [pix][pred_cs], torch's fp32 rounding (no contraction), so that outside the hole
// (m = 0) the result is the input flow itself.
__global__ void rfc_combine_f32(const float* __restrict__ pred, int pred_cs, const float* __restrict__ gt,
                                const float* __restrict__ masks, float* __restrict__ out, int T, long long HW,
                                int reverse, long long pred_tstride) {
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)T * HW) return;
  const long long t = idx / HW, p = idx - t * HW;
  const long long ts = reverse ? (T - 1 - t) : t;
  const float* pr = pred + (ts * pred_tstride + p) * pred_cs;
  const float m = masks[idx], k = __fsub_rn(1.f, m);
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const long long o = (t * 2 + c) * HW + p;
    out[o] = __fadd_rn(__fmul_rn(pr[c], m), __fmul_rn(gt[o], k));
  }
}

// ------------------------------------------------------------------------------------------------
// Modulated deformable sampling (torchvision.ops.deform_conv2d im2col stage; call sites
// recurrent_flow_completion.py:44-53 and propainter.py:73-82), 3x3, stride 1, pad 1, dil 1, 16 offset groups.
// offs row = raw output of conv_offset[-1]: channels [0,288) -> offsets, (g*9+k)*2+{0:dy,1:dx}, passed through
// max_mag*tanh (+ flow (dy,dx) for the feature path); channels [288,432) -> sigmoid modulation, g*9+k.
// cols[m][k*C + c] = mask * bilinear(x[c], y-1+ky+dy, x-1+kx+dx); zero outside (h<=-1 || h>=H ...).
// One thread per (pixel, tap, group): the 4 bilinear weights are computed once and applied to the
// group's C/16 contiguous channels with 16-byte loads.
// ------------------------------------------------------------------------------------------------
template <int CPG>  // channels per offset group: 8 or 16
__global__ void dcn_sample(const PPDcnArgs a) {
  // grid = (chunks of one image's H*W*144 (pixel, group, tap) items, images): 32-bit index math
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (unsigned)(a.H * a.W * 144)) return;
  dcn_sample_item<CPG, false>(a, idx, blockIdx.y);
}

// The fp32 form of dcn_sample for flow completion (16 groups of 16 channels, C = C0 + C1 = 256): inputs are split-tf32
// tensors [pix][hi C0 | lo C0] / [pix][hi C1 | lo C1] read as x = hi + lo (exact), offsets plain fp32, columns written
// split [pix][hi 9C | lo 9C].  Offset 5*tanh and the sigmoid modulation use the fp32-accurate ppx forms (tanhf / __expf
// are approximations under --use_fast_math); the bilinear weights and sums follow torchvision's CPU
// bilinear_interpolate ((w1*v1 + w2*v2) + w3*v3) + w4*v4 with every product and sum rounded on its own.
__global__ void dcn_sample_f32(const float* __restrict__ x0, int C0, const float* __restrict__ x1, int C1,
                               const float* __restrict__ offs, int offs_cs, float max_mag, float* __restrict__ cols,
                               int H, int W) {
  constexpr int CPG = 16;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (unsigned)(H * W * 144)) return;
  const int n = blockIdx.y, C = C0 + C1;
  const int gk = idx % 144u, pix = idx / 144u;
  const int g = gk / 9, k = gk - g * 9;
  const int x = pix % (unsigned)W, y = pix / (unsigned)W;
  const long long m = (long long)n * H * W + pix;
  const float* o = offs + m * offs_cs;
  const float dy = __fmul_rn(max_mag, ppx::tanh_acc(o[2 * gk]));
  const float dx = __fmul_rn(max_mag, ppx::tanh_acc(o[2 * gk + 1]));
  const float mod = __fdiv_rn(1.f, __fadd_rn(1.f, ppx::exp_acc(-o[288 + gk])));
  const float py = __fadd_rn((float)(y - 1 + k / 3), dy), px = __fadd_rn((float)(x - 1 + k % 3), dx);
  float* dhi = cols + m * (long long)(18 * C) + k * C + g * CPG;
  float* dlo = dhi + 9 * C;
  const bool inside = py > -1.f && py < (float)H && px > -1.f && px < (float)W;
  const int c = g * CPG;  // channel inside cat(x0, x1)
  const float* src;
  int Cs;
  if (c < C0) { src = x0 + c; Cs = C0; }
  else { src = x1 + (c - C0); Cs = C1; }
  src += (long long)n * H * W * 2 * Cs;
  const float fy = floorf(py), fx = floorf(px);
  const int yl = (int)fy, xl = (int)fx;
  const float lh = __fsub_rn(py, fy), lw = __fsub_rn(px, fx);
  const float hh = __fsub_rn(1.f, lh), hw = __fsub_rn(1.f, lw);
  const float wc[4] = {__fmul_rn(hh, hw), __fmul_rn(hh, lw), __fmul_rn(lh, hw), __fmul_rn(lh, lw)};
#pragma unroll
  for (int v = 0; v < CPG / 4; ++v) {
    float val[4] = {0.f, 0.f, 0.f, 0.f};
    if (inside) {
#pragma unroll
      for (int corner = 0; corner < 4; ++corner) {
        const int yy = yl + (corner >> 1), xx = xl + (corner & 1);
        float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
          const float* s = src + ((long long)yy * W + xx) * 2 * Cs + 4 * v;
          const float4 h = *reinterpret_cast<const float4*>(s), l = *reinterpret_cast<const float4*>(s + Cs);
          q = make_float4(__fadd_rn(h.x, l.x), __fadd_rn(h.y, l.y), __fadd_rn(h.z, l.z), __fadd_rn(h.w, l.w));
        }
        const float qv[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float t = __fmul_rn(wc[corner], qv[e]);
          val[e] = corner == 0 ? t : __fadd_rn(val[e], t);
        }
      }
    }
    float hi[4], lo[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float r = __fmul_rn(mod, val[e]);
      hi[e] = ppx::tf32_rna(r);
      lo[e] = __fsub_rn(r, hi[e]);
    }
    reinterpret_cast<float4*>(dhi)[v] = make_float4(hi[0], hi[1], hi[2], hi[3]);
    reinterpret_cast<float4*>(dlo)[v] = make_float4(lo[0], lo[1], lo[2], lo[3]);
  }
}

// ------------------------------------------------------------------------------------------------
// Learnable feature propagation, per step (model/propainter.py:157-176): fb check of the 1/4-res flows,
// bilinear warp of the propagated feature, and assembly of the DCN condition
//   cond = cat(cur[C], warped[C], flow[2], valid[1], mask_cur[2])  -> [H][W][2C+8] (3 pad channels = 0)
// One thread per (pixel, 8-channel vector of C); vector 0 also writes the 5 scalar channels.
// ------------------------------------------------------------------------------------------------
__global__ void featprop_cond(const __half* __restrict__ cur, int cur_cs, const __half* __restrict__ prop,
                              int prop_cs, const __half2* __restrict__ flow_prop,
                              const __half2* __restrict__ flow_check, const __half* __restrict__ mask2,
                              int mask_cs, __half* __restrict__ cond, int cond_cs, int N, int H, int W, int C) {
  const int C8 = C / 8;
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)N * H * W * C8) return;
  const int c8 = idx % C8;
  const long long pg = idx / C8;          // pixel over all N images
  const int HWi = H * W;
  const int img = pg / HWi;
  const int p = pg - (long long)img * HWi;  // pixel inside the image
  const int x = p % W, y = p / W;
  // re-base every per-image tensor
  cur += (long long)img * HWi * cur_cs;
  prop += (long long)img * HWi * prop_cs;
  flow_prop += (long long)img * HWi;
  flow_check += (long long)img * HWi;
  mask2 += (long long)img * HWi * mask_cs;
  cond += (long long)img * HWi * cond_cs;
  const float2 fp = __half22float2(flow_prop[p]);
  const float sx = sample_coord((float)x + fp.x, W), sy = sample_coord((float)y + fp.y, H);
  const Bilin b = bilin_setup(sx, sy, W, H);
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const float ws[4] = {b.w00, b.w01, b.w10, b.w11};
#pragma unroll
  for (int corner = 0; corner < 4; ++corner) {
    if (ws[corner] == 0.f) continue;
    const int yy = b.y0 + (corner >> 1), xx = b.x0 + (corner & 1);
    const uint4 q = *reinterpret_cast<const uint4*>(prop + ((long long)yy * W + xx) * prop_cs + c8 * 8);
    const __half2* hq = reinterpret_cast<const __half2*>(&q);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(hq[e]);
      acc[2 * e] += ws[corner] * f.x;
      acc[2 * e + 1] += ws[corner] * f.y;
    }
  }
  __half* cp = cond + (long long)p * cond_cs;
  *reinterpret_cast<uint4*>(cp + c8 * 8) = *reinterpret_cast<const uint4*>(cur + (long long)p * cur_cs + c8 * 8);
  __align__(16) __half2 h[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(acc[2 * e], acc[2 * e + 1]);
  *reinterpret_cast<uint4*>(cp + C + c8 * 8) = *reinterpret_cast<uint4*>(h);
  if (c8 == 0) {
    const float valid = fb_valid(fp, sample_flow2(flow_check, b, W));
    const float2 mk = __half22float2(*reinterpret_cast<const __half2*>(mask2 + (long long)p * mask_cs));
    __align__(16) __half2 s[4];
    s[0] = __floats2half2_rn(fp.x, fp.y);
    s[1] = __floats2half2_rn(valid, mk.x);
    s[2] = __floats2half2_rn(mk.y, 0.f);
    s[3] = __floats2half2_rn(0.f, 0.f);
    *reinterpret_cast<uint4*>(cp + 2 * C) = *reinterpret_cast<uint4*>(s);
  }
}

// F.interpolate(scale_factor=1/4, bilinear, align_corners=False) == mean of the centre 2x2 of each 4x4 block;
// the reference then divides the flow by 4 (propainter.py:389-406).  [n,2,H,W] f32 -> [n][H/4][W/4][2] fp16.
__global__ void downsample_flow4(const float* __restrict__ src, __half2* __restrict__ dst, int n, int H, int W) {
  const int h = H / 4, w = W / 4;
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)n * h * w) return;
  const int x = idx % w;
  long long t = idx / w;
  const int y = t % h;
  const int i = t / h;
  float v[2];
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const float* s = src + ((long long)(i * 2 + c) * H + 4 * y + 1) * W + 4 * x + 1;
    v[c] = 0.25f * (0.25f * (s[0] + s[1] + s[W] + s[W + 1]));
  }
  dst[idx] = __floats2half2_rn(v[0], v[1]);
}

// F.interpolate(scale_factor=1/4, 'nearest') picks source index 4*i.  [n,1,H,W] f32 -> fp16 slice.
__global__ void downsample_mask4(const float* __restrict__ src, __half* __restrict__ dst, int dst_cs, int dst_co,
                                 int n, int H, int W) {
  const int h = H / 4, w = W / 4;
  long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)n * h * w) return;
  const int x = idx % w;
  long long t = idx / w;
  const int y = t % h;
  const int i = t / h;
  dst[idx * dst_cs + dst_co] = __float2half_rn(src[((long long)i * H + 4 * y) * W + 4 * x]);
}

}  // namespace

template <class E>
int pp_k_imgprop_step(const E* cur, const E* prop_in, E* prop_out, const E* flow_prop, const E* flow_check, int H,
                      int W, cudaStream_t st) {
  using S = ImgOf<E>;
  using Pix = typename S::Pix;
  using Flow = typename S::Flow;
  imgprop_step<S><<<nblocks((long long)H * W), TPB, 0, st>>>(
      reinterpret_cast<const Pix*>(cur), reinterpret_cast<const Pix*>(prop_in), reinterpret_cast<Pix*>(prop_out),
      reinterpret_cast<const Flow*>(flow_prop), reinterpret_cast<const Flow*>(flow_check), H, W);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}
template int pp_k_imgprop_step(const __half*, const __half*, __half*, const __half*, const __half*, int, int, cudaStream_t);
template int pp_k_imgprop_step(const float*, const float*, float*, const float*, const float*, int, int, cudaStream_t);

template <class E>
int pp_k_imgprop_run(const E* in4, E* bwd, E* fwd, const E* ff, const E* fbk, const float* masks, int T, int H, int W,
                     int* scratch, cudaStream_t st) {
  using S = ImgOf<E>;
  static int grid_max = 0;      // one per storage type: the fp32 kernel has its own register footprint
  if (grid_max == 0) {
    int sms = 0, per_sm = 0;
    PP_TRY(pp_num_sms(&sms));
    PP_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, imgprop_persistent<S>, 256, 0));
    PP_REQUIRE(per_sm >= 1, "imgprop: persistent kernel does not fit an SM");
    grid_max = sms * (per_sm < 2 ? per_sm : 2);
  }
  const int init[8] = {W, H, -1, -1, 0, 0, 0, 0};
  PP_CUDA_CHECK(cudaMemcpyAsync(scratch, init, sizeof(init), cudaMemcpyHostToDevice, st));
  const long long total = (long long)T * H * W;
  const long long want = (total + 256 * 16 - 1) / (256 * 16);
  mask_bbox<<<(int)(want < 1184 ? want : 1184), 256, 0, st>>>(masks, total, H * W, W, scratch);
  PP_CUDA_CHECK(cudaGetLastError());
  using Pix = typename S::Pix;
  using Flow = typename S::Flow;
  const Pix* a0 = reinterpret_cast<const Pix*>(in4);
  Pix* a1 = reinterpret_cast<Pix*>(bwd);
  Pix* a2 = reinterpret_cast<Pix*>(fwd);
  const Flow* a3 = reinterpret_cast<const Flow*>(ff);
  const Flow* a4 = reinterpret_cast<const Flow*>(fbk);
  const int* a8 = scratch;
  unsigned int* a9 = reinterpret_cast<unsigned int*>(scratch + 4);
  void* args[] = {&a0, &a1, &a2, &a3, &a4, &T, &H, &W, &a8, &a9};
  PP_CUDA_CHECK(cudaLaunchCooperativeKernel((const void*)imgprop_persistent<S>, dim3(grid_max), dim3(256), args, 0, st));
  return PP_OK;
}
template int pp_k_imgprop_run(const __half*, __half*, __half*, const __half*, const __half*, const float*, int, int, int,
                              int*, cudaStream_t);
template int pp_k_imgprop_run(const float*, float*, float*, const float*, const float*, const float*, int, int, int, int*,
                              cudaStream_t);

template <class E>
int pp_k_imgprop_pack(const float* frames, const float* masks, E* dst, int T, int H, int W, cudaStream_t st) {
  using S = ImgOf<E>;
  const long long HW = (long long)H * W, total = HW * T;
  imgprop_pack<S><<<nblocks(total), TPB, 0, st>>>(frames, masks, reinterpret_cast<typename S::Pix*>(dst), HW, total);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}
template int pp_k_imgprop_pack(const float*, const float*, __half*, int, int, int, cudaStream_t);
template int pp_k_imgprop_pack(const float*, const float*, float*, int, int, int, cudaStream_t);

template <class E>
int pp_k_imgprop_finish(const E* prop, const float* frames, const float* masks, float* upd_frames, float* upd_masks,
                        int T, int H, int W, cudaStream_t st) {
  using S = ImgOf<E>;
  const long long HW = (long long)H * W, total = HW * T;
  imgprop_finish<S><<<nblocks(total), TPB, 0, st>>>(reinterpret_cast<const typename S::Pix*>(prop), frames, masks,
                                                    upd_frames, upd_masks, HW, total);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}
template int pp_k_imgprop_finish(const __half*, const float*, const float*, float*, float*, int, int, int, cudaStream_t);
template int pp_k_imgprop_finish(const float*, const float*, const float*, float*, float*, int, int, int, cudaStream_t);

template <class E>
int pp_k_flow_to_nhwc2(const float* src, E* dst, int n, int H, int W, cudaStream_t st) {
  using S = ImgOf<E>;
  const long long HW = (long long)H * W, total = HW * n;
  if (total == 0) return PP_OK;
  flow_to_nhwc2<S><<<nblocks(total), TPB, 0, st>>>(src, reinterpret_cast<typename S::Flow*>(dst), HW, total);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}
template int pp_k_flow_to_nhwc2(const float*, __half*, int, int, int, cudaStream_t);
template int pp_k_flow_to_nhwc2(const float*, float*, int, int, int, cudaStream_t);

int pp_k_rfc_pack_input(const float* flows, const float* masks, __half* dst, long long dst_tstride_pix, int T, int H,
                        int W, int reverse_time, cudaStream_t st) {
  const long long HW = (long long)H * W;
  rfc_pack_input<<<nblocks(HW * T), TPB, 0, st>>>(flows, masks, reinterpret_cast<uint4*>(dst), T, HW, reverse_time,
                                                  dst_tstride_pix);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_rfc_combine(const __half* pred, int pred_cs, long long pred_tstride_pix, const float* gt, const float* masks,
                     float* out, int T, int H, int W, int reverse_time, cudaStream_t st) {
  const long long HW = (long long)H * W;
  rfc_combine<<<nblocks(HW * T), TPB, 0, st>>>(pred, pred_cs, gt, masks, out, T, HW, reverse_time, pred_tstride_pix);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_dcn_sample(const __half* x0, int x0_cs, int x0_co, int C0, const __half* x1, int x1_cs, int x1_co, int C1,
                    const __half* offs, int offs_cs, const __half* flow, int flow_cs, int flow_co, float max_mag,
                    __half* cols, int N, int H, int W, cudaStream_t st) {
  const int C = C0 + C1;
  PP_REQUIRE(C == 128 || C == 256, "dcn_sample: C=%d must be 128 or 256 (16 offset groups)", C);
  PP_REQUIRE(C0 % 16 == 0, "dcn_sample: C0=%d", C0);
  if ((long long)N * H * W == 0) return PP_OK;
  PP_REQUIRE(N <= 65535 && (long long)H * W * 144 < (1LL << 31), "dcn_sample: %d images of %dx%d exceed the grid limits", N, W, H);
  PPDcnArgs a;
  a.x0 = x0; a.x0_cs = x0_cs; a.x0_co = x0_co; a.C0 = C0;
  a.x1 = x1; a.x1_cs = x1_cs; a.x1_co = x1_co;
  a.offs = offs; a.offs_cs = offs_cs;
  a.flow = flow; a.flow_cs = flow_cs; a.flow_co = flow_co;
  a.max_mag = max_mag; a.cols = cols; a.C = C; a.N = N; a.H = H; a.W = W;
  if (pp_prog_recording()) return pp_prog_record_dcn(a);     // multi-layer program (conv_halo.cu): runs inside it
  const dim3 grid(pp_ceil_div(H * W * 144, TPB), N);
  if (C == 128) dcn_sample<8><<<grid, TPB, 0, st>>>(a);
  else dcn_sample<16><<<grid, TPB, 0, st>>>(a);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_rfc_pack_input(const float* flows, const float* masks, float* dst, long long dst_tstride_pix, int T, int H,
                        int W, int reverse_time, cudaStream_t st) {
  const long long HW = (long long)H * W;
  if (HW * T == 0) return PP_OK;
  rfc_pack_input_f32<<<nblocks(HW * T), TPB, 0, st>>>(flows, masks, reinterpret_cast<float4*>(dst), T, HW, reverse_time,
                                                      dst_tstride_pix);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_rfc_combine(const float* pred, int pred_cs, long long pred_tstride_pix, const float* gt, const float* masks,
                     float* out, int T, int H, int W, int reverse_time, cudaStream_t st) {
  const long long HW = (long long)H * W;
  if (HW * T == 0) return PP_OK;
  rfc_combine_f32<<<nblocks(HW * T), TPB, 0, st>>>(pred, pred_cs, gt, masks, out, T, HW, reverse_time, pred_tstride_pix);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_dcn_sample(const float* x0, int C0, const float* x1, int C1, const float* offs, int offs_cs, float max_mag,
                    float* cols, int N, int H, int W, cudaStream_t st) {
  PP_REQUIRE(C0 + C1 == 256 && C0 % 16 == 0, "dcn_sample (fp32): C0=%d C1=%d must be 16-channel groups of 256", C0, C1);
  PP_REQUIRE((C1 == 0 || x1 != nullptr) && x0 != nullptr && offs != nullptr && cols != nullptr,
             "dcn_sample (fp32): null pointer");
  if ((long long)N * H * W == 0) return PP_OK;
  PP_REQUIRE(N <= 65535 && (long long)H * W * 144 < (1LL << 31), "dcn_sample: %d images of %dx%d exceed the grid limits", N, W, H);
  const dim3 grid(pp_ceil_div(H * W * 144, TPB), N);
  dcn_sample_f32<<<grid, TPB, 0, st>>>(x0, C0, x1, C1, offs, offs_cs, max_mag, cols, H, W);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_featprop_cond(const __half* cur, int cur_cs, const __half* prop, int prop_cs, const __half* flow_prop,
                       const __half* flow_check, const __half* mask2, int mask_cs, __half* cond, int cond_cs, int N,
                       int H, int W, int C, cudaStream_t st) {
  PP_REQUIRE(C % 8 == 0 && cond_cs >= 2 * C + 8, "featprop_cond: bad channel counts");
  featprop_cond<<<nblocks((long long)N * H * W * (C / 8)), TPB, 0, st>>>(
      cur, cur_cs, prop, prop_cs, reinterpret_cast<const __half2*>(flow_prop),
      reinterpret_cast<const __half2*>(flow_check), mask2, mask_cs, cond, cond_cs, N, H, W, C);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_downsample_flow4(const float* flow, __half* dst, int n, int H, int W, cudaStream_t st) {
  const long long total = (long long)n * (H / 4) * (W / 4);
  if (total == 0) return PP_OK;
  downsample_flow4<<<nblocks(total), TPB, 0, st>>>(flow, reinterpret_cast<__half2*>(dst), n, H, W);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

int pp_k_downsample_mask4(const float* m, __half* dst, int dst_cs, int dst_co, int n, int H, int W, cudaStream_t st) {
  const long long total = (long long)n * (H / 4) * (W / 4);
  if (total == 0) return PP_OK;
  downsample_mask4<<<nblocks(total), TPB, 0, st>>>(m, dst, dst_cs, dst_co, n, H, W);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}

// Modulated deformable sampling (torchvision.ops.deform_conv2d im2col stage; call sites
// recurrent_flow_completion.py:44-53 and propainter.py:73-82), 3x3, stride 1, pad 1, dil 1, 16 offset groups.
// One work item = one (pixel, offset group, tap): the 4 bilinear weights are computed once and applied to the group's
// C/16 contiguous channels with 16-byte loads.  Shared by the stand-alone kernel (kernels_prop.cu) and the multi-layer
// program kernel (conv_halo.cu), where the inputs were written by other SMs earlier in the same kernel and therefore
// must be read through L2 (COHERENT = ld.global.cg).
#pragma once
#include "pp_common.cuh"

struct PPDcnArgs {
  const __half* x0; int x0_cs, x0_co, C0;
  const __half* x1; int x1_cs, x1_co;
  const __half* offs; int offs_cs;
  const __half* flow; int flow_cs, flow_co;
  float max_mag;
  __half* cols;
  int C, N, H, W;
};

template <bool COHERENT>
__device__ __forceinline__ float dcn_ldh(const __half* p) {
  if (COHERENT) {
    const unsigned short u = __ldcg(reinterpret_cast<const unsigned short*>(p));
    return __half2float(__ushort_as_half(u));
  }
  return __half2float(*p);
}

// idx in [0, H*W*144): (pixel, g*9 + k); n = image
template <int CPG, bool COHERENT>
__device__ __forceinline__ void dcn_sample_item(const PPDcnArgs& a, unsigned idx, int n) {
  const int H = a.H, W = a.W, C = a.C;
  const int gk = idx % 144u;           // g*9 + k  (g-major like the offset channels)
  const int pix = idx / 144u;
  const int g = gk / 9, k = gk - g * 9;
  const int x = pix % (unsigned)W, y = pix / (unsigned)W;
  const long long m = (long long)n * H * W + pix;
  const __half* o = a.offs + m * a.offs_cs;
  float dy = a.max_mag * tanhf(dcn_ldh<COHERENT>(o + 2 * gk));
  float dx = a.max_mag * tanhf(dcn_ldh<COHERENT>(o + 2 * gk + 1));
  if (a.flow != nullptr) {
    dx += dcn_ldh<COHERENT>(a.flow + m * a.flow_cs + a.flow_co);
    dy += dcn_ldh<COHERENT>(a.flow + m * a.flow_cs + a.flow_co + 1);
  }
  const float mod = 1.f / (1.f + __expf(-dcn_ldh<COHERENT>(o + 288 + gk)));
  const float py = (float)(y - 1 + k / 3) + dy, px = (float)(x - 1 + k % 3) + dx;
  float acc[CPG];
#pragma unroll
  for (int i = 0; i < CPG; ++i) acc[i] = 0.f;
  if (py > -1.f && py < (float)H && px > -1.f && px < (float)W) {
    const float fy = floorf(py), fx = floorf(px);
    const int y0 = (int)fy, xx0 = (int)fx;
    const float ay = py - fy, ax = px - fx;
    const int c = g * CPG;  // channel inside cat(x0, x1)
    const __half* src;
    int cs;
    if (c < a.C0) { src = a.x0 + a.x0_co + c; cs = a.x0_cs; }
    else { src = a.x1 + a.x1_co + (c - a.C0); cs = a.x1_cs; }
    src += (long long)n * H * W * cs;
#pragma unroll
    for (int corner = 0; corner < 4; ++corner) {
      const int yy = y0 + (corner >> 1), xx = xx0 + (corner & 1);
      if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
      const float w = ((corner >> 1) ? ay : 1.f - ay) * ((corner & 1) ? ax : 1.f - ax);
      const uint4* vp = reinterpret_cast<const uint4*>(src + ((long long)yy * W + xx) * cs);
      uint4 qv[CPG / 8];
#pragma unroll
      for (int v = 0; v < CPG / 8; ++v) qv[v] = COHERENT ? __ldcg(vp + v) : vp[v];
#pragma unroll
      for (int v = 0; v < CPG / 8; ++v) {
        const __half2* hq = reinterpret_cast<const __half2*>(&qv[v]);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(hq[e]);
          acc[v * 8 + 2 * e] += w * f.x;
          acc[v * 8 + 2 * e + 1] += w * f.y;
        }
      }
    }
  }
  __half* d = a.cols + m * (long long)(9 * C) + k * C + g * CPG;
  __align__(16) __half2 h[CPG / 2];
#pragma unroll
  for (int e = 0; e < CPG / 2; ++e) h[e] = __floats2half2_rn(mod * acc[2 * e], mod * acc[2 * e + 1]);
#pragma unroll
  for (int v = 0; v < CPG / 8; ++v) reinterpret_cast<uint4*>(d)[v] = reinterpret_cast<uint4*>(h)[v];
}

// Sparse window attention of the temporal transformer (SparseWindowAttention.forward,
// model/modules/sparse_transformer.py:201-393) as a flash-style kernel: no window / rolled / pooled K,V
// tensors are materialised -- keys are gathered by index straight from the token grid.
//
// Per (window, head):
//   masked window   : queries = all t*45 window tokens; keys = for every 2nd frame (T_ind parity):
//                     45 own tokens + 148 ring tokens (circularly rolled neighbours) + n_pool pooled tokens
//   unmasked window : per frame, 45 queries x its own 45 keys
// scale 1/sqrt(128), softmax, PV.  fp16 operands, fp32 accumulation and softmax statistics.
//
// This file: warp-level mma.sync.m16n8k16 kernel used for the UNMASKED windows (45 queries x 45 keys per frame,
// a shape far below a wgmma tile); masked windows -- where the FLOPs are -- run on the wgmma kernel
// in attention_tc.cu.  CTA = 4 warps = 64 query rows, key tiles of 64.
#include "attention.cuh"
#include "kernels.cuh"

namespace {

constexpr int D = 128;      // head dim
constexpr int BQ = 64;      // query rows per CTA
constexpr int BKEY = 64;    // keys per tile
constexpr int NT = 128;     // threads
constexpr int WIN_TOK = 45; // 5 x 9
constexpr int RING = 193;   // 45 own + 148 ring indices per window

using AttnParams = PPAttnParams;

__device__ __forceinline__ uint32_t swz(int row, int chunk) {  // byte offset of a 16-byte chunk in a [rows][128] tile
  return (uint32_t)(row * 256 + ((chunk ^ (row & 7)) << 4));
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __launch_bounds__(NT) window_attention(const AttnParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  uint8_t* sQ = smem;                    // 64 x 256 B
  uint8_t* sK = smem + BQ * 256;         // 2 stages x 64 x 256 B
  uint8_t* sV = sK + 2 * BKEY * 256;     // 2 stages
  const int win = blockIdx.y >> 2, head = blockIdx.y & 3;
  const int sw = blockIdx.z;                 // sliding window of the batch
  const int t = p.sw_t[sw];
  const int frame_base = p.sw_frame_off[sw];
  const int n_tind = (t - p.parity + 1) / 2;
  const bool masked = p.win_flags[sw * p.n_win + win] != 0;
  if (masked && p.only_unmasked) return;     // masked windows run on the wgmma kernel (attention_tc.cu)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  int nq, nk, q_frame0;
  if (masked) {
    nq = t * WIN_TOK;
    if ((int)blockIdx.x * BQ >= nq) return;
    nk = n_tind * (RING + p.n_pool);
    q_frame0 = frame_base;
  } else {
    if ((int)blockIdx.x >= t) return;
    nq = WIN_TOK;
    nk = WIN_TOK;
    q_frame0 = frame_base + blockIdx.x;
  }
  const int q0 = masked ? blockIdx.x * BQ : 0;
  const int* ring = p.ring_idx + win * RING;
  const long long ntok = (long long)p.nh * p.nw;
  const int kpf = RING + p.n_pool;

  // ---- Q tile -> smem (rows beyond nq are clamped; never stored)
  for (int i = tid; i < BQ * 16; i += NT) {
    const int r = i >> 4, ch = i & 15;
    int qi = min(q0 + r, nq - 1);
    const int fr = q_frame0 + qi / WIN_TOK, pos = qi % WIN_TOK;
    const __half* src = p.q + ((long long)fr * ntok + ring[pos]) * p.qkv_cs + head * D + ch * 8;
    ppx::cp_async16(ppx::smem_u32(sQ) + swz(r, ch), src, 16);
  }
  ppx::cp_async_commit();

  auto load_kv = [&](int tile, int stage) {
    for (int i = tid; i < BKEY * 16; i += NT) {
      const int r = i >> 4, ch = i & 15;
      const int j = tile * BKEY + r;
      const __half* ks = p.k; const __half* vs = p.v;
      uint32_t nbytes = 0;
      if (j < nk) {
        nbytes = 16;
        int fr, w;
        if (masked) { const int fi = j / kpf; w = j - fi * kpf; fr = frame_base + p.parity + 2 * fi; }
        else { fr = q_frame0; w = j; }
        if (w < RING) {
          const long long off = ((long long)fr * ntok + ring[w]) * p.qkv_cs + head * D + ch * 8;
          ks = p.k + off; vs = p.v + off;
        } else {
          const long long off = ((long long)fr * p.n_pool + (w - RING)) * p.pool_cs + head * D + ch * 8;
          ks = p.pk + off; vs = p.pv + off;
        }
      }
      ppx::cp_async16(ppx::smem_u32(sK + stage * BKEY * 256) + swz(r, ch), ks, nbytes);
      ppx::cp_async16(ppx::smem_u32(sV + stage * BKEY * 256) + swz(r, ch), vs, nbytes);
    }
    ppx::cp_async_commit();
  };

  const int ntiles = (nk + BKEY - 1) / BKEY;
  load_kv(0, 0);

  float o[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float row_max[2] = {-1e30f, -1e30f}, row_sum[2] = {0.f, 0.f};
  uint32_t qf[8][4];

  for (int tile = 0; tile < ntiles; ++tile) {
    const int stage = tile & 1;
    if (tile + 1 < ntiles) { load_kv(tile + 1, stage ^ 1); ppx::cp_async_wait<1>(); }
    else { ppx::cp_async_wait<0>(); }
    __syncthreads();
    if (tile == 0) {
#pragma unroll
      for (int ks = 0; ks < 8; ++ks)
        ldsm_x4(ppx::smem_u32(sQ) + swz(warp * 16 + (lane & 15), ks * 2 + (lane >> 4)), qf[ks]);
    }
    const uint32_t kbase = ppx::smem_u32(sK + stage * BKEY * 256);
    const uint32_t vbase = ppx::smem_u32(sV + stage * BKEY * 256);
    // ---- S = Q K^T  (16 x 64 per warp)
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {  // pairs of 8-key n-tiles
        uint32_t b[4];
        ldsm_x4(kbase + swz(np * 16 + (lane & 7) + ((lane >> 4) << 3), ks * 2 + ((lane >> 3) & 1)), b);
        mma16816(s[2 * np], qf[ks], b[0], b[1]);
        mma16816(s[2 * np + 1], qf[ks], b[2], b[3]);
      }
    }
    // ---- online softmax (rows g and g+8 of the warp's 16)
    const int kcol0 = tile * BKEY + 2 * (lane & 3);
    float tmax[2] = {-1e30f, -1e30f};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = kcol0 + nt * 8 + (e & 1);
        float x = s[nt][e] * p.scale_log2;
        if (col >= nk) x = -1e30f;
        s[nt][e] = x;
        tmax[e >> 1] = fmaxf(tmax[e >> 1], x);
      }
    }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 1));
      tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 2));
      const float nm = fmaxf(row_max[r], tmax[r]);
      corr[r] = exp2f(row_max[r] - nm);
      row_max[r] = nm;
      row_sum[r] *= corr[r];
    }
    uint32_t pf[4][4];  // P as A fragments: 4 k-steps of 16 keys
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = exp2f(s[nt][0] - row_max[0]), p1 = exp2f(s[nt][1] - row_max[0]);
      const float p2 = exp2f(s[nt][2] - row_max[1]), p3 = exp2f(s[nt][3] - row_max[1]);
      row_sum[0] += p0 + p1;
      row_sum[1] += p2 + p3;
      pf[nt >> 1][(nt & 1) * 2] = pack_h2(p0, p1);
      pf[nt >> 1][(nt & 1) * 2 + 1] = pack_h2(p2, p3);
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) { o[i][0] *= corr[0]; o[i][1] *= corr[0]; o[i][2] *= corr[1]; o[i][3] *= corr[1]; }
    // ---- O += P V
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int dp = 0; dp < 8; ++dp) {  // pairs of 8-wide d tiles
        uint32_t b[4];
        ldsm_x4_t(vbase + swz(ks * 16 + (lane & 15), dp * 2 + (lane >> 4)), b);
        mma16816(o[2 * dp], pf[ks], b[0], b[1]);
        mma16816(o[2 * dp + 1], pf[ks], b[2], b[3]);
      }
    }
    __syncthreads();
  }

  // ---- normalise and store (unpadded grid; padding queries are dropped)
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float sum = row_sum[r];
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    const float inv = 1.f / sum;
    const int qi = q0 + warp * 16 + (lane >> 2) + r * 8;
    if (qi >= nq) continue;
    const int fr = q_frame0 + qi / WIN_TOK, pos = qi % WIN_TOK;
    const int tok = ring[pos];
    const int ty = tok / p.nw, tx = tok - ty * p.nw;
    if (ty >= p.gh || tx >= p.gw) continue;
    __half* dst = p.out + (((long long)fr * p.gh + ty) * p.gw + tx) * p.out_cs + head * D + 2 * (lane & 3);
#pragma unroll
    for (int nt = 0; nt < 16; ++nt)
      *reinterpret_cast<__half2*>(dst + nt * 8) = __floats2half2_rn(o[nt][2 * r] * inv, o[nt][2 * r + 1] * inv);
  }
}

}  // namespace

int pp_k_attention(const __half* q, const __half* k, const __half* v, int qkv_cs, const __half* pk, const __half* pv,
                   int pool_cs, __half* out, int out_cs, const int* win_flags, const int* ring_idx,
                   const int* sw_frame_off, const int* sw_t, int n_sliding, int t_max, int gh, int gw, int nh, int nw,
                   int n_pool, int t_parity, int* key_tab, int key_tab_stride, cudaStream_t st) {
  PP_REQUIRE(nh % 5 == 0 && nw % 9 == 0, "attention: padded grid %dx%d is not a multiple of the 5x9 window", nh, nw);
  AttnParams p;
  p.q = q; p.k = k; p.v = v; p.qkv_cs = qkv_cs; p.pk = pk; p.pv = pv; p.pool_cs = pool_cs;
  p.out = out; p.out_cs = out_cs; p.win_flags = win_flags; p.ring_idx = ring_idx;
  p.sw_frame_off = sw_frame_off; p.sw_t = sw_t;
  p.gh = gh; p.gw = gw; p.nh = nh; p.nw = nw; p.nww = nw / 9; p.n_pool = n_pool; p.parity = t_parity;
  p.n_win = (nh / 5) * (nw / 9);
  p.scale_log2 = 1.4426950408889634f / sqrtf((float)D);
  p.only_unmasked = 1;
  p.key_tab = key_tab; p.key_tab_stride = key_tab_stride;
  PP_TRY(pp_launch_attention_tc(p, n_sliding, t_max, st));   // masked windows: wgmma
  dim3 grid(t_max, p.n_win * 4, n_sliding);                  // unmasked windows: one 45x45 problem per frame
  const size_t smem = (size_t)(BQ + 4 * BKEY) * 256;
  static bool attr_set = false;
  if (!attr_set) {
    PP_CUDA_CHECK(cudaFuncSetAttribute(window_attention, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = true;
  }
  window_attention<<<grid, NT, smem, st>>>(p);
  PP_CUDA_CHECK(cudaGetLastError());
  return PP_OK;
}
